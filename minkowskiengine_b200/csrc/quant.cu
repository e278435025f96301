// fp8 operands of the e4m3 forward (meb200_conv_forward_fp8): per-tensor quantisation of the features
// and per-output-channel quantisation of the weights; and of the fp8 dgrad (meb200_conv_dgrad_fp8):
// per-tensor e5m2 quantisation of the output gradient and per-input-channel e4m3 weights.
//
// All use the same arithmetic, so that a torch expression reproduces the bytes exactly (e4m3 below;
// e5m2 the same with 57344, its largest finite value, in place of 448):
//   amax  = max |x| over the finite values (a max is exact and order-free: deterministic)
//   scale = amax / 448, inv = 448 / amax                 (both IEEE divisions, rounded to nearest)
//           scale = inv = 1 when amax = 0
//           inv = FLT_MAX, scale = 1 / FLT_MAX when 448 / amax overflows (amax < 448 / FLT_MAX):
//           scale stays the reciprocal of inv, so that q * scale still approximates x
//   q     = cvt.rn.satfinite.e4m3(x * inv)                (the product rounded to nearest in fp32)
// x * inv lies within rounding of [-448, 448] for a finite x, so the conversion rounds to nearest
// even; +-inf saturates to +-448 and NaN stays NaN.  448 is the largest finite e4m3 value.
#include <float.h>

#include <algorithm>

#include "common.cuh"
#include "conv_tc.cuh"
#include "fp8.cuh"

namespace meb200 {

constexpr uint32_t kQThreads = 256;
constexpr uint32_t kQMaxCtas = 1024;

// The max of every thread's m over the CTA, valid in thread 0 (the other threads return false).
__device__ __forceinline__ bool cta_max(float m, float &m_out) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, d));
  __shared__ float wm[kQThreads / 32];
  if ((threadIdx.x & 31) == 0) wm[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x != 0) return false;
  for (uint32_t w = 1; w < kQThreads / 32; ++w) m = fmaxf(m, wm[w]);
  m_out = m;
  return true;
}

// The CTA's max, valid in thread 0 (the other threads return false).
template <typename T, bool VEC>
__device__ __forceinline__ bool cta_amax(const T *__restrict__ x, uint64_t count, float &m_out) {
  constexpr uint32_t V = VEC ? 16 / sizeof(T) : 1;
  float m = 0.f;
  const uint64_t n_vec = count / V, stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n_vec; i += stride) {
    float f[V];
    load_f32<T, V>(x + i * V, f);
#pragma unroll
    for (uint32_t j = 0; j < V; ++j) m = fmaxf(m, finite_abs(f[j]));
  }
  if (blockIdx.x == 0)                                    // elements past the last vector
    for (uint64_t i = n_vec * V + threadIdx.x; i < count; i += blockDim.x)
      m = fmaxf(m, finite_abs(to_f32<T>(x[i])));
  return cta_max(m, m_out);
}

// Launch 1: per-CTA max of |x| over the finite values, combined with an atomic max on the fp32 bits
// (non-negative floats order as their bit patterns).  The last CTA to finish writes scale[0] = scale,
// scale[1] = inv and leaves the workspace zero again.  ws: [0] amax bits, [1] CTAs done (a ticket
// that wraps to 0 at the last CTA).
template <typename T, bool VEC, typename F>
__global__ void __launch_bounds__(kQThreads) k_amax(const T *__restrict__ x, uint64_t count,
                                                   float *__restrict__ scale, uint32_t *ws) {
  float m;
  if (!cta_amax<T, VEC>(x, count, m)) return;
  atomicMax(ws, __float_as_uint(m));
  __threadfence();
  if (atomicInc(ws + 1, gridDim.x - 1) != gridDim.x - 1) return;
  const float amax = __uint_as_float(atomicExch(ws, 0u));  // every CTA's max has landed
  float s, inv;
  fp8_scales<F>(amax, s, inv);
  scale[0] = s;
  scale[1] = inv;
}

// Launch 2: q = fp8(x * inv), 16 elements (16 output bytes) per thread and step.  RECORD: also
// returns the thread's max |x| over the finite values it converted (else 0, computed by nothing).
template <typename T, bool VEC, typename F, bool RECORD>
__device__ __forceinline__ float quant_body(const T *__restrict__ x, uint64_t count, float inv,
                                            uint8_t *__restrict__ q) {
  float m = 0.f;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  if constexpr (VEC) {
    constexpr uint32_t V = 16 / sizeof(T);
    const uint64_t n16 = count / 16;
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n16; i += stride) {
      uint32_t w[4];
#pragma unroll
      for (uint32_t h = 0; h < 16 / V; ++h) {
        float f[V];
        load_f32<T, V>(x + i * 16 + h * V, f);
#pragma unroll
        for (uint32_t j = 0; j < V; j += 2) {
          const uint32_t e = h * V + j;           // element of the 16: byte e of the store
          const uint32_t b = F::cvt2(__fmul_rn(f[j], inv), __fmul_rn(f[j + 1], inv));
          if (e % 4 == 0) w[e / 4] = b; else w[e / 4] |= b << 16;
          if (RECORD) m = fmaxf(m, fmaxf(finite_abs(f[j]), finite_abs(f[j + 1])));
        }
      }
      *reinterpret_cast<uint4 *>(q + i * 16) = make_uint4(w[0], w[1], w[2], w[3]);
    }
    if (blockIdx.x == 0)
      for (uint64_t i = n16 * 16 + threadIdx.x; i < count; i += blockDim.x) {
        const float v = to_f32<T>(x[i]);
        q[i] = fp8_byte<F>(v, inv);
        if (RECORD) m = fmaxf(m, finite_abs(v));
      }
  } else {
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < count; i += stride) {
      const float v = to_f32<T>(x[i]);
      q[i] = fp8_byte<F>(v, inv);
      if (RECORD) m = fmaxf(m, finite_abs(v));
    }
  }
  return m;
}

template <typename T, bool VEC, typename F>
__global__ void __launch_bounds__(kQThreads) k_quant(const T *__restrict__ x, uint64_t count,
                                                    const float *__restrict__ scale,
                                                    uint8_t *__restrict__ q) {
  quant_body<T, VEC, F, false>(x, count, __ldg(scale + 1), q);
}

// Convert and record (delayed scaling): k_quant at the given scale, and the CTA's max |x| over the
// finite values atomically maxed into *slot (fp32 bits), in the same pass.
template <typename T, bool VEC, typename F>
__global__ void __launch_bounds__(kQThreads) k_quant_record(const T *__restrict__ x,
                                                           uint64_t count,
                                                           const float *__restrict__ scale,
                                                           uint8_t *__restrict__ q,
                                                           uint32_t *slot) {
  float m;
  if (cta_max(quant_body<T, VEC, F, true>(x, count, __ldg(scale + 1), q), m))
    atomicMax(slot, __float_as_uint(m));
}

uint64_t quantize_e4m3_workspace_bytes() { return 16; }

static uint32_t quant_ctas(uint64_t count) {
  return (uint32_t)std::min<uint64_t>(std::max<uint64_t>(cdiv(count, 16ull * kQThreads), 1),
                                      std::min<uint32_t>(kQMaxCtas, 4 * num_sms()));
}

template <typename F>
static int quantize_dynamic(const void *in, int dtype, uint64_t count, void *out, float *scale,
                            void *workspace, cudaStream_t stream) {
  const bool vec = aligned(16, in, out);
  const uint32_t ctas = quant_ctas(count);
  uint32_t *ws = reinterpret_cast<uint32_t *>(workspace);
  uint8_t *q = reinterpret_cast<uint8_t *>(out);
  MEB_DISPATCH_DTYPE(dtype, {
    const T *x = reinterpret_cast<const T *>(in);
    if (vec) {
      k_amax<T, true, F><<<ctas, kQThreads, 0, stream>>>(x, count, scale, ws);
      MEB_LAUNCH_OK();
      k_quant<T, true, F><<<ctas, kQThreads, 0, stream>>>(x, count, scale, q);
    } else {
      k_amax<T, false, F><<<ctas, kQThreads, 0, stream>>>(x, count, scale, ws);
      MEB_LAUNCH_OK();
      k_quant<T, false, F><<<ctas, kQThreads, 0, stream>>>(x, count, scale, q);
    }
    MEB_LAUNCH_OK();
  });
  return MEB200_OK;
}

int quantize_e4m3(const void *in, int dtype, uint64_t count, void *out, float *scale,
                  void *workspace, cudaStream_t stream) {
  return quantize_dynamic<E4M3>(in, dtype, count, out, scale, workspace, stream);
}

int quantize_e5m2(const void *in, int dtype, uint64_t count, void *out, float *scale,
                  void *workspace, cudaStream_t stream) {
  return quantize_dynamic<E5M2>(in, dtype, count, out, scale, workspace, stream);
}

// ---- static scales --------------------------------------------------------------------------------
// Calibration: amax = max(amax, max |x| over the finite values), k_amax's CTA max and atomic max on
// the fp32 bits, with nothing to count or reset: any number of calls accumulate into one float.
template <typename T, bool VEC>
__global__ void __launch_bounds__(kQThreads) k_amax_acc(const T *__restrict__ x, uint64_t count,
                                                       uint32_t *amax) {
  float m;
  if (cta_amax<T, VEC>(x, count, m)) atomicMax(amax, __float_as_uint(m));
}

__global__ void k_scales(const float *__restrict__ amax, float *__restrict__ scale) {
  float s, inv;
  fp8_scales<E4M3>(*amax, s, inv);
  scale[0] = s;
  scale[1] = inv;
}

int amax_accumulate(const void *in, int dtype, uint64_t count, float *amax, cudaStream_t stream) {
  if (count == 0) return MEB200_OK;
  const uint32_t ctas = quant_ctas(count);
  uint32_t *a = reinterpret_cast<uint32_t *>(amax);
  MEB_DISPATCH_DTYPE(dtype, {
    const T *x = reinterpret_cast<const T *>(in);
    if (aligned(16, in)) k_amax_acc<T, true><<<ctas, kQThreads, 0, stream>>>(x, count, a);
    else k_amax_acc<T, false><<<ctas, kQThreads, 0, stream>>>(x, count, a);
    MEB_LAUNCH_OK();
  });
  return MEB200_OK;
}

int e4m3_scales_from_amax(const float *amax, float *scale, cudaStream_t stream) {
  k_scales<<<1, 1, 0, stream>>>(amax, scale);
  MEB_LAUNCH_OK();
  return MEB200_OK;
}

int quantize_e4m3_static(const void *in, int dtype, uint64_t count, void *out, const float *scale,
                         cudaStream_t stream) {
  if (count == 0) return MEB200_OK;
  const uint32_t ctas = quant_ctas(count);
  uint8_t *q = reinterpret_cast<uint8_t *>(out);
  MEB_DISPATCH_DTYPE(dtype, {
    const T *x = reinterpret_cast<const T *>(in);
    if (aligned(16, in, out)) k_quant<T, true, E4M3><<<ctas, kQThreads, 0, stream>>>(x, count, scale, q);
    else k_quant<T, false, E4M3><<<ctas, kQThreads, 0, stream>>>(x, count, scale, q);
    MEB_LAUNCH_OK();
  });
  return MEB200_OK;
}

// ---- delayed scaling --------------------------------------------------------------------------
template <typename F>
static int quantize_record_as(const void *in, int dtype, uint64_t count, void *out,
                              const float *scale, float *slot, cudaStream_t stream) {
  const uint32_t ctas = quant_ctas(count);
  uint8_t *q = reinterpret_cast<uint8_t *>(out);
  uint32_t *a = reinterpret_cast<uint32_t *>(slot);
  MEB_DISPATCH_DTYPE(dtype, {
    const T *x = reinterpret_cast<const T *>(in);
    if (aligned(16, in, out))
      k_quant_record<T, true, F><<<ctas, kQThreads, 0, stream>>>(x, count, scale, q, a);
    else
      k_quant_record<T, false, F><<<ctas, kQThreads, 0, stream>>>(x, count, scale, q, a);
    MEB_LAUNCH_OK();
  });
  return MEB200_OK;
}

int quantize_record(const void *in, int dtype, uint64_t count, int format, void *out,
                    const float *scale, float *slot, cudaStream_t stream) {
  if (count == 0) return MEB200_OK;
  return format == MEB200_FP8_E5M2
             ? quantize_record_as<E5M2>(in, dtype, count, out, scale, slot, stream)
             : quantize_record_as<E4M3>(in, dtype, count, out, scale, slot, stream);
}

// One thread per entry: history [L, H] (newest first) takes the step's slot in front and drops its
// oldest value, amax = the max of the new history, (scale, inv) = fp8_scales(min(amax * 2^margin,
// FLT_MAX)) in the entry's format (e4m3 below n_e4m3, e5m2 from there), next_cur = 0.
__global__ void __launch_bounds__(128) k_fp8_roll(const float *__restrict__ cur,
                                                  float *__restrict__ hist, uint32_t n_e4m3,
                                                  uint32_t L, uint32_t H, int margin,
                                                  float *__restrict__ next_cur,
                                                  float *__restrict__ scales) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= L) return;
  float *h = hist + (size_t)i * H;
  float v = cur[i], amax = 0.f;
  for (uint32_t k = 0; k < H; ++k) {
    const float older = h[k];
    h[k] = v;
    amax = fmaxf(amax, v);
    v = older;
  }
  const float a = fminf(ldexpf(amax, margin), FLT_MAX);
  float s, inv;
  if (i < n_e4m3) fp8_scales<E4M3>(a, s, inv);
  else fp8_scales<E5M2>(a, s, inv);
  scales[2 * (size_t)i] = s;
  scales[2 * (size_t)i + 1] = inv;
  next_cur[i] = 0.f;
}

int fp8_roll(const float *cur, float *hist, uint32_t n_e4m3, uint32_t n_e5m2, uint32_t H,
             int margin, float *next_cur, float *scales, cudaStream_t stream) {
  const uint32_t L = n_e4m3 + n_e5m2;
  if (L == 0) return MEB200_OK;
  k_fp8_roll<<<cdiv(L, 128u), 128, 0, stream>>>(cur, hist, n_e4m3, L, H, margin, next_cur, scales);
  MEB_LAUNCH_OK();
  return MEB200_OK;
}

// Weights: one CTA per 32 output channels.  Pass 1: the amax of each column over all K * c_in rows
// (8 row phases per column, combined with fmaxf: order-free).  Pass 2: 32 x 32 tiles transposed
// through shared memory into w_t [K, c_out, c_in], as k_pack_w does.
__global__ void __launch_bounds__(256) k_pack_w_e4m3(const float *__restrict__ W, uint32_t K,
                                                     uint32_t c_in, uint32_t c_out,
                                                     uint8_t *__restrict__ Wt,
                                                     float *__restrict__ w_scale) {
  __shared__ float tile[32][33];
  __shared__ float inv_s[32];
  const uint32_t tx = threadIdx.x & 31, ty = threadIdx.x >> 5, co0 = blockIdx.x * 32;
  const uint32_t co = co0 + tx;
  const uint64_t rows = (uint64_t)K * c_in;
  float m = 0.f;
  if (co < c_out)
    for (uint64_t r = ty; r < rows; r += 8) m = fmaxf(m, finite_abs(W[r * c_out + co]));
  tile[ty][tx] = m;
  __syncthreads();
  if (ty == 0) {
    for (uint32_t i = 1; i < 8; ++i) m = fmaxf(m, tile[i][tx]);
    float s, inv;
    fp8_scales<E4M3>(m, s, inv);
    inv_s[tx] = inv;
    if (co < c_out) w_scale[co] = s;
  }
  __syncthreads();
  for (uint32_t k = 0; k < K; ++k)
    for (uint32_t ci0 = 0; ci0 < c_in; ci0 += 32) {
      const size_t base = (size_t)k * c_in * c_out;
      for (uint32_t i = ty; i < 32; i += 8)
        if (ci0 + i < c_in && co < c_out) tile[i][tx] = W[base + (size_t)(ci0 + i) * c_out + co];
      __syncthreads();
      for (uint32_t i = ty; i < 32; i += 8)
        if (co0 + i < c_out && ci0 + tx < c_in)
          Wt[base + (size_t)(co0 + i) * c_in + ci0 + tx] = fp8_byte<E4M3>(tile[tx][i], inv_s[i]);
      __syncthreads();
    }
}

int conv_pack_weights_e4m3(const float *W, uint32_t K, uint32_t c_in, uint32_t c_out, void *w_t,
                           float *w_scale, cudaStream_t stream) {
  k_pack_w_e4m3<<<cdiv(c_out, 32), 256, 0, stream>>>(W, K, c_in, c_out,
                                                     reinterpret_cast<uint8_t *>(w_t), w_scale);
  MEB_LAUNCH_OK();
  return MEB200_OK;
}

// The dgrad's weights: one CTA per input channel ci.  The amax of row ci over all (k, co) (thread
// phases combined with fmaxf: order-free), then the row's bytes in place, [K, c_in, c_out].
__global__ void __launch_bounds__(256) k_pack_w_e4m3_dgrad(const float *__restrict__ W, uint32_t K,
                                                           uint32_t c_in, uint32_t c_out,
                                                           uint8_t *__restrict__ Wc,
                                                           float *__restrict__ w_scale) {
  __shared__ float wm[8];
  __shared__ float inv_s;
  const uint32_t ci = blockIdx.x;
  float m = 0.f;
  for (uint32_t k = 0; k < K; ++k)
    for (uint32_t co = threadIdx.x; co < c_out; co += 256)
      m = fmaxf(m, finite_abs(W[((size_t)k * c_in + ci) * c_out + co]));
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, d));
  if ((threadIdx.x & 31) == 0) wm[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (uint32_t w = 1; w < 8; ++w) m = fmaxf(m, wm[w]);
    float s, inv;
    fp8_scales<E4M3>(m, s, inv);
    w_scale[ci] = s;
    inv_s = inv;
  }
  __syncthreads();
  const float inv = inv_s;
  for (uint32_t k = 0; k < K; ++k)
    for (uint32_t co = threadIdx.x; co < c_out; co += 256) {
      const size_t e = ((size_t)k * c_in + ci) * c_out + co;
      Wc[e] = fp8_byte<E4M3>(W[e], inv);
    }
}

int conv_pack_weights_e4m3_dgrad(const float *W, uint32_t K, uint32_t c_in, uint32_t c_out,
                                 void *w_c, float *w_scale, cudaStream_t stream) {
  k_pack_w_e4m3_dgrad<<<c_in, 256, 0, stream>>>(W, K, c_in, c_out, reinterpret_cast<uint8_t *>(w_c),
                                                w_scale);
  MEB_LAUNCH_OK();
  return MEB200_OK;
}

}  // namespace meb200
