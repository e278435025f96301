// SIMT gather-GEMM sparse convolution (output-stationary, no atomics on features).
//
// Reference semantics: ConvolutionForwardKernelCPU / ConvolutionBackwardKernelCPU
// (src/convolution_kernel.hpp:33-144): out[o] = sum_k in[i_k(o)] W_k ;
// dIn[i] = sum_k dOut[o_k(i)] W_k^T ; dW_k = sum_o in[i_k(o)]^T dOut[o].
// Unlike the reference GPU kernels (src/convolution_kernel.cu:114-287: one launch per
// offset, per-element atomicAdd scatter) one launch covers all offsets of a layer and each
// output row is produced by exactly one CTA from the k-major neighbour table.
#include "conv_simt.cuh"

#include <algorithm>

namespace meb200 {

constexpr int TM = 64, TN = 64, TK = 16;

// out[r, n] = sum_k sum_c A[nbr[k][r], c] * Wk(c, n)
//   TRANS_W = false: Wk(c, n) = W[k][c][n]   (W is [K, c_a, c_n])        -> forward
//   TRANS_W = true : Wk(c, n) = W[k][n][c]   (W is [K, c_n, c_a])        -> dgrad
template <typename TIn, typename TOut, bool TRANS_W>
__global__ void __launch_bounds__(256)
k_conv_gather_gemm(const TIn *__restrict__ A, uint32_t c_a, const TIn *__restrict__ W, uint32_t K,
                   uint32_t c_n, const int32_t *__restrict__ nbr, uint32_t n_rows,
                   TOut *__restrict__ out) {
  __shared__ float As[TK][TM + 4];
  __shared__ float Bs[TK][TN + 4];
  __shared__ int32_t s_idx[TM];

  const uint32_t row0 = blockIdx.x * TM, n0 = blockIdx.y * TN;
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (uint32_t k = 0; k < K; ++k) {
    __syncthreads();  // previous iteration's readers of s_idx / tiles are done
    int has = 0;
    if (tid < TM) {
      uint32_t r = row0 + tid;
      int32_t v = (r < n_rows) ? __ldg(nbr + (size_t)k * n_rows + r) : -1;
      s_idx[tid] = v;
      has = v >= 0;
    }
    if (!__syncthreads_or(has)) continue;
    const TIn *Wk = W + (size_t)k * c_a * c_n;
    for (uint32_t c0 = 0; c0 < c_a; c0 += TK) {
      // A tile: TM x TK gathered rows (consecutive threads -> consecutive channels)
#pragma unroll
      for (int j = 0; j < (TM * TK) / 256; ++j) {
        int e = tid + j * 256, r = e / TK, c = e % TK;
        int32_t src = s_idx[r];
        float v = 0.f;
        if (src >= 0 && c0 + c < c_a) v = to_f32<TIn>(A[(size_t)src * c_a + c0 + c]);
        As[c][r] = v;
      }
      // B tile: TK x TN of Wk
#pragma unroll
      for (int j = 0; j < (TK * TN) / 256; ++j) {
        int e = tid + j * 256;
        int kk, nn;
        if (TRANS_W) { nn = e / TK; kk = e % TK; } else { kk = e / TN; nn = e % TN; }
        float v = 0.f;
        if (c0 + kk < c_a && n0 + nn < c_n) {
          size_t off = TRANS_W ? (size_t)(n0 + nn) * c_a + (c0 + kk)
                               : (size_t)(c0 + kk) * c_n + (n0 + nn);
          v = to_f32<TIn>(Wk[off]);
        }
        Bs[kk][nn] = v;
      }
      __syncthreads();
#pragma unroll
      for (int kk = 0; kk < TK; ++kk) {
        float a[4], b[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) a[i] = As[kk][ty * 4 + i];
#pragma unroll
        for (int j = 0; j < 4; ++j) b[j] = Bs[kk][tx * 4 + j];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
      }
      __syncthreads();
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    uint32_t r = row0 + ty * 4 + i;
    if (r >= n_rows) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      uint32_t n = n0 + tx * 4 + j;
      if (n < c_n) out[(size_t)r * c_n + n] = from_f32<TOut>(acc[i][j]);
    }
  }
}

// part[split][k][ci][co] = sum over rows o in this CTA's split of in[nbr[k][o]][ci] * dOut[o][co]
// Every element of the split's slot is stored once (zeros included); with one split the slot is
// dW itself, otherwise launch_split_sum adds the slots in split order.
template <typename T>
__global__ void __launch_bounds__(256)
k_conv_wgrad(const T *__restrict__ in, const T *__restrict__ grad_out, uint32_t c_in,
             uint32_t c_out, const int32_t *__restrict__ out_nbr, uint32_t n_out,
             uint32_t rows_per_split, uint32_t tiles_n, float *__restrict__ part) {
  __shared__ float As[TK][TM + 4];  // [row in chunk][ci]
  __shared__ float Bs[TK][TN + 4];  // [row in chunk][co]
  __shared__ int32_t s_idx[TK];

  const uint32_t k = blockIdx.x;
  const uint32_t ci0 = (blockIdx.z / tiles_n) * TM, co0 = (blockIdx.z % tiles_n) * TN;
  const uint32_t r_begin = blockIdx.y * rows_per_split;
  const uint32_t r_end = min(r_begin + rows_per_split, n_out);
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (uint32_t r0 = r_begin; r0 < r_end; r0 += TK) {
    __syncthreads();
    int has = 0;
    if (tid < TK) {
      uint32_t r = r0 + tid;
      int32_t v = (r < r_end) ? __ldg(out_nbr + (size_t)k * n_out + r) : -1;
      s_idx[tid] = v;
      has = v >= 0;
    }
    if (!__syncthreads_or(has)) continue;
#pragma unroll
    for (int j = 0; j < (TK * TM) / 256; ++j) {
      int e = tid + j * 256, rr = e / TM, c = e % TM;
      int32_t src = s_idx[rr];
      float a = 0.f, b = 0.f;
      if (src >= 0) {
        if (ci0 + c < c_in) a = to_f32<T>(in[(size_t)src * c_in + ci0 + c]);
        if (co0 + c < c_out) b = to_f32<T>(grad_out[(size_t)(r0 + rr) * c_out + co0 + c]);
      }
      As[rr][c] = a;
      Bs[rr][c] = b;
    }
    __syncthreads();
#pragma unroll
    for (int rr = 0; rr < TK; ++rr) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = As[rr][ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) b[j] = Bs[rr][tx * 4 + j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
  }
  float *dWk = part + ((size_t)blockIdx.y * gridDim.x + k) * c_in * c_out;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    uint32_t ci = ci0 + ty * 4 + i;
    if (ci >= c_in) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      uint32_t co = co0 + tx * 4 + j;
      if (co < c_out) dWk[(size_t)ci * c_out + co] = acc[i][j];
    }
  }
}

// ---- tiny input-channel count (the network stem: c_in <= 4, e.g. RGB -> 32, K = 125) -------
// Too few channels for a GEMM tile; both passes are bound by the latency of the neighbour-table
// scan and of the row gathers behind it, so both keep many independent loads in flight.
//
// Forward: persistent CTAs (W staged to shared memory once per CTA as fp32 [K][c_in][CO]),
// one thread per output row with all CO outputs in registers.  Offsets are walked in batches
// of SK: the SK table entries of the NEXT batch and the SK gathered rows of THIS batch are
// issued before the FMAs, so a thread has up to 2*SK independent loads outstanding instead of
// a dependent (index -> row) chain per offset.
constexpr int SK = 8;

template <typename TOut, int CO>
__device__ __forceinline__ void store_row(TOut *__restrict__ dst, const float (&acc)[CO],
                                          uint32_t c_out) {
  if constexpr (sizeof(TOut) == 2) {
    if (c_out == (uint32_t)CO) {  // rows are CO*2 bytes: 16 B aligned for CO in {32, 64}
#pragma unroll
      for (int v = 0; v < CO / 8; ++v) {
        TOut t[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) t[j] = from_f32<TOut>(acc[8 * v + j]);
        reinterpret_cast<uint4 *>(dst)[v] = *reinterpret_cast<const uint4 *>(t);
      }
      return;
    }
  }
#pragma unroll
  for (int i = 0; i < CO; ++i)
    if ((uint32_t)i < c_out) dst[i] = from_f32<TOut>(acc[i]);
}

template <typename T, typename TOut, int CO>
__global__ void __launch_bounds__(128)
k_conv_small_cin_fwd(const T *__restrict__ in, uint32_t c_in, const T *__restrict__ W, uint32_t K,
                     uint32_t c_out, const int32_t *__restrict__ nbr, uint32_t n_out,
                     TOut *__restrict__ out) {
  extern __shared__ float Ws[];  // [K][c_in][CO], zero padded past c_out
  for (uint32_t e = threadIdx.x; e < K * c_in * CO; e += blockDim.x) {
    uint32_t co = e % CO, kc = e / CO;
    Ws[e] = co < c_out ? to_f32<T>(W[(size_t)kc * c_out + co]) : 0.f;
  }
  __syncthreads();
  const uint32_t n_tiles = (n_out + 127) / 128;
  for (uint32_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const uint32_t o = tile * 128 + threadIdx.x;
    const bool live = o < n_out;
    const int32_t *col = nbr + o;
    float acc[CO];
#pragma unroll
    for (int i = 0; i < CO; ++i) acc[i] = 0.f;
    int32_t idx[SK];
#pragma unroll
    for (int j = 0; j < SK; ++j)
      idx[j] = (live && (uint32_t)j < K) ? __ldg(col + (size_t)j * n_out) : -1;
    for (uint32_t k0 = 0; k0 < K; k0 += SK) {
      int32_t nxt[SK];
#pragma unroll
      for (int j = 0; j < SK; ++j) {
        const uint32_t kk = k0 + SK + j;
        nxt[j] = (live && kk < K) ? __ldg(col + (size_t)kk * n_out) : -1;
      }
      float x[SK][4];
#pragma unroll
      for (int j = 0; j < SK; ++j)
#pragma unroll
        for (int c = 0; c < 4; ++c)
          x[j][c] = (idx[j] >= 0 && (uint32_t)c < c_in)
                        ? to_f32<T>(in[(size_t)idx[j] * c_in + c]) : 0.f;
#pragma unroll
      for (int j = 0; j < SK; ++j) {
        if (idx[j] < 0) continue;
        const float *wk = Ws + (size_t)(k0 + j) * c_in * CO;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          if ((uint32_t)c >= c_in) break;
          const float4 *w4 = reinterpret_cast<const float4 *>(wk + c * CO);
#pragma unroll
          for (int v = 0; v < CO / 4; ++v) {
            const float4 w = w4[v];
            acc[4 * v + 0] = fmaf(x[j][c], w.x, acc[4 * v + 0]);
            acc[4 * v + 1] = fmaf(x[j][c], w.y, acc[4 * v + 1]);
            acc[4 * v + 2] = fmaf(x[j][c], w.z, acc[4 * v + 2]);
            acc[4 * v + 3] = fmaf(x[j][c], w.w, acc[4 * v + 3]);
          }
        }
      }
#pragma unroll
      for (int j = 0; j < SK; ++j) idx[j] = nxt[j];
    }
    if (live) store_row<TOut, CO>(out + (size_t)o * c_out, acc, c_out);
  }
}

// dW[k][c][co] = sum_o in[nbr[k][o]][c] * dOut[o][co] for c_in <= 4, c_out <= 64.
// Warp <-> (offset k, row slice, 32-channel slab).  The table column is scanned 256 rows at a
// time (8 independent coalesced loads per lane); hits are compacted with ballot/popc into a
// per-warp shared-memory list, and the list is consumed 32 hits at a time with lane <-> hit:
// every lane fetches its own dOut row slab (vector loads) and input row and accumulates a private
// [CIN][32] tile in registers, so 32 row fetches are in flight per warp instead of one.  The
// 32 private tiles are folded with butterfly shuffles once per warp and stored to the row slice's
// slot part[slice][k][c][co] (dW itself with one slice); launch_split_sum adds the slots in order.
constexpr int WG_SCAN = 256;             // table entries scanned per round (8 per lane)
constexpr int WG_LIST = WG_SCAN + 32;    // + carried remainder (< 32)

template <typename T>
__device__ __forceinline__ void load_slab32(const T *__restrict__ p, uint32_t nco, bool vec,
                                            float (&g)[32]) {
  if (vec) {  // nco == 32 and p is 16 B aligned
    constexpr int PER = 16 / sizeof(T);
#pragma unroll
    for (int v = 0; v < 32 / PER; ++v) {
      const uint4 q = __ldg(reinterpret_cast<const uint4 *>(p) + v);
      T t[PER];
      *reinterpret_cast<uint4 *>(t) = q;
#pragma unroll
      for (int j = 0; j < PER; ++j) g[v * PER + j] = to_f32<T>(t[j]);
    }
  } else {
#pragma unroll
    for (int j = 0; j < 32; ++j) g[j] = (uint32_t)j < nco ? to_f32<T>(p[j]) : 0.f;
  }
}

template <typename T, int CIN>
__global__ void __launch_bounds__(256, 1)
k_conv_small_cin_wgrad(const T *__restrict__ in, const T *__restrict__ gout, uint32_t c_out,
                       uint32_t K, const int32_t *__restrict__ nbr, uint32_t n_out,
                       uint32_t rows_per_block, float *__restrict__ part) {
  __shared__ uint2 s_hits[8][WG_LIST];  // (output row, input row) per warp
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t k = blockIdx.y * 8 + warp;
  if (k >= K) return;  // warps never synchronise with each other below
  const uint32_t co0 = blockIdx.z * 32;
  const uint32_t nco = min(32u, c_out - co0);
  const bool vec = nco == 32 && ((size_t)c_out * sizeof(T)) % 16 == 0 &&
                   ((size_t)co0 * sizeof(T)) % 16 == 0 &&
                   (reinterpret_cast<uintptr_t>(gout) & 15) == 0;
  const uint32_t r0 = blockIdx.x * rows_per_block;
  const uint32_t r1 = min(r0 + rows_per_block, n_out);
  const int32_t *nbr_k = nbr + (size_t)k * n_out;
  uint2 *list = s_hits[warp];
  const uint32_t lt = (1u << lane) - 1u;

  float acc[CIN][32];
#pragma unroll
  for (int c = 0; c < CIN; ++c)
#pragma unroll
    for (int j = 0; j < 32; ++j) acc[c][j] = 0.f;

  auto consume = [&](const uint2 h) {
    float g[32];
    load_slab32<T>(gout + (size_t)h.x * c_out + co0, nco, vec, g);
    float x[CIN];
#pragma unroll
    for (int c = 0; c < CIN; ++c) x[c] = to_f32<T>(in[(size_t)h.y * CIN + c]);
#pragma unroll
    for (int c = 0; c < CIN; ++c)
#pragma unroll
      for (int j = 0; j < 32; ++j) acc[c][j] = fmaf(x[c], g[j], acc[c][j]);
  };

  uint32_t cnt = 0;
  for (uint32_t o0 = r0; o0 < r1; o0 += WG_SCAN) {
    int32_t idx[WG_SCAN / 32];
#pragma unroll
    for (int j = 0; j < WG_SCAN / 32; ++j) {
      const uint32_t o = o0 + j * 32 + lane;
      idx[j] = o < r1 ? __ldg(nbr_k + o) : -1;
    }
#pragma unroll
    for (int j = 0; j < WG_SCAN / 32; ++j) {
      const unsigned m = __ballot_sync(0xffffffffu, idx[j] >= 0);
      if (idx[j] >= 0) list[cnt + __popc(m & lt)] = make_uint2(o0 + j * 32 + lane, (uint32_t)idx[j]);
      cnt += __popc(m);
    }
    __syncwarp();
    uint32_t done = 0;
    while (cnt - done >= 32) {
      consume(list[done + lane]);
      done += 32;
    }
    if (done) {  // move the remainder (< 32 hits) to the front of the list
      const uint32_t rem = cnt - done;
      uint2 t = make_uint2(0, 0);
      if (lane < rem) t = list[done + lane];
      __syncwarp();
      if (lane < rem) list[lane] = t;
      cnt = rem;
    }
    __syncwarp();
  }
  if (lane < cnt) consume(list[lane]);

#pragma unroll
  for (int c = 0; c < CIN; ++c) {
    float *dst = part + (((size_t)blockIdx.x * K + k) * CIN + c) * c_out + co0;
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      float v = acc[c][j];
#pragma unroll
      for (int s = 16; s > 0; s >>= 1) v += __shfl_xor_sync(0xffffffffu, v, s);
      if (lane == (uint32_t)j && (uint32_t)j < nco) dst[j] = v;
    }
  }
}

bool conv_small_cin_supported(uint32_t c_in, uint32_t c_out) {
  return c_in >= 1 && c_in <= 4 && c_out <= 64;
}

template <typename T, typename TOut>
static int launch_small_fwd(const void *in, uint32_t c_in, const void *W, uint32_t K,
                            uint32_t c_out, const int32_t *nbr, uint32_t n_out, void *out,
                            cudaStream_t stream) {
  const int CO = c_out <= 32 ? 32 : 64;
  size_t smem = (size_t)K * c_in * CO * sizeof(float);
  if (smem > 200 * 1024) return MEB200_ERR_UNSUPPORTED;
  // persistent CTAs: as many as fit beside each other (shared memory bound), W staged once each
  unsigned per_sm = (unsigned)std::max<size_t>(1, std::min<size_t>(8, (220 * 1024) / (smem + 1024)));
  unsigned grid = std::min<unsigned>(cdiv(n_out, 128), per_sm * num_sms());
  if (CO == 32) {
    auto kern = k_conv_small_cin_fwd<T, TOut, 32>;
    MEB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    kern<<<grid, 128, smem, stream>>>((const T *)in, c_in, (const T *)W, K, c_out, nbr, n_out, (TOut *)out);
  } else {
    auto kern = k_conv_small_cin_fwd<T, TOut, 64>;
    MEB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    kern<<<grid, 128, smem, stream>>>((const T *)in, c_in, (const T *)W, K, c_out, nbr, n_out, (TOut *)out);
  }
  MEB_LAUNCH_OK();
  return MEB200_OK;
}

int conv_small_cin_forward(const void *in, int in_dtype, uint32_t c_in, const void *W, uint32_t K,
                           uint32_t c_out, const int32_t *nbr, uint32_t n_out, void *out,
                           int out_dtype, cudaStream_t stream) {
  if (n_out == 0) return MEB200_OK;
  MEB_DISPATCH_DTYPE_OUT(in_dtype, out_dtype,
                         return launch_small_fwd<T, TO>(in, c_in, W, K, c_out, nbr, n_out, out, stream));
}

// Row slices k_conv_small_cin_wgrad plans: one 8-warp CTA per SM (register tiles), aiming at
// ~4 CTAs per SM over the whole grid.
static uint32_t small_wgrad_slices(uint32_t c_out, uint32_t K) {
  const uint32_t kgroups = cdiv(K, 8), slabs = cdiv(c_out, 32);
  return std::max<uint32_t>(1, cdiv(4ull * num_sms(), (uint64_t)kgroups * slabs));
}

// Rows per slice for `slices` slices: whole scan rounds, >= 4 each.
static uint32_t small_wgrad_rows(uint32_t n_out, uint32_t slices) {
  const uint32_t rows_per_block = cdiv(cdiv(n_out, slices), WG_SCAN) * WG_SCAN;
  return std::max<uint32_t>(rows_per_block, 4 * WG_SCAN);
}

template <typename T>
static int launch_small_wgrad(const void *in, const void *gout, uint32_t c_in, uint32_t K,
                              uint32_t c_out, const int32_t *nbr, uint32_t n_out, float *dW,
                              void *workspace, uint64_t workspace_bytes, cudaStream_t stream) {
  const uint32_t rows_per_block = small_wgrad_rows(
      n_out, workspace_splits(small_wgrad_slices(c_out, K), workspace, workspace_bytes,
                              (uint64_t)K * c_in * c_out * sizeof(float)));
  dim3 grid(cdiv(n_out, rows_per_block), cdiv(K, 8), cdiv(c_out, 32));
  float *part = grid.x > 1 ? reinterpret_cast<float *>(workspace) : dW;
  const T *x = (const T *)in, *g = (const T *)gout;
  switch (c_in) {
    case 1: k_conv_small_cin_wgrad<T, 1><<<grid, 256, 0, stream>>>(x, g, c_out, K, nbr, n_out, rows_per_block, part); break;
    case 2: k_conv_small_cin_wgrad<T, 2><<<grid, 256, 0, stream>>>(x, g, c_out, K, nbr, n_out, rows_per_block, part); break;
    case 3: k_conv_small_cin_wgrad<T, 3><<<grid, 256, 0, stream>>>(x, g, c_out, K, nbr, n_out, rows_per_block, part); break;
    case 4: k_conv_small_cin_wgrad<T, 4><<<grid, 256, 0, stream>>>(x, g, c_out, K, nbr, n_out, rows_per_block, part); break;
    default: return MEB200_ERR_UNSUPPORTED;
  }
  MEB_LAUNCH_OK();
  if (grid.x == 1) return MEB200_OK;
  return launch_split_sum(part, dW, (size_t)K * c_in * c_out, grid.x, stream);
}

int conv_small_cin_wgrad(const void *in, const void *grad_out, int dtype, uint32_t c_in, uint32_t K,
                         uint32_t c_out, const int32_t *out_nbr, uint32_t n_out, float *grad_weight,
                         void *workspace, uint64_t workspace_bytes, cudaStream_t stream) {
  if (n_out == 0 || K == 0) {
    MEB_CUDA(cudaMemsetAsync(grad_weight, 0, (size_t)K * c_in * c_out * sizeof(float), stream));
    return MEB200_OK;
  }
  MEB_DISPATCH_DTYPE(dtype, return launch_small_wgrad<T>(in, grad_out, c_in, K, c_out, out_nbr,
                                                         n_out, grad_weight, workspace,
                                                         workspace_bytes, stream));
}

template <typename TIn, typename TOut>
static int launch_gg(const void *A, uint32_t c_a, const void *W, uint32_t K, uint32_t c_n,
                     bool trans_w, const int32_t *nbr, uint32_t n_rows, void *out,
                     cudaStream_t stream) {
  dim3 grid(cdiv(n_rows, TM), cdiv(c_n, TN));
  if (trans_w)
    k_conv_gather_gemm<TIn, TOut, true><<<grid, 256, 0, stream>>>(
        (const TIn *)A, c_a, (const TIn *)W, K, c_n, nbr, n_rows, (TOut *)out);
  else
    k_conv_gather_gemm<TIn, TOut, false><<<grid, 256, 0, stream>>>(
        (const TIn *)A, c_a, (const TIn *)W, K, c_n, nbr, n_rows, (TOut *)out);
  MEB_LAUNCH_OK();
  return MEB200_OK;
}

int conv_forward_simt(const void *in, int in_dtype, uint32_t n_in, uint32_t c_in,
                      const void *weight, uint32_t K, uint32_t c_out, bool trans_w,
                      const int32_t *nbr, uint32_t n_out, void *out, int out_dtype,
                      cudaStream_t stream) {
  (void)n_in;
  if (n_out == 0) return MEB200_OK;
  MEB_DISPATCH_DTYPE_OUT(in_dtype, out_dtype,
                         return launch_gg<T, TO>(in, c_in, weight, K, c_out, trans_w, nbr, n_out,
                                                 out, stream));
}

// Row splits k_conv_wgrad plans: enough CTAs for ~4 waves, each split at least 8 * TK rows.
static uint32_t simt_wgrad_splits(uint32_t c_in, uint32_t c_out, uint32_t K, uint32_t n_out) {
  const uint64_t tiles = (uint64_t)cdiv(c_in, TM) * cdiv(c_out, TN);
  const uint64_t splits = std::max<uint64_t>(1, cdiv(4ull * num_sms(), (uint64_t)K * tiles));
  return (uint32_t)std::min<uint64_t>({splits, cdiv(n_out, 8 * TK), 65535});
}

// Rows per split for `splits` splits: a multiple of TK.
static uint32_t simt_wgrad_rows(uint32_t n_out, uint32_t splits) {
  return cdiv(cdiv(n_out, splits), TK) * TK;
}

uint64_t conv_wgrad_simt_workspace_bytes(uint32_t c_in, uint32_t c_out, uint32_t K,
                                         uint32_t n_out) {
  if (n_out == 0 || K == 0 || c_in == 0 || c_out == 0) return 0;
  const uint32_t rows = conv_small_cin_supported(c_in, c_out)
                            ? small_wgrad_rows(n_out, small_wgrad_slices(c_out, K))
                            : simt_wgrad_rows(n_out, simt_wgrad_splits(c_in, c_out, K, n_out));
  const uint32_t splits = cdiv(n_out, rows);
  return splits > 1 ? (uint64_t)splits * K * c_in * c_out * sizeof(float) : 0;
}

int conv_wgrad_simt(const void *in, const void *grad_out, int dtype, uint32_t c_in, uint32_t K,
                    uint32_t c_out, const int32_t *out_nbr, uint32_t n_out, float *grad_weight,
                    void *workspace, uint64_t workspace_bytes, cudaStream_t stream) {
  if (n_out == 0 || K == 0) {
    MEB_CUDA(cudaMemsetAsync(grad_weight, 0, (size_t)K * c_in * c_out * sizeof(float), stream));
    return MEB200_OK;
  }
  const uint32_t tiles_n = cdiv(c_out, TN), tiles = cdiv(c_in, TM) * tiles_n;
  MEB_CHECK_ARG(tiles <= 65535, "too many channel tiles");
  const uint32_t rows_per_split = simt_wgrad_rows(
      n_out, workspace_splits(simt_wgrad_splits(c_in, c_out, K, n_out), workspace,
                              workspace_bytes, (uint64_t)K * c_in * c_out * sizeof(float)));
  const uint32_t splits = cdiv(n_out, rows_per_split);
  float *part = splits > 1 ? reinterpret_cast<float *>(workspace) : grad_weight;
  dim3 grid(K, splits, tiles);
  MEB_DISPATCH_DTYPE(dtype, k_conv_wgrad<T><<<grid, 256, 0, stream>>>(
                                (const T *)in, (const T *)grad_out, c_in, c_out, out_nbr, n_out,
                                rows_per_split, tiles_n, part));
  MEB_LAUNCH_OK();
  if (splits == 1) return MEB200_OK;
  return launch_split_sum(part, grad_weight, (size_t)K * c_in * c_out, splits, stream);
}

}  // namespace meb200
