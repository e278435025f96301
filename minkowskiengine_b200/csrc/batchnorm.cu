// Batch normalisation over the rows of an [N, C] feature matrix (training and inference),
// the first "next" row of SURVEY.md §8(f): the reference applies torch.nn.BatchNorm1d to `.F`
// (MinkowskiNormalization.py:51-99); torch's channels-last kernels run ~8x off the HBM
// roofline on [800k, 96] bf16 and cost 18 % of a MinkUNet34C step, so the four passes are
// provided here as streaming kernels: 16-byte row-segment loads, per-thread fp32 partials over
// a strided set of rows, combined in a fixed order: per CTA in shared memory, then the CTAs' fp64
// partials by the last CTA in block order (no floating-point atomics: results do not depend on
// the order in which threads or CTAs finish).
//
//   stats      : S1[c] = sum_r x[r,c],  S2[c] = sum_r x[r,c]^2                 (fp64 [2C])
//   finalize   : mean, invstd (biased var, eps) + running-stat update (unbiased var)
//   apply      : y = (x - mean) * invstd * w + b                        (optional ReLU)
//   bwd_reduce : G1[c] = sum_r dy,  G2[c] = sum_r dy * (x - mean) * invstd   (fp64 [2C])
//   bwd_apply  : dx = (dy - G1/n - xhat * G2/n) * invstd * w
#include "common.cuh"
#include "peer.cuh"

namespace meb200 {

constexpr int kBnThreads = 256;

template <typename T> struct Vec8;   // eight consecutive channels = one 16-byte (bf16/fp16) load
template <> struct Vec8<__nv_bfloat16> {
  using Raw = uint4;     // the 16 bytes as loaded; unpacked to fp32 only when used
  static __device__ __forceinline__ Raw load_raw(const __nv_bfloat16 *p) { return *reinterpret_cast<const uint4 *>(p); }
  static __device__ __forceinline__ void unpack(const Raw &v, float (&f)[8]) {
    const __nv_bfloat162 *h = reinterpret_cast<const __nv_bfloat162 *>(&v);
#pragma unroll
    for (int i = 0; i < 4; ++i) { float2 t = __bfloat1622float2(h[i]); f[2 * i] = t.x; f[2 * i + 1] = t.y; }
  }
  static __device__ __forceinline__ void load(const __nv_bfloat16 *p, float (&f)[8]) {
    uint4 v = *reinterpret_cast<const uint4 *>(p);
    const __nv_bfloat162 *h = reinterpret_cast<const __nv_bfloat162 *>(&v);
#pragma unroll
    for (int i = 0; i < 4; ++i) { float2 t = __bfloat1622float2(h[i]); f[2 * i] = t.x; f[2 * i + 1] = t.y; }
  }
  static __device__ __forceinline__ void store(__nv_bfloat16 *p, const float (&f)[8]) {
    uint4 v;
    __nv_bfloat162 *h = reinterpret_cast<__nv_bfloat162 *>(&v);
#pragma unroll
    for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
    *reinterpret_cast<uint4 *>(p) = v;
  }
};
template <> struct Vec8<__half> {
  using Raw = uint4;
  static __device__ __forceinline__ Raw load_raw(const __half *p) { return *reinterpret_cast<const uint4 *>(p); }
  static __device__ __forceinline__ void unpack(const Raw &v, float (&f)[8]) {
    const __half2 *h = reinterpret_cast<const __half2 *>(&v);
#pragma unroll
    for (int i = 0; i < 4; ++i) { float2 t = __half22float2(h[i]); f[2 * i] = t.x; f[2 * i + 1] = t.y; }
  }
  static __device__ __forceinline__ void load(const __half *p, float (&f)[8]) {
    uint4 v = *reinterpret_cast<const uint4 *>(p);
    const __half2 *h = reinterpret_cast<const __half2 *>(&v);
#pragma unroll
    for (int i = 0; i < 4; ++i) { float2 t = __half22float2(h[i]); f[2 * i] = t.x; f[2 * i + 1] = t.y; }
  }
  static __device__ __forceinline__ void store(__half *p, const float (&f)[8]) {
    uint4 v;
    __half2 *h = reinterpret_cast<__half2 *>(&v);
#pragma unroll
    for (int i = 0; i < 4; ++i) h[i] = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
    *reinterpret_cast<uint4 *>(p) = v;
  }
};
template <> struct Vec8<float> {
  struct Raw { float4 a, b; };
  static __device__ __forceinline__ Raw load_raw(const float *p) {
    Raw r; r.a = reinterpret_cast<const float4 *>(p)[0]; r.b = reinterpret_cast<const float4 *>(p)[1]; return r;
  }
  static __device__ __forceinline__ void unpack(const Raw &v, float (&f)[8]) {
    f[0] = v.a.x; f[1] = v.a.y; f[2] = v.a.z; f[3] = v.a.w; f[4] = v.b.x; f[5] = v.b.y; f[6] = v.b.z; f[7] = v.b.w;
  }
  static __device__ __forceinline__ void load(const float *p, float (&f)[8]) {
    float4 a = reinterpret_cast<const float4 *>(p)[0], b = reinterpret_cast<const float4 *>(p)[1];
    f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
  }
  static __device__ __forceinline__ void store(float *p, const float (&f)[8]) {
    reinterpret_cast<float4 *>(p)[0] = make_float4(f[0], f[1], f[2], f[3]);
    reinterpret_cast<float4 *>(p)[1] = make_float4(f[4], f[5], f[6], f[7]);
  }
};

// Thread t of a CTA owns channel group (t % G) — 8 channels — and walks rows
// (t / G) + i * rows_per_pass of the CTA's row range.  G = C / 8.
struct BnGeom {
  uint32_t G, rows_per_pass, active;   // active = G * rows_per_pass threads do work
};
__device__ __forceinline__ BnGeom bn_geom(uint32_t C) {
  BnGeom g;
  g.G = C / 8;
  g.rows_per_pass = kBnThreads / g.G;
  g.active = g.G * g.rows_per_pass;
  return g;
}

// What the LAST CTA of a reduction does with the totals (ticket != NULL): the work of the
// separate finalize launch / gradient conversion, and it leaves the CTA slots of `sums` and the
// ticket zero again, so one workspace serves every layer of a stream without a memset per use (a MinkUNet34C step
// spent ~250 of its ~1030 launches on 2 KB memsets and 1-CTA finalize kernels).
struct BnTail {
  uint32_t *ticket;
  double *totals_out;                                   // [2C] copy of the totals, or NULL
  float *mean, *invstd, *running_mean, *running_var;    // MODE 0: finalize (mean NULL = skip)
  double count;
  float eps, momentum;
  float *grad_weight, *grad_bias;                       // MODE 1: fp32 parameter gradients, or NULL
  // synchronised layers (peer_bases != NULL): the last CTA also runs the exchange of csrc/peer.cu
  // — local totals into this rank's symmetric-memory slot, publish / wait, sum over the ranks —
  // so a synchronised pass has the launches of a local one (MODE 0: finalize from the global
  // totals and the global row count; MODE 1: global totals to totals_out, LOCAL ones to the
  // parameter gradients, which DDP averages itself)
  uint8_t *const *peer_bases;
  uint64_t peer_slot_offset;
  uint32_t peer_seq, peer_rank, peer_world;
  double *total_rows_out;                               // MODE 0, synchronised: global row count
  long long *num_batches_tracked;                       // MODE 0: incremented once (may be NULL)
};
constexpr uint32_t kBnMaxC = 2048;
constexpr uint32_t kBnMaxCtas = 512;     // reduction CTAs: each owns a [2C] fp64 slot
constexpr size_t kBnPartialBytes = (size_t)kBnMaxCtas * 2 * kBnMaxC * sizeof(double);
constexpr size_t kBnWorkspaceBytes = kBnPartialBytes + 64;   // CTA partials, then the ticket
// dynamic shared memory of k_bn_reduce: per-thread partials [rows_per_pass][2C] fp32, later the
// totals [2C] fp64 + a [256] fp64 combine scratch
inline size_t bn_reduce_smem(uint32_t C) {
  const size_t rpp = kBnThreads / (C / 8);
  const size_t a = rpp * 2 * C * sizeof(float), b = (2 * (size_t)C + kBnThreads) * sizeof(double);
  return a > b ? a : b;
}

// TWO per-channel sums: MODE 0: (x, x^2); MODE 1: (dy, dy * xhat)
template <typename T, int MODE>
__global__ void __launch_bounds__(kBnThreads)
k_bn_reduce(const T *__restrict__ a, const T *__restrict__ x, const T *__restrict__ ymask,
            const float *__restrict__ mean, const float *__restrict__ invstd, uint32_t n,
            uint32_t C, uint32_t rows_per_cta, double *sums, const BnTail tail) {
  // sums: [gridDim.x][2C] fp64, this CTA's slot written once
  extern __shared__ double s_dyn[];
  float *s_part = reinterpret_cast<float *>(s_dyn);        // [rows_per_pass][2C]
  const uint32_t C2 = 2 * C;
  const BnGeom g = bn_geom(C);
  if (threadIdx.x < g.active) {
    const uint32_t cg = threadIdx.x % g.G, r0 = threadIdx.x / g.G;
    const uint32_t row_begin = blockIdx.x * rows_per_cta;
    const uint32_t row_end = min(row_begin + rows_per_cta, n);
    float s1[8], s2[8], m[8], is[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) { s1[i] = 0.f; s2[i] = 0.f; m[i] = 0.f; is[i] = 1.f; }
    if (MODE == 1) {
#pragma unroll
      for (int i = 0; i < 8; ++i) { m[i] = mean[cg * 8 + i]; is[i] = invstd[cg * 8 + i]; }
    }
    // four rows per iteration: the loads of all four (up to 12 x 16 B) are issued before the
    // first use — one row per iteration left the passes latency bound (1.2 TB/s on [800k, 96])
    constexpr int U = 4;
    const uint32_t step = g.rows_per_pass;
    for (uint32_t r = row_begin + r0; r < row_end; r += U * step) {
      typename Vec8<T>::Raw ra[U], rx[U], ry[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const uint32_t ru = min(r + u * step, row_end - 1);     // clamped: tail rows are skipped below
        ra[u] = Vec8<T>::load_raw(a + (size_t)ru * C + cg * 8);
        if (MODE == 1) {
          rx[u] = Vec8<T>::load_raw(x + (size_t)ru * C + cg * 8);
          if (ymask != nullptr) ry[u] = Vec8<T>::load_raw(ymask + (size_t)ru * C + cg * 8);
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (r + u * step >= row_end) break;
        float va[8];
        Vec8<T>::unpack(ra[u], va);
        if (MODE == 0) {
#pragma unroll
          for (int i = 0; i < 8; ++i) { s1[i] += va[i]; s2[i] = fmaf(va[i], va[i], s2[i]); }
        } else {
          float vx[8];
          Vec8<T>::unpack(rx[u], vx);
          if (ymask != nullptr) {      // ReLU folded into the layer: dy passes where y > 0
            float vy[8];
            Vec8<T>::unpack(ry[u], vy);
#pragma unroll
            for (int i = 0; i < 8; ++i) va[i] = vy[i] > 0.f ? va[i] : 0.f;
          }
#pragma unroll
          for (int i = 0; i < 8; ++i) { s1[i] += va[i]; s2[i] = fmaf(va[i], (vx[i] - m[i]) * is[i], s2[i]); }
        }
      }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      s_part[r0 * C2 + cg * 8 + i] = s1[i];
      s_part[r0 * C2 + C + cg * 8 + i] = s2[i];
    }
  }
  __syncthreads();
  for (uint32_t i = threadIdx.x; i < C2; i += kBnThreads) {
    double v = 0.0;
    for (uint32_t r = 0; r < g.rows_per_pass; ++r) v += (double)s_part[r * C2 + i];
    sums[(size_t)blockIdx.x * C2 + i] = v;
  }
  __shared__ bool s_last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_last = atomicAdd(tail.ticket, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  // totals over the CTAs in block order; J threads per value when 2C < 256, combined in j order.
  // Each slot is read by one thread and cleared as it is read (the workspace is left zero).
  auto take = [](double *p) { const double v = __ldcg(p); *p = 0.0; return v; };
  double *s_tot = s_dyn, *s_scr = s_dyn + C2;
  const uint32_t J = C2 >= kBnThreads ? 1u : kBnThreads / C2;
  if (J == 1) {
    for (uint32_t i = threadIdx.x; i < C2; i += kBnThreads) {
      double v = 0.0;
      for (uint32_t b = 0; b < gridDim.x; ++b) v += take(sums + (size_t)b * C2 + i);
      s_tot[i] = v;
    }
  } else {
    if (threadIdx.x < J * C2) {
      const uint32_t i = threadIdx.x % C2, j = threadIdx.x / C2;
      double v = 0.0;
      for (uint32_t b = j; b < gridDim.x; b += J) v += take(sums + (size_t)b * C2 + i);
      s_scr[j * C2 + i] = v;
    }
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < C2; i += kBnThreads) {
      double v = 0.0;
      for (uint32_t j = 0; j < J; ++j) v += s_scr[j * C2 + i];
      s_tot[i] = v;
    }
  }
  __syncthreads();
  double count = tail.count;
  const bool synced = tail.peer_bases != nullptr;
  if (synced) {
    double *slot = reinterpret_cast<double *>(tail.peer_bases[tail.peer_rank] + tail.peer_slot_offset);
    for (uint32_t c = threadIdx.x; c < C; c += kBnThreads) {
      const double t1 = s_tot[c], t2 = s_tot[C + c];
      slot[c] = t1;
      slot[C + c] = t2;
      if (MODE == 1) {
        if (tail.grad_bias != nullptr) tail.grad_bias[c] = (float)t1;
        if (tail.grad_weight != nullptr) tail.grad_weight[c] = (float)t2;
      }
    }
    if (MODE == 0 && threadIdx.x == 0) slot[2 * C] = tail.count;
    peer_publish_and_wait(tail.peer_bases, tail.peer_seq, tail.peer_rank, tail.peer_world);
    if (MODE == 0) {
      __shared__ double s_count;
      if (threadIdx.x == 0) {
        double t = 0.0;
        for (uint32_t r = 0; r < tail.peer_world; ++r)
          t += ld_relaxed_sys_f64(reinterpret_cast<const double *>(tail.peer_bases[r] + tail.peer_slot_offset) + 2 * C);
        s_count = t;
        if (tail.total_rows_out != nullptr) *tail.total_rows_out = t;
      }
      __syncthreads();
      count = s_count;
    }
  }
  for (uint32_t c = threadIdx.x; c < C; c += kBnThreads) {
    double t1, t2;
    if (synced) {
      t1 = 0.0; t2 = 0.0;
      for (uint32_t r = 0; r < tail.peer_world; ++r) {       // rank order: identical on all ranks
        const double *ps = reinterpret_cast<const double *>(tail.peer_bases[r] + tail.peer_slot_offset);
        t1 += ld_relaxed_sys_f64(ps + c);
        t2 += ld_relaxed_sys_f64(ps + C + c);
      }
    } else {
      t1 = s_tot[c];
      t2 = s_tot[C + c];
    }
    if (tail.totals_out != nullptr) { tail.totals_out[c] = t1; tail.totals_out[C + c] = t2; }
    if (MODE == 0) {
      if (tail.mean != nullptr) {
        const double mu = t1 / count;
        double var = t2 / count - mu * mu;
        if (var < 0) var = 0;
        tail.mean[c] = (float)mu;
        tail.invstd[c] = (float)(1.0 / sqrt(var + (double)tail.eps));
        if (tail.running_mean != nullptr) {
          const double unbiased = count > 1 ? var * count / (count - 1) : var;
          const double mom = tail.momentum;
          tail.running_mean[c] = (float)((1.0 - mom) * tail.running_mean[c] + mom * mu);
          tail.running_var[c] = (float)((1.0 - mom) * tail.running_var[c] + mom * unbiased);
        }
      }
    } else if (!synced) {
      if (tail.grad_bias != nullptr) tail.grad_bias[c] = (float)t1;
      if (tail.grad_weight != nullptr) tail.grad_weight[c] = (float)t2;
    }
  }
  if (threadIdx.x == 0) {
    *tail.ticket = 0u;
    if (MODE == 0 && tail.num_batches_tracked != nullptr) *tail.num_batches_tracked += 1;
  }
}

__global__ void k_bn_finalize(const double *__restrict__ sums, double count,
                              const double *__restrict__ d_count, uint32_t C, float eps,
                              float momentum, float *__restrict__ running_mean,
                              float *__restrict__ running_var, float *__restrict__ mean,
                              float *__restrict__ invstd) {
  uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  if (d_count != nullptr) count = *d_count;
  double mu = sums[c] / count;
  double var = sums[C + c] / count - mu * mu;
  if (var < 0) var = 0;
  mean[c] = (float)mu;
  invstd[c] = (float)(1.0 / sqrt(var + (double)eps));
  if (running_mean != nullptr) {
    double unbiased = count > 1 ? var * count / (count - 1) : var;
    running_mean[c] = (float)((1.0 - momentum) * running_mean[c] + momentum * mu);
    running_var[c] = (float)((1.0 - momentum) * running_var[c] + momentum * unbiased);
  }
}

// MODE 0: y = (x - mean) * invstd * w + b (+ ReLU);  MODE 1: dx from dy (see file header)
template <typename T, int MODE>
__global__ void __launch_bounds__(kBnThreads)
k_bn_apply(const T *__restrict__ a, const T *__restrict__ x, const T *__restrict__ aux,
           const float *__restrict__ mean, const float *__restrict__ invstd,
           const float *__restrict__ weight, const float *__restrict__ bias,
           const double *__restrict__ gsums, double count, const double *__restrict__ d_count,
           uint32_t n, uint32_t C, uint32_t rows_per_cta, int relu, T *__restrict__ out,
           T *__restrict__ out2) {
  // aux: MODE 0 = residual added before the ReLU (may be NULL); MODE 1 = the layer's fused output
  // y whose sign is the ReLU mask (may be NULL).  out2 (MODE 1, may be NULL) = masked dy, the
  // gradient of the residual branch.
  const BnGeom g = bn_geom(C);
  if (threadIdx.x >= g.active) return;
  if (d_count != nullptr) count = *d_count;
  const uint32_t cg = threadIdx.x % g.G, r0 = threadIdx.x / g.G;
  const uint32_t row_begin = blockIdx.x * rows_per_cta;
  const uint32_t row_end = min(row_begin + rows_per_cta, n);
  float sc[8], sh[8], m[8], is[8], k1[8], k2[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const uint32_t c = cg * 8 + i;
    m[i] = mean[c];
    is[i] = invstd[c];
    const float w = weight != nullptr ? weight[c] : 1.f;
    if (MODE == 0) {
      sc[i] = is[i] * w;
      sh[i] = (bias != nullptr ? bias[c] : 0.f) - m[i] * sc[i];
    } else {
      sc[i] = is[i] * w;
      k1[i] = (float)(gsums[c] / count);
      k2[i] = (float)(gsums[C + c] / count);
    }
  }
  constexpr int U = 4;      // rows per iteration, all loads first (see k_bn_reduce)
  const uint32_t step = g.rows_per_pass;
  for (uint32_t r = row_begin + r0; r < row_end; r += U * step) {
    typename Vec8<T>::Raw ra[U], rb[U], rc[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const uint32_t ru = min(r + u * step, row_end - 1);
      ra[u] = Vec8<T>::load_raw(a + (size_t)ru * C + cg * 8);
      if (MODE == 1) rb[u] = Vec8<T>::load_raw(x + (size_t)ru * C + cg * 8);
      if (aux != nullptr) rc[u] = Vec8<T>::load_raw(aux + (size_t)ru * C + cg * 8);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const uint32_t ru = r + u * step;
      if (ru >= row_end) break;
      float va[8], vo[8], vc[8];
      Vec8<T>::unpack(ra[u], va);
      if (aux != nullptr) Vec8<T>::unpack(rc[u], vc);
      if (MODE == 0) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          float y = fmaf(va[i], sc[i], sh[i]) + (aux != nullptr ? vc[i] : 0.f);
          vo[i] = relu ? fmaxf(y, 0.f) : y;
        }
      } else {
        float vb[8];
        Vec8<T>::unpack(rb[u], vb);
        if (aux != nullptr) {
#pragma unroll
          for (int i = 0; i < 8; ++i) va[i] = vc[i] > 0.f ? va[i] : 0.f;
        }
        if (out2 != nullptr) Vec8<T>::store(out2 + (size_t)ru * C + cg * 8, va);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          float xhat = (vb[i] - m[i]) * is[i];
          vo[i] = (va[i] - k1[i] - xhat * k2[i]) * sc[i];
        }
      }
      Vec8<T>::store(out + (size_t)ru * C + cg * 8, vo);
    }
  }
}

static inline uint32_t bn_rows_per_cta(uint32_t n, uint32_t C, unsigned *grid) {
  const uint32_t rows_per_pass = kBnThreads / (C / 8);
  // ~8 CTAs per SM, at least 4 passes each
  uint32_t want = 8u * (uint32_t)num_sms();
  uint32_t rows = cdiv(n, want);
  uint32_t min_rows = 8 * rows_per_pass;
  if (rows < min_rows) rows = min_rows;
  rows = cdiv(rows, rows_per_pass) * rows_per_pass;
  *grid = cdiv(n, rows);
  return rows;
}

}  // namespace meb200

using namespace meb200;

#define MEB_BN_CHECK(C)                                                                   \
  MEB_CHECK_ARG((C) % 8 == 0 && (C) >= 8 && (C) <= 2048, "batch norm: C must be a multiple of 8 in [8, 2048] (got %u)", (unsigned)(C))

extern "C" {

int meb200_bn_finalize(const double *sums, double count, const double *d_count, uint32_t C,
                       float eps, float momentum, float *running_mean, float *running_var,
                       float *mean, float *invstd, void *stream_) {
  cudaStream_t s = (cudaStream_t)stream_;
  MEB_CHECK_ARG(sums && mean && invstd && (count > 0 || d_count != nullptr), "finalize arguments");
  k_bn_finalize<<<cdiv(C, 128), 128, 0, s>>>(sums, count, d_count, C, eps, momentum, running_mean, running_var, mean, invstd);
  MEB_LAUNCH_OK();
  return MEB200_OK;
}

int meb200_bn_apply_fused(const void *x, int dtype, uint32_t n, uint32_t C, const float *mean,
                          const float *invstd, const float *weight, const float *bias,
                          const void *residual, int relu, void *y, void *stream_) {
  cudaStream_t s = (cudaStream_t)stream_;
  MEB_BN_CHECK(C);
  if (n == 0) return MEB200_OK;
  unsigned grid;
  uint32_t rows = bn_rows_per_cta(n, C, &grid);
  MEB_DISPATCH_DTYPE(dtype, k_bn_apply<T, 0><<<grid, kBnThreads, 0, s>>>(
                                (const T *)x, nullptr, (const T *)residual, mean, invstd, weight,
                                bias, nullptr, 1.0, nullptr, n, C, rows, relu, (T *)y, nullptr));
  MEB_LAUNCH_OK();
  return MEB200_OK;
}

static int bn_launch_reduce(int mode, const void *a, const void *x, const void *ymask, int dtype,
                            uint32_t n, uint32_t C, const float *mean, const float *invstd,
                            double *sums, const BnTail &tail, cudaStream_t s) {
  unsigned grid;
  uint32_t rows = bn_rows_per_cta(n, C, &grid);
  if (grid > kBnMaxCtas) {          // one workspace slot per CTA
    const uint32_t rpp = kBnThreads / (C / 8);
    rows = cdiv(cdiv(n, kBnMaxCtas), rpp) * rpp;
    grid = cdiv(n, rows);
  }
  if (grid == 0) grid = 1;          // an empty rank still takes part in the exchange
  const size_t smem = bn_reduce_smem(C);
  MEB_DISPATCH_DTYPE(dtype,
    if (mode == 0)
      k_bn_reduce<T, 0><<<grid, kBnThreads, smem, s>>>((const T *)a, nullptr, nullptr, nullptr,
                                                      nullptr, n, C, rows, sums, tail);
    else
      k_bn_reduce<T, 1><<<grid, kBnThreads, smem, s>>>((const T *)a, (const T *)x,
                                                      (const T *)ymask, mean, invstd, n, C, rows,
                                                      sums, tail));
  MEB_LAUNCH_OK();
  return MEB200_OK;
}

uint64_t meb200_bn_workspace_bytes(void) { return kBnWorkspaceBytes; }

static inline uint32_t *bn_ticket(void *workspace) {
  return reinterpret_cast<uint32_t *>(reinterpret_cast<uint8_t *>(workspace) + kBnPartialBytes);
}

int meb200_bn_forward_train(const void *x, int dtype, uint32_t n, uint32_t C, const float *weight,
                            const float *bias, const void *residual, int relu, float eps,
                            float momentum, float *running_mean, float *running_var,
                            long long *num_batches_tracked, void *workspace, float *mean,
                            float *invstd, void *y, void *stream_) {
  cudaStream_t s = (cudaStream_t)stream_;
  MEB_BN_CHECK(C);
  MEB_CHECK_ARG(n > 0 && workspace && mean && invstd && y, "bn forward: empty input / null buffer");
  BnTail tail{};
  tail.ticket = bn_ticket(workspace);
  tail.num_batches_tracked = num_batches_tracked;
  tail.mean = mean; tail.invstd = invstd; tail.running_mean = running_mean; tail.running_var = running_var;
  tail.count = (double)n; tail.eps = eps; tail.momentum = momentum;
  int rc = bn_launch_reduce(0, x, nullptr, nullptr, dtype, n, C, nullptr, nullptr,
                            (double *)workspace, tail, s);
  if (rc != MEB200_OK) return rc;
  return meb200_bn_apply_fused(x, dtype, n, C, mean, invstd, weight, bias, residual, relu, y, stream_);
}

int meb200_bn_stats_to(const void *x, int dtype, uint32_t n, uint32_t C, void *workspace,
                       double *sums_out, void *stream_) {
  cudaStream_t s = (cudaStream_t)stream_;
  MEB_BN_CHECK(C);
  MEB_CHECK_ARG(workspace && sums_out, "bn stats: null buffer");
  if (n == 0) {
    MEB_CUDA(cudaMemsetAsync(sums_out, 0, 2 * (size_t)C * sizeof(double), s));
    return MEB200_OK;
  }
  BnTail tail{};
  tail.ticket = bn_ticket(workspace);
  tail.totals_out = sums_out;
  return bn_launch_reduce(0, x, nullptr, nullptr, dtype, n, C, nullptr, nullptr,
                          (double *)workspace, tail, s);
}

int meb200_bn_backward_reduce_to(const void *dy, const void *x, const void *y_mask, int dtype,
                                 uint32_t n, uint32_t C, const float *mean, const float *invstd,
                                 void *workspace, double *sums_out, float *grad_weight,
                                 float *grad_bias, void *stream_) {
  cudaStream_t s = (cudaStream_t)stream_;
  MEB_BN_CHECK(C);
  MEB_CHECK_ARG(workspace && sums_out, "bn backward reduce: null buffer");
  if (n == 0) {
    MEB_CUDA(cudaMemsetAsync(sums_out, 0, 2 * (size_t)C * sizeof(double), s));
    if (grad_weight) MEB_CUDA(cudaMemsetAsync(grad_weight, 0, (size_t)C * sizeof(float), s));
    if (grad_bias) MEB_CUDA(cudaMemsetAsync(grad_bias, 0, (size_t)C * sizeof(float), s));
    return MEB200_OK;
  }
  BnTail tail{};
  tail.ticket = bn_ticket(workspace);
  tail.totals_out = sums_out;
  tail.grad_weight = grad_weight;
  tail.grad_bias = grad_bias;
  return bn_launch_reduce(1, dy, x, y_mask, dtype, n, C, mean, invstd, (double *)workspace, tail, s);
}

static void bn_tail_peer(BnTail &tail, const void *peer_bases_dev, uint64_t slot_offset,
                         uint32_t seq, uint32_t rank, uint32_t world) {
  tail.peer_bases = (uint8_t *const *)peer_bases_dev;
  tail.peer_slot_offset = slot_offset;
  tail.peer_seq = seq; tail.peer_rank = rank; tail.peer_world = world;
}
#define MEB_PEER_CHECK()                                                                          \
  MEB_CHECK_ARG(peer_bases_dev != nullptr && world >= 1 && world <= 256 && rank < world &&        \
                    slot_offset_bytes >= 1024 && slot_offset_bytes % 8 == 0 && seq != 0,         \
                "peer exchange: bases / rank %u of %u / slot offset / sequence number",          \
                (unsigned)rank, (unsigned)world)

int meb200_bn_forward_train_peer(const void *x, int dtype, uint32_t n, uint32_t C,
                                 const float *weight, const float *bias, const void *residual,
                                 int relu, float eps, float momentum, float *running_mean,
                                 float *running_var, long long *num_batches_tracked,
                                 void *workspace, const void *peer_bases_dev,
                                 uint64_t slot_offset_bytes, uint32_t seq, uint32_t rank,
                                 uint32_t world, float *mean, float *invstd, double *total_rows,
                                 void *y, void *stream_) {
  cudaStream_t s = (cudaStream_t)stream_;
  MEB_BN_CHECK(C);
  MEB_CHECK_ARG(workspace && mean && invstd && total_rows && (y || n == 0), "bn forward: null buffer");
  MEB_PEER_CHECK();
  BnTail tail{};
  tail.ticket = bn_ticket(workspace);
  tail.mean = mean; tail.invstd = invstd; tail.running_mean = running_mean; tail.running_var = running_var;
  tail.count = (double)n; tail.eps = eps; tail.momentum = momentum;
  tail.total_rows_out = total_rows;
  tail.num_batches_tracked = num_batches_tracked;
  bn_tail_peer(tail, peer_bases_dev, slot_offset_bytes, seq, rank, world);
  int rc = bn_launch_reduce(0, x, nullptr, nullptr, dtype, n, C, nullptr, nullptr,
                            (double *)workspace, tail, s);
  if (rc != MEB200_OK || n == 0) return rc;
  return meb200_bn_apply_fused(x, dtype, n, C, mean, invstd, weight, bias, residual, relu, y, stream_);
}

int meb200_bn_backward_reduce_peer(const void *dy, const void *x, const void *y_mask, int dtype,
                                   uint32_t n, uint32_t C, const float *mean, const float *invstd,
                                   void *workspace, const void *peer_bases_dev,
                                   uint64_t slot_offset_bytes, uint32_t seq, uint32_t rank,
                                   uint32_t world, double *sums_out, float *grad_weight,
                                   float *grad_bias, void *stream_) {
  cudaStream_t s = (cudaStream_t)stream_;
  MEB_BN_CHECK(C);
  MEB_CHECK_ARG(workspace && sums_out, "bn backward reduce: null buffer");
  MEB_PEER_CHECK();
  BnTail tail{};
  tail.ticket = bn_ticket(workspace);
  tail.totals_out = sums_out;
  tail.grad_weight = grad_weight;
  tail.grad_bias = grad_bias;
  bn_tail_peer(tail, peer_bases_dev, slot_offset_bytes, seq, rank, world);
  return bn_launch_reduce(1, dy, x, y_mask, dtype, n, C, mean, invstd, (double *)workspace, tail, s);
}

int meb200_bn_backward_apply_fused(const void *dy, const void *x, const void *y_mask, int dtype,
                                   uint32_t n, uint32_t C, const float *mean, const float *invstd,
                                   const float *weight, const double *sums, double count,
                                   const double *d_count, void *dx, void *d_residual,
                                   void *stream_) {
  cudaStream_t s = (cudaStream_t)stream_;
  MEB_BN_CHECK(C);
  if (n == 0) return MEB200_OK;
  MEB_CHECK_ARG(count > 0 || d_count != nullptr, "count");
  unsigned grid;
  uint32_t rows = bn_rows_per_cta(n, C, &grid);
  MEB_DISPATCH_DTYPE(dtype, k_bn_apply<T, 1><<<grid, kBnThreads, 0, s>>>(
                                (const T *)dy, (const T *)x, (const T *)y_mask, mean, invstd,
                                weight, nullptr, sums, count, d_count, n, C, rows, 0, (T *)dx,
                                (T *)d_residual));
  MEB_LAUNCH_OK();
  return MEB200_OK;
}

}
