// Hopper (sm_90a) sparse convolution on the tensor cores: warpgroup MMA (wgmma.mma_async) with
// both operands gathered into shared memory by cp.async, fp32 accumulators in registers.
//
//   forward / dgrad : out[r, :] = sum_k A[nbr[k][r], :] @ B_k              (k_conv_wg)
//   wgrad           : dW[k]     += In[rows_in, :]^T @ dOut[rows_out, :]     (k_wgrad_wg)
//
// Replaces the reference's per-offset SIMT tile-matmul with per-element atomicAdd
// (src/convolution_kernel.cu:114-180,320-496): forward and dgrad write every output row exactly
// once (no atomics, no zero fill, deterministic) and the fp32 accumulator stays in registers
// until the epilogue converts it.
//
// Shared-memory tiles use the no-swizzle "core matrix" layout wgmma reads directly: 16-byte
// chunk j (channels 8j..8j+7) of tile row r lives at ((r / 8) * chunks + j) * 128 + (r % 8) * 16,
// so every gathered 16-byte piece of a feature row is one cp.async (missing neighbours are
// zero-filled by the copy).  Forward tiles are read K-major (tile rows = M / N); wgrad tiles hold
// rows of the reduction axis and are read MN-major (transposed) by the same instruction.
//
// CTA = 2 warpgroups (256 threads).  A ring of tc::kStages stages; every thread issues the copies
// of stage s + 2 before the MMAs of stage s, one __syncthreads per stage, and each warpgroup keeps
// one wgmma group in flight behind the barrier.
#include <stdlib.h>
#include <string.h>
#include <type_traits>

#include "conv_tc.cuh"
#include "ptx.cuh"
#include "tc_config.h"

namespace meb200 {

using namespace ptx;
using tc::kStages;

constexpr int kThreads = 256;
constexpr uint32_t kNoLimit = 0xFFFFFFFFu;

// byte offset of 16-byte chunk j of tile row r (tile of `chunks` chunks per row)
__device__ __forceinline__ uint32_t cm_off(uint32_t r, uint32_t j, uint32_t chunks) {
  return (((r >> 3) * chunks + j) << 7) + ((r & 7u) << 4);
}

template <typename T>
constexpr bool kIsBf16 = std::is_same<T, __nv_bfloat16>::value;

template <typename T>
__device__ __forceinline__ uint32_t pack2(float a, float b);
template <>
__device__ __forceinline__ uint32_t pack2<__nv_bfloat16>(float a, float b) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t *>(&h);
}
template <>
__device__ __forceinline__ uint32_t pack2<__half>(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t *>(&h);
}

__device__ __forceinline__ uint8_t *align1k(uint8_t *p) {
  return reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(p) + 1023) & ~uintptr_t(1023));
}

// =====================================================================================
// forward / dgrad
// =====================================================================================
struct FwdParams {
  const void *A;          // [n_a, c_red] gathered operand (stem: [n_a, 4])
  const void *B;          // [K][*][c_red] operand B (reduction contiguous), at this slice's row 0
  const int32_t *nbr;     // [K, n_rows]
  void *out;              // [n_rows, out_ld], at this slice's column 0
  uint64_t b_k_stride;    // elements between the offsets of B
  uint32_t c_red, c_cols, K, n_rows;
  uint32_t n_a;           // rows of A (gather indices >= n_a read as zero rows)
  uint32_t out_ld, bk, out_f32;
  uint32_t stem_K;        // > 0: network stem, virtual channel 4 k + c = A[nbr[k][r]][c], k < stem_K
};

// NT wgmma instructions of N = NI columns each cover the c_cols = NI * NT columns of the slice.
template <typename T, int NI, int NT>
__global__ void __launch_bounds__(kThreads, 1) k_conv_wg(const FwdParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t s0 = smem_u32(align1k(smem_raw));
  const uint32_t tid = threadIdx.x, wg = tid >> 7, warp = tid >> 5, lane = tid & 31;
  const uint32_t row0 = blockIdx.x * tc::kFwdRows;
  const uint32_t bk = p.bk, ch = bk / 8, lch = bk == 64 ? 3 : (bk == 32 ? 2 : 1);
  const uint32_t a_bytes = tc::kFwdRows * bk * 2, stage_bytes = a_bytes + p.c_cols * bk * 2;
  const uint32_t nch = p.c_red / bk, n_st = p.K * nch;
  const T *A = reinterpret_cast<const T *>(p.A);
  const T *B = reinterpret_cast<const T *>(p.B);
  const uint32_t ar = tid >> 1, arow = row0 + ar;     // two threads per tile row of A
  const bool row_ok = arow < p.n_rows;

  auto load = [&](uint32_t s) {
    const uint32_t k = s / nch, c0 = (s - k * nch) * bk;
    const uint32_t base = s0 + (s % kStages) * stage_bytes;
    if (p.stem_K == 0) {
      const int32_t src = row_ok ? __ldg(p.nbr + (size_t)k * p.n_rows + arow) : -1;
      const bool ok = src >= 0 && (uint32_t)src < p.n_a;
      const T *rp = A + (size_t)(ok ? src : 0) * p.c_red + c0;
      for (uint32_t j = tid & 1u; j < ch; j += 2)
        cp_async16(base + cm_off(ar, j, ch), rp + 8 * j, ok ? 16u : 0u);
    } else {
      // chunk j = virtual channels c0 + 8j..: offsets (c0 + 8j) / 4 + {0, 1}, 8 bytes each
      for (uint32_t j = tid & 1u; j < ch; j += 2)
        for (uint32_t h = 0; h < 2; ++h) {
          const uint32_t kk = (c0 + 8 * j) / 4 + h;
          const int32_t src =
              (row_ok && kk < p.stem_K) ? __ldg(p.nbr + (size_t)kk * p.n_rows + arow) : -1;
          const bool ok = src >= 0 && (uint32_t)src < p.n_a;
          cp_async8(base + cm_off(ar, j, ch) + 8 * h, A + (size_t)(ok ? src : 0) * 4, ok ? 8u : 0u);
        }
    }
    const T *Bk = B + (size_t)k * p.b_k_stride + c0;
    const uint32_t nb = p.c_cols * ch;
    for (uint32_t i = tid; i < nb; i += kThreads) {
      const uint32_t n = i >> lch, j = i & (ch - 1);
      cp_async16(base + a_bytes + cm_off(n, j, ch), Bk + (size_t)n * p.c_red + 8 * j, 16u);
    }
  };

  float acc[NT][NI / 2];
#pragma unroll
  for (int i = 0; i < NT; ++i)
#pragma unroll
    for (int q = 0; q < NI / 2; ++q) acc[i][q] = 0.f;

  for (uint32_t s = 0; s < kStages - 2; ++s) {
    if (s < n_st) load(s);
    cp_async_commit();
  }
  const uint32_t sbo = ch * 128;        // next 8 rows; the next 8 channels are 128 B on (lbo)
  for (uint32_t s = 0; s < n_st; ++s) {
    cp_async_wait<kStages - 3>();       // this thread's copies of stage s have landed
    fence_proxy_async();
    __syncthreads();                    // ... everybody's; the MMAs of stage s - 2 have retired
    if (s + kStages - 2 < n_st) load(s + kStages - 2);   // into the slot of stage s - 2
    cp_async_commit();
    const uint32_t a0 = s0 + (s % kStages) * stage_bytes + wg * 64 * bk * 2;
    const uint32_t b0 = s0 + (s % kStages) * stage_bytes + a_bytes;
    wgmma_fence();
    for (uint32_t kk = 0; kk < bk / 16; ++kk) {
      const uint64_t da = wgmma_desc(a0 + kk * 256, 128, sbo);
#pragma unroll
      for (int i = 0; i < NT; ++i)
        wgmma<NI, kIsBf16<T>, 0, 0>(acc[i], da, wgmma_desc(b0 + i * NI * bk * 2 + kk * 256, 128, sbo));
    }
    wgmma_commit();
    wgmma_wait<1>();
  }
  wgmma_wait<0>();

  const uint32_t g = lane >> 2, t = lane & 3;
  const uint32_t rbase = row0 + wg * 64 + (warp & 3) * 16 + g;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const uint32_t r = rbase + 8 * h;
    if (r >= p.n_rows) continue;
#pragma unroll
    for (int i = 0; i < NT; ++i)
#pragma unroll
      for (int j = 0; j < NI / 8; ++j) {
        const uint32_t col = i * NI + 8 * j + 2 * t;
        const float v0 = acc[i][4 * j + 2 * h], v1 = acc[i][4 * j + 2 * h + 1];
        if (p.out_f32)
          *reinterpret_cast<float2 *>(reinterpret_cast<float *>(p.out) + (size_t)r * p.out_ld + col) =
              make_float2(v0, v1);
        else
          *reinterpret_cast<uint32_t *>(reinterpret_cast<T *>(p.out) + (size_t)r * p.out_ld + col) =
              pack2<T>(v0, v1);
      }
  }
}

// =====================================================================================
// wgrad:  dW[k][ci][co] += sum over (input row i, output row o) pairs of offset k of
//         In[i][ci] * dOut[o][co]
// GEMM view: D[M = ci][N = co] over the reduction axis "pair"; a stage = 64 pairs.  One CTA owns
// (offset k, 128 input channels, a share of the pairs).  With one share per offset it stores its
// sums into dW; otherwise share s stores into partial[s] and launch_split_sum adds the shares in
// order, so the result does not depend on the order in which CTAs finish.  The pairs come from
//   pair mode   : the compacted lists of meb200_kernel_map_pairs (segments (row chunk, offset),
//                 padded with -1); the CTA takes the same fraction of every chunk's segment
//   dense mode  : all output rows o of the table, i = nbr[k][o]
//   stem mode   : dense, M = virtual channels 4 k + c of 4-channel input rows (K = 1 layer)
// =====================================================================================
struct WgParams {
  const void *in;          // [n_in, c_in] (stem: [n_in, 4], c_in = virtual channels)
  const void *gout;        // [n_out, c_out]
  const int32_t *nbr;      // [K, n_out] (dense and stem modes)
  const int32_t *pin, *pout, *seg;   // pair mode when pin != NULL; seg[n_chunks * K + 1]
  float *dW;               // [K, c_in, c_out]
  float *partial;          // [n_splits][K, c_in, c_out] when n_splits > 1
  uint32_t c_in, c_out, K, n_in, n_out, n_chunks, n_splits;
  uint32_t stem_K;         // > 0: stem mode
};

// This CTA's share [lo, hi) of chunk c's pairs of offset k, in whole 64-pair stages.
__device__ __forceinline__ void wg_range(const WgParams &p, uint32_t k, uint32_t c, uint32_t &lo,
                                         uint32_t &hi) {
  uint32_t a = 0, b = p.n_out;
  if (p.pin != nullptr) {
    a = (uint32_t)__ldg(p.seg + (size_t)c * p.K + k);
    b = (uint32_t)__ldg(p.seg + (size_t)c * p.K + k + 1);
  }
  const uint64_t n = (b - a + tc::kWgRows - 1) / tc::kWgRows;
  lo = a + (uint32_t)(n * blockIdx.x / p.n_splits) * tc::kWgRows;
  hi = a + (uint32_t)(n * (blockIdx.x + 1) / p.n_splits) * tc::kWgRows;
  if (hi > b) hi = b;
  if (lo > hi) lo = hi;
}

template <typename T, int NI, int NT>
__global__ void __launch_bounds__(kThreads, 1) k_wgrad_wg(const WgParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t s0 = smem_u32(align1k(smem_raw));
  const uint32_t tid = threadIdx.x, wg = tid >> 7, warp = tid >> 5, lane = tid & 31;
  const uint32_t k = blockIdx.z, ci0 = blockIdx.y * tc::kWgChannels;
  constexpr uint32_t kChA = tc::kWgChannels / 8;                    // 16 chunks per A row
  constexpr uint32_t a_bytes = tc::kWgRows * tc::kWgChannels * 2;
  const uint32_t chB = p.c_out / 8, stage_bytes = a_bytes + tc::kWgRows * p.c_out * 2;
  const uint32_t n_chunks = p.pin != nullptr ? p.n_chunks : 1u;
  const T *In = reinterpret_cast<const T *>(p.in);
  const T *G = reinterpret_cast<const T *>(p.gout);

  uint32_t n_st = 0;
  for (uint32_t c = 0; c < n_chunks; ++c) {
    uint32_t lo, hi;
    wg_range(p, k, c, lo, hi);
    n_st += (hi - lo + tc::kWgRows - 1) / tc::kWgRows;
  }
  // producer cursor: stage [pos, min(pos + 64, end)) of chunk wc
  uint32_t wc = 0, pos = 0, end = 0;
  auto open = [&]() {
    for (; wc < n_chunks; ++wc) {
      wg_range(p, k, wc, pos, end);
      if (pos < end) return;
    }
  };
  open();

  const uint32_t ar = tid >> 2;         // four threads per A row
  auto load = [&](uint32_t s) {
    const uint32_t base = s0 + (s % kStages) * stage_bytes;
    const uint32_t e = pos;             // this stage's first pair
    if (p.stem_K == 0) {
      int32_t src = -1;
      if (e + ar < end)
        src = p.pin != nullptr ? __ldg(p.pin + e + ar) : __ldg(p.nbr + (size_t)k * p.n_out + e + ar);
      const bool ok = src >= 0 && (uint32_t)src < p.n_in;
      const T *rp = In + (size_t)(ok ? src : 0) * p.c_in + ci0;
#pragma unroll
      for (uint32_t m = 0; m < 4; ++m) {
        const uint32_t j = (tid & 3u) + 4 * m;
        const bool okj = ok && ci0 + 8 * j < p.c_in;
        cp_async16(base + cm_off(ar, j, kChA), okj ? rp + 8 * j : In, okj ? 16u : 0u);
      }
    } else {
#pragma unroll
      for (uint32_t m = 0; m < 4; ++m) {
        const uint32_t j = (tid & 3u) + 4 * m;
#pragma unroll
        for (uint32_t h = 0; h < 2; ++h) {
          const uint32_t kk = (ci0 + 8 * j) / 4 + h;
          const int32_t src = (e + ar < end && kk < p.stem_K)
                                  ? __ldg(p.nbr + (size_t)kk * p.n_out + e + ar) : -1;
          const bool ok = src >= 0 && (uint32_t)src < p.n_in;
          cp_async8(base + cm_off(ar, j, kChA) + 8 * h, In + (size_t)(ok ? src : 0) * 4, ok ? 8u : 0u);
        }
      }
    }
    const uint32_t nb = tc::kWgRows * chB;
    for (uint32_t i = tid; i < nb; i += kThreads) {
      const uint32_t r = i / chB, j = i - r * chB;
      int32_t o = -1;
      if (e + r < end) o = p.pin != nullptr ? __ldg(p.pout + e + r) : (int32_t)(e + r);
      const bool ok = o >= 0 && (uint32_t)o < p.n_out;
      cp_async16(base + a_bytes + cm_off(r, j, chB), G + (size_t)(ok ? o : 0) * p.c_out + 8 * j,
                 ok ? 16u : 0u);
    }
    pos += tc::kWgRows;
    if (pos >= end) { ++wc; open(); }
  };

  float acc[NT][NI / 2];
#pragma unroll
  for (int i = 0; i < NT; ++i)
#pragma unroll
    for (int q = 0; q < NI / 2; ++q) acc[i][q] = 0.f;

  for (uint32_t s = 0; s < kStages - 2; ++s) {
    if (s < n_st) load(s);
    cp_async_commit();
  }
  // (a warpgroup whose 64 channels lie past c_in multiplies the zero-filled half of the tile:
  // branching around wgmma would serialise the instructions of the whole kernel)
  for (uint32_t s = 0; s < n_st; ++s) {
    cp_async_wait<kStages - 3>();
    fence_proxy_async();
    __syncthreads();
    if (s + kStages - 2 < n_st) load(s + kStages - 2);
    cp_async_commit();
    // MN-major: the next 8 channels are 128 B on (sbo), the next 8 rows one row of chunks (lbo)
    const uint32_t a0 = s0 + (s % kStages) * stage_bytes + wg * 8 * 128;
    const uint32_t b0 = s0 + (s % kStages) * stage_bytes + a_bytes;
    wgmma_fence();
#pragma unroll
    for (uint32_t kk = 0; kk < tc::kWgRows / 16; ++kk) {
      const uint64_t da = wgmma_desc(a0 + kk * 2 * kChA * 128, kChA * 128, 128);
#pragma unroll
      for (int i = 0; i < NT; ++i)
        wgmma<NI, kIsBf16<T>, 1, 1>(
            acc[i], da, wgmma_desc(b0 + i * (NI / 8) * 128 + kk * 2 * chB * 128, chB * 128, 128));
    }
    wgmma_commit();
    wgmma_wait<1>();
  }
  wgmma_wait<0>();

  const uint32_t g = lane >> 2, t = lane & 3;
  const uint32_t cbase = ci0 + wg * 64 + (warp & 3) * 16 + g;
  const size_t dw_elems = (size_t)p.K * p.c_in * p.c_out;   // every element written by one CTA
  float *dWk = (p.n_splits > 1 ? p.partial + blockIdx.x * dw_elems : p.dW) + (size_t)k * p.c_in * p.c_out;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const uint32_t ci = cbase + 8 * h;
    if (ci >= p.c_in) continue;
#pragma unroll
    for (int i = 0; i < NT; ++i)
#pragma unroll
      for (int j = 0; j < NI / 8; ++j) {
        *reinterpret_cast<float2 *>(dWk + (size_t)ci * p.c_out + i * NI + 8 * j + 2 * t) =
            make_float2(acc[i][4 * j + 2 * h], acc[i][4 * j + 2 * h + 1]);
      }
  }
}


// ---- weight packing ----------------------------------------------------------------------------
// Per-optimizer-step weight packing: fp32 master W[k][ci][co] -> feature dtype in the two
// operand-B layouts of the wgmma kernels, in one pass:
//   Wc [k][ci][co]  dgrad operand B            Wt [k][co][ci]  forward operand B
// One CTA packs the 32 x 32 tile (k, ci0.., co0..).
template <typename T>
__device__ __forceinline__ void pack_tile(const float *__restrict__ W, T *__restrict__ Wc,
                                          T *__restrict__ Wt, uint32_t c_in, uint32_t c_out,
                                          uint32_t k, uint32_t ci0, uint32_t co0) {
  __shared__ float tile[32][33];
  const size_t base = (size_t)k * c_in * c_out;
  const uint32_t tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (uint32_t i = ty; i < 32; i += 8)
    if (ci0 + i < c_in && co0 + tx < c_out) {
      const float v = W[base + (size_t)(ci0 + i) * c_out + co0 + tx];
      tile[i][tx] = v;
      Wc[base + (size_t)(ci0 + i) * c_out + co0 + tx] = from_f32<T>(v);
    }
  __syncthreads();
  for (uint32_t i = ty; i < 32; i += 8)
    if (co0 + i < c_out && ci0 + tx < c_in)
      Wt[base + (size_t)(co0 + i) * c_in + ci0 + tx] = from_f32<T>(tile[tx][i]);
}

template <typename T>
__global__ void __launch_bounds__(256)
k_pack_w(const float *__restrict__ W, T *__restrict__ Wc, T *__restrict__ Wt, uint32_t c_in,
         uint32_t c_out) {
  pack_tile<T>(W, Wc, Wt, c_in, c_out, blockIdx.z, blockIdx.y * 32, blockIdx.x * 32);
}

// All layers of a network in ONE launch (the weights of every layer change together, at the
// optimizer step): job j re-packs one [K, c_in, c_out] tensor exactly as k_pack_w does; a CTA
// finds its job by binary search over the jobs' first-tile indices.
template <typename T>
__global__ void __launch_bounds__(256)
k_pack_w_batched(const PackJob *__restrict__ jobs, uint32_t n_jobs) {
  uint32_t lo = 0, hi = n_jobs - 1;
  while (lo < hi) {                       // last job whose tile_begin <= blockIdx.x
    const uint32_t mid = (lo + hi + 1) >> 1;
    if (jobs[mid].tile_begin <= blockIdx.x) lo = mid; else hi = mid - 1;
  }
  const PackJob job = jobs[lo];
  const uint32_t c_in = job.c_in, c_out = job.c_out;
  const uint32_t tx_n = (c_out + 31u) / 32u, ty_n = (c_in + 31u) / 32u;
  uint32_t t = blockIdx.x - job.tile_begin;
  const uint32_t bx = t % tx_n; t /= tx_n;
  const uint32_t by = t % ty_n, bz = t / ty_n;
  pack_tile<T>(reinterpret_cast<const float *>(job.w), reinterpret_cast<T *>(job.w_cast),
               reinterpret_cast<T *>(job.w_t), c_in, c_out, bz, by * 32, bx * 32);
}

int conv_pack_weights_batched(const PackJob *jobs_dev, uint32_t n_jobs, uint32_t total_tiles,
                              int dtype, cudaStream_t stream) {
  if (n_jobs == 0 || total_tiles == 0) return MEB200_OK;
  if (dtype == MEB200_BF16)
    k_pack_w_batched<__nv_bfloat16><<<total_tiles, 256, 0, stream>>>(jobs_dev, n_jobs);
  else
    k_pack_w_batched<__half><<<total_tiles, 256, 0, stream>>>(jobs_dev, n_jobs);
  MEB_LAUNCH_OK();
  return MEB200_OK;
}

int conv_pack_weights(const float *W, uint32_t K, uint32_t c_in, uint32_t c_out, int dtype,
                      void *w_cast, void *w_t, cudaStream_t stream) {
  dim3 grid(cdiv(c_out, 32), cdiv(c_in, 32), K);
  if (dtype == MEB200_BF16)
    k_pack_w<__nv_bfloat16><<<grid, 256, 0, stream>>>(W, (__nv_bfloat16 *)w_cast,
                                                      (__nv_bfloat16 *)w_t, c_in, c_out);
  else
    k_pack_w<__half><<<grid, 256, 0, stream>>>(W, (__half *)w_cast, (__half *)w_t, c_in, c_out);
  MEB_LAUNCH_OK();
  return MEB200_OK;
}

// Opt a kernel in to >48 KB of dynamic shared memory.  The attribute is per (function, device):
// the flags are keyed on the function pointer VALUE and the current device (a single static flag
// would be shared by every instantiation of a kernel template).
static int ensure_big_smem(const void *fn) {
  constexpr int kMaxDev = 16, kMaxFn = 256;
  static const void *fns[kMaxFn];
  static uint16_t done[kMaxFn];
  static int n_fns = 0;
  int dev = 0;
  MEB_CUDA(cudaGetDevice(&dev));
  int slot = -1;
  for (int i = 0; i < n_fns; ++i) if (fns[i] == fn) { slot = i; break; }
  if (slot >= 0 && dev < kMaxDev && (done[slot] >> dev & 1)) return MEB200_OK;
  MEB_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
  if (slot < 0 && n_fns < kMaxFn) { slot = n_fns++; fns[slot] = fn; done[slot] = 0; }
  if (slot >= 0 && dev < kMaxDev) done[slot] |= (uint16_t)(1u << dev);
  return MEB200_OK;
}
#define MEB_BIG_SMEM(kern) do { int rc__ = ensure_big_smem((const void *)(kern)); if (rc__ != MEB200_OK) return rc__; } while (0)

// ---- launches ---------------------------------------------------------------------------------
// c_cols (a multiple of 16, <= 256) -> NT instructions of the widest N in {64, 32, 16} dividing it
#define MEB_COLS_DISPATCH(cols, L)                                                      \
  switch ((cols) / 16) {                                                                \
    case 1: return L(16, 1);   case 2: return L(32, 1);   case 3: return L(16, 3);      \
    case 4: return L(64, 1);   case 5: return L(16, 5);   case 6: return L(32, 3);      \
    case 7: return L(16, 7);   case 8: return L(64, 2);   case 9: return L(16, 9);      \
    case 10: return L(32, 5);  case 11: return L(16, 11); case 12: return L(64, 3);     \
    case 13: return L(16, 13); case 14: return L(32, 7);  case 15: return L(16, 15);    \
    case 16: return L(64, 4);  default: break;                                          \
  }

template <typename T, int NI, int NT>
static int launch_fwd(const FwdParams &p, cudaStream_t stream) {
  auto kern = k_conv_wg<T, NI, NT>;
  MEB_BIG_SMEM(kern);
  kern<<<cdiv(p.n_rows, tc::kFwdRows), kThreads, tc::fwd_smem_bytes(p.bk, p.c_cols), stream>>>(p);
  count_tc_launch();
  MEB_LAUNCH_OK();
  return MEB200_OK;
}
template <typename T>
static int dispatch_fwd(const FwdParams &p, cudaStream_t stream) {
#define MEB_L(NI, NT) launch_fwd<T, NI, NT>(p, stream)
  MEB_COLS_DISPATCH(p.c_cols, MEB_L)
#undef MEB_L
  set_error("conv tc: %u output columns per launch", p.c_cols);
  return MEB200_ERR_UNSUPPORTED;
}
static int run_fwd(int dtype, const FwdParams &p, cudaStream_t stream) {
  return dtype == MEB200_BF16 ? dispatch_fwd<__nv_bfloat16>(p, stream)
                              : dispatch_fwd<__half>(p, stream);
}

template <typename T, int NI, int NT>
static int launch_wgrad(const WgParams &p, dim3 grid, cudaStream_t stream) {
  auto kern = k_wgrad_wg<T, NI, NT>;
  MEB_BIG_SMEM(kern);
  kern<<<grid, kThreads, tc::wgrad_smem_bytes(p.c_out), stream>>>(p);
  count_tc_launch();
  MEB_LAUNCH_OK();
  return MEB200_OK;
}
template <typename T>
static int dispatch_wgrad(const WgParams &p, dim3 grid, cudaStream_t stream) {
#define MEB_L(NI, NT) launch_wgrad<T, NI, NT>(p, grid, stream)
  MEB_COLS_DISPATCH(p.c_out, MEB_L)
#undef MEB_L
  set_error("wgrad tc: %u output channels", p.c_out);
  return MEB200_ERR_UNSUPPORTED;
}
static uint32_t wgrad_planned_splits(uint32_t c_in, uint32_t K, uint32_t est_stages) {
  return tc::wgrad_splits(est_stages, K, cdiv(c_in, tc::kWgChannels), (uint32_t)num_sms());
}

uint64_t conv_wgrad_workspace_bytes(uint32_t c_in, uint32_t c_out, uint32_t K, uint32_t n_out) {
  const uint32_t splits = wgrad_planned_splits(c_in, K, cdiv(n_out, tc::kWgRows));
  return splits > 1 ? (uint64_t)splits * K * c_in * c_out * sizeof(float) : 0;
}

// grid = (row splits, 128-channel tiles of c_in, offsets).  The splits are what the workspace
// holds of the planned ones (one split: no workspace, the CTAs store into dW directly).
static int run_wgrad(int dtype, WgParams p, uint32_t K_grid, uint32_t est_stages, void *workspace,
                     uint64_t workspace_bytes, cudaStream_t stream) {
  const uint32_t m_tiles = cdiv(p.c_in, tc::kWgChannels);
  const size_t dw_elems = (size_t)K_grid * p.c_in * p.c_out;
  p.n_splits = workspace_splits(wgrad_planned_splits(p.c_in, K_grid, est_stages), workspace,
                                workspace_bytes, dw_elems * sizeof(float));
  p.partial = p.n_splits > 1 ? reinterpret_cast<float *>(workspace) : nullptr;
  const dim3 grid(p.n_splits, m_tiles, K_grid);
  const int rc = dtype == MEB200_BF16 ? dispatch_wgrad<__nv_bfloat16>(p, grid, stream)
                                      : dispatch_wgrad<__half>(p, grid, stream);
  if (rc != MEB200_OK || p.n_splits == 1) return rc;
  return launch_split_sum(p.partial, p.dW, dw_elems, p.n_splits, stream);
}

// ---- forward / dgrad ----------------------------------------------------------------------------
bool conv_tc_supported(int dtype, uint32_t c_reduce, uint32_t c_cols) {
  if (dtype != MEB200_BF16 && dtype != MEB200_F16) return false;
  if (tc::fwd_bk(c_reduce) == 0) return false;
  return c_cols % 16 == 0 && c_cols >= 16 && c_cols <= 1024;
}

int conv_forward_tc(const void *A, int dtype, uint32_t n_a, uint32_t c_reduce, const void *B,
                    uint32_t K, uint32_t c_cols, const int32_t *nbr, uint32_t n_rows, void *out,
                    int out_dtype, cudaStream_t stream) {
  if (n_rows == 0) return MEB200_OK;
  MEB_CHECK_ARG(conv_tc_supported(dtype, c_reduce, c_cols), "shape not supported by tc path");
  if (!aligned(16, A, B)) {
    set_error("conv tc: operands must be 16-byte aligned");
    return MEB200_ERR_UNSUPPORTED;
  }
  const uint8_t *Wb = reinterpret_cast<const uint8_t *>(B);
  // one launch per slice of <= 256 output columns
  const size_t out_esz = out_dtype == MEB200_F32 ? 4 : 2;
  for (uint32_t n0 = 0; n0 < c_cols; n0 += tc::kMaxCols) {
    FwdParams p{};
    p.A = A; p.B = Wb + (size_t)n0 * c_reduce * 2; p.nbr = nbr;
    p.out = reinterpret_cast<uint8_t *>(out) + (size_t)n0 * out_esz;
    p.b_k_stride = (uint64_t)c_cols * c_reduce;
    p.c_red = c_reduce; p.c_cols = c_cols - n0 < tc::kMaxCols ? c_cols - n0 : tc::kMaxCols;
    p.K = K; p.n_rows = n_rows; p.n_a = n_a; p.out_ld = c_cols;
    p.bk = tc::fwd_bk(c_reduce); p.out_f32 = out_dtype == MEB200_F32;
    const int rc = run_fwd(dtype, p, stream);
    if (rc != MEB200_OK) return rc;
  }
  return MEB200_OK;
}

// ---- network stem: rows of 4 channels, see FwdParams::stem_K ------------------------------------
static uint32_t stem_virtual(uint32_t K) { return 4u * ((K + 15u) / 16u * 16u); }

bool conv_stem_tc_supported(int dtype, uint32_t K, uint32_t c_cols) {
  if (dtype != MEB200_BF16 && dtype != MEB200_F16) return false;
  return K >= 1 && c_cols % 16 == 0 && c_cols >= 16 && c_cols <= tc::kMaxCols;
}

int conv_stem_forward_tc(const void *A4, int dtype, uint32_t K, const void *Wv, uint32_t c_cols,
                         const int32_t *nbr, uint32_t n_rows, void *out, int out_dtype,
                         cudaStream_t stream) {
  if (n_rows == 0) return MEB200_OK;
  MEB_CHECK_ARG(conv_stem_tc_supported(dtype, K, c_cols), "stem forward: K=%u c_out=%u", K, c_cols);
  if (!aligned(8, A4) || !aligned(16, Wv)) {
    set_error("stem forward: operands must be 8 / 16-byte aligned");
    return MEB200_ERR_UNSUPPORTED;
  }
  FwdParams p{};
  p.A = A4; p.B = Wv; p.nbr = nbr; p.out = out;
  p.c_red = stem_virtual(K); p.c_cols = c_cols; p.K = 1; p.n_rows = n_rows; p.n_a = kNoLimit;
  p.out_ld = c_cols; p.bk = tc::fwd_bk(p.c_red); p.out_f32 = out_dtype == MEB200_F32;
  p.stem_K = K;
  return run_fwd(dtype, p, stream);
}

bool conv_stem_wgrad_tc_supported(int dtype, uint32_t K, uint32_t c_out) {
  return conv_stem_tc_supported(dtype, K, c_out);
}

// dWv: [4 * 16 ceil(K / 16), c_out] fp32 (virtual channel 4 k + c), zero-filled here.
int conv_stem_wgrad_tc(const void *in4, const void *grad_out, int dtype, uint32_t K,
                       uint32_t c_out, const int32_t *nbr, uint32_t n_rows, float *dWv,
                       void *workspace, uint64_t workspace_bytes, cudaStream_t stream) {
  MEB_CHECK_ARG(conv_stem_wgrad_tc_supported(dtype, K, c_out), "stem wgrad: K=%u c_out=%u", K, c_out);
  const uint32_t V = stem_virtual(K);
  if (n_rows == 0) {
    MEB_CUDA(cudaMemsetAsync(dWv, 0, (size_t)V * c_out * sizeof(float), stream));
    return MEB200_OK;
  }
  if (!aligned(8, in4) || !aligned(16, grad_out)) {
    set_error("stem wgrad: operands must be 8 / 16-byte aligned");
    return MEB200_ERR_UNSUPPORTED;
  }
  WgParams p{};
  p.in = in4; p.gout = grad_out; p.nbr = nbr; p.dW = dWv;
  p.c_in = V; p.c_out = c_out; p.K = 1; p.n_in = kNoLimit; p.n_out = n_rows; p.n_chunks = 1;
  p.stem_K = K;
  return run_wgrad(dtype, p, 1, cdiv(n_rows, tc::kWgRows), workspace, workspace_bytes, stream);
}

// ---- wgrad ---------------------------------------------------------------------------------------
bool conv_wgrad_tc_supported(int dtype, uint32_t c_in, uint32_t c_out) {
  if (dtype != MEB200_BF16 && dtype != MEB200_F16) return false;
  return c_in % 8 == 0 && c_in >= 16 && c_out % 16 == 0 && c_out >= 16 && c_out <= tc::kMaxCols;
}

int conv_wgrad_tc(const void *in, const void *grad_out, int dtype, uint32_t c_in, uint32_t K,
                  uint32_t c_out, const int32_t *out_nbr, uint32_t n_out, float *grad_weight,
                  void *workspace, uint64_t workspace_bytes, cudaStream_t stream) {
  if (!conv_wgrad_tc_supported(dtype, c_in, c_out) || !aligned(16, in, grad_out)) {
    set_error("wgrad tc: shape or alignment outside the tensor-core path (c_in=%u c_out=%u)",
              c_in, c_out);
    return MEB200_ERR_UNSUPPORTED;
  }
  if (n_out == 0 || K == 0) {
    MEB_CUDA(cudaMemsetAsync(grad_weight, 0, (size_t)K * c_in * c_out * sizeof(float), stream));
    return MEB200_OK;
  }
  WgParams p{};
  p.in = in; p.gout = grad_out; p.nbr = out_nbr; p.dW = grad_weight;
  p.c_in = c_in; p.c_out = c_out; p.K = K; p.n_in = kNoLimit; p.n_out = n_out; p.n_chunks = 1;
  return run_wgrad(dtype, p, K, cdiv(n_out, tc::kWgRows), workspace, workspace_bytes, stream);
}

// K <= 1023 keeps the segment count (chunks * K) of the chunked lists in range
bool conv_wgrad_uses_pairs(int dtype, uint32_t c_in, uint32_t c_out, uint32_t K) {
  return K >= 1 && K <= 1023 && conv_wgrad_tc_supported(dtype, c_in, c_out);
}

int conv_wgrad_pairs(const void *in, const void *grad_out, int dtype, uint32_t c_in, uint32_t K,
                     uint32_t c_out, const int32_t *pairs_in, const int32_t *pairs_out,
                     const int32_t *seg_start, uint32_t n_chunks, uint32_t n_out,
                     float *grad_weight, void *workspace, uint64_t workspace_bytes,
                     cudaStream_t stream) {
  if (!conv_wgrad_uses_pairs(dtype, c_in, c_out, K) || !aligned(16, in, grad_out)) {
    set_error("wgrad pairs: shape or alignment outside the tensor-core path (c_in=%u c_out=%u K=%u)",
              c_in, c_out, K);
    return MEB200_ERR_UNSUPPORTED;
  }
  if (n_out == 0) {
    MEB_CUDA(cudaMemsetAsync(grad_weight, 0, (size_t)K * c_in * c_out * sizeof(float), stream));
    return MEB200_OK;
  }
  WgParams p{};
  p.in = in; p.gout = grad_out; p.pin = pairs_in; p.pout = pairs_out; p.seg = seg_start;
  p.dW = grad_weight; p.c_in = c_in; p.c_out = c_out; p.K = K; p.n_in = kNoLimit;
  p.n_out = n_out; p.n_chunks = n_chunks;
  // splits from the estimate "a third of the K * n_out table entries are pairs"
  return run_wgrad(dtype, p, K, n_out / (3 * tc::kWgRows) + 1, workspace, workspace_bytes, stream);
}

}  // namespace meb200
