// Hopper (sm_90a) sparse convolution on the tensor cores: warpgroup MMA (wgmma.mma_async) with
// both operands gathered into shared memory by cp.async, fp32 accumulators in registers.
//
//   forward / dgrad : out[r, :] = sum_k A[nbr[k][r], :] @ B_k              (k_conv_wg)
//   wgrad           : dW[k]     += In[rows_in, :]^T @ dOut[rows_out, :]     (k_wgrad_wg)
//
// Operands are bf16 / fp16, or fp32 words multiplied in TF32 (MEB200_TF32: k_conv_wg<float, ..>
// for forward / dgrad, k_wgrad_tf32 for the weight gradient, whose MN-major operands tf32 wgmma
// cannot read).  The forward also runs on e4m3 bytes (meb200_conv_forward_fp8:
// k_conv_wg<__nv_fp8_e4m3, ..>, 32 channels per k-step, always with its epilogue), and the fp8
// dgrad on e5m2 gradients against e4m3 weights (meb200_conv_dgrad_fp8: k_conv_wg<__nv_fp8_e5m2,
// ..>, the same staging with the e5m2 x e4m3 MMA).  k_conv_wg_q is
// the forward with the epilogue that also stores an e4m3 shadow of its output (the _q entries).
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
#include <stddef.h>
#include <stdlib.h>
#include <string.h>
#include <type_traits>

#include <cuda_fp8.h>

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
constexpr bool kIsTf32 = std::is_same<T, float>::value;   // fp32 storage, tf32 MMAs
// fp8 operands: e4m3 both sides (the forward), or e5m2 A against e4m3 B (the dgrad: T names A)
template <typename T>
constexpr bool kIsE5M2 = std::is_same<T, __nv_fp8_e5m2>::value;
template <typename T>
constexpr bool kIsFp8 = std::is_same<T, __nv_fp8_e4m3>::value || kIsE5M2<T>;

template <typename T>
__device__ __forceinline__ uint32_t pack2(float a, float b);
template <typename T>
__device__ __forceinline__ float2 unpack2(uint32_t u);
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

template <>
__device__ __forceinline__ float2 unpack2<__nv_bfloat16>(uint32_t u) {
  return __bfloat1622float2(*reinterpret_cast<__nv_bfloat162 *>(&u));
}
template <>
__device__ __forceinline__ float2 unpack2<__half>(uint32_t u) {
  return __half22float2(*reinterpret_cast<__half2 *>(&u));
}

__device__ __forceinline__ uint8_t *align1k(uint8_t *p) {
  return reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(p) + 1023) & ~uintptr_t(1023));
}

// =====================================================================================
// forward / dgrad
// =====================================================================================
struct FwdParams {
  const void *A;          // [n_a, c_red] gathered operand (stem: [n_a, 4])
  const void *B;          // [K][*][c_red] operand B (reduction contiguous), at this launch's row 0
  const int32_t *nbr;     // [K, n_rows]
  void *out;              // [n_rows, out_ld], at this launch's column 0
  uint64_t b_k_stride;    // elements between the offsets of B
  uint32_t c_red, K, n_rows;
  uint32_t c_cols;        // columns of one CTA: column slice blockIdx.y starts at blockIdx.y * c_cols
  uint32_t n_a;           // rows of A (gather indices >= n_a read as zero rows)
  uint32_t out_ld, bk, out_f32;
  union {
    uint32_t stem_K;      // > 0: network stem, virtual channel 4 k + c = A[nbr[k][r]][c], k < stem_K
    // e4m3 kernels (which have no stem mode): device fp32, the activation scale.  It shares the
    // 8-byte slot of stem_K and its padding, so the parameter block keeps its layout.
    const float *a_scale;
  };
  // tile order (meb200_kernel_map, K <= 32), or both NULL: nbr is then the table in slot order,
  // tile t runs the offsets of tile_mask[t] and writes slot s to row slot_row[s]
  const int32_t *slot_row;
  const uint32_t *tile_mask;
  // epilogue of the EPI kernels (meb200_conv_epilogue): scale / shift at this launch's column 0,
  // res (may be NULL) laid out as out
  const float *scale, *shift;
  const void *res;
  uint32_t relu;
};
static_assert(sizeof(FwdParams) == 128 && offsetof(FwdParams, slot_row) == 80, "FwdParams layout");

// NT wgmma instructions of N = NI columns each cover the c_cols = NI * NT columns of the slice.
// grid = (128-row tiles, column slices).  EPI: apply the epilogue of p before the conversion (a
// template parameter, so that the plain forward and the dgrad compile as if it did not exist).
// TO: the 16-bit output type (out_f32: fp32), T itself except for fp8 operands, whose kernels
// multiply the accumulator by *p.a_scale first.  e4m3 kernels always run the epilogue; the e5m2
// dgrad kernels (EPI = false) only multiply column col by p.scale[col], the weight scale.
//
// Q (the _q kernels): also store the shadow, the e4m3 copy of the output at the next layer's static
// scale: q[orow, col] = e4m3(round_TO(v) * q_scale[1]), v the final epilogue value, so that the
// bytes are those meb200_quantize_e4m3_static makes of the stored output.
template <typename T, int NI, int NT, bool EPI, typename TO, bool Q>
__device__ __forceinline__ void conv_wg(const FwdParams &p, uint8_t *q, const float *q_scale) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t s0 = smem_u32(align1k(smem_raw));
  const uint32_t tid = threadIdx.x, wg = tid >> 7, warp = tid >> 5, lane = tid & 31;
  const uint32_t row0 = blockIdx.x * tc::kFwdRows;
  // a stage holds `width` bytes of every row: ch 16-byte chunks of kEpc elements, bk channels
  constexpr uint32_t kEpc = 16 / sizeof(T);
  const uint32_t bk = p.bk, width = bk * sizeof(T), ch = width / 16;
  const uint32_t lch = width == 128 ? 3 : (width == 64 ? 2 : 1);
  const uint32_t a_bytes = tc::kFwdRows * width, stage_bytes = a_bytes + p.c_cols * width;
  const bool ordered = p.tile_mask != nullptr;
  const uint32_t tmask = ordered ? __ldg(p.tile_mask + blockIdx.x) : 0u;
  const uint32_t nch = p.c_red / bk, n_st = (ordered ? __popc(tmask) : p.K) * nch;
  const T *A = reinterpret_cast<const T *>(p.A);
  const T *B = reinterpret_cast<const T *>(p.B) + (size_t)blockIdx.y * p.c_cols * p.c_red;
  const uint32_t col0 = blockIdx.y * p.c_cols;
  const uint32_t ar = tid >> 1, arow = row0 + ar;     // two threads per tile row of A
  const bool row_ok = arow < p.n_rows;

  // producer cursor: offset ld_k (the set bits of tmask in ascending order when ordered), chunk ld_c
  uint32_t ld_rem = tmask, ld_k = ordered ? __ffs(tmask) - 1 : 0, ld_c = 0;
  auto load = [&](uint32_t s) {
    const uint32_t k = ld_k, c0 = ld_c * bk;
    if (++ld_c == nch) {
      ld_c = 0;
      if (ordered) { ld_rem &= ld_rem - 1; ld_k = __ffs(ld_rem) - 1; } else ++ld_k;
    }
    const uint32_t base = s0 + (s % kStages) * stage_bytes;
    if (kIsTf32<T> || kIsFp8<T> || p.stem_K == 0) {
      const int32_t src = row_ok ? __ldg(p.nbr + (size_t)k * p.n_rows + arow) : -1;
      const bool ok = src >= 0 && (uint32_t)src < p.n_a;
      const T *rp = A + (size_t)(ok ? src : 0) * p.c_red + c0;
      for (uint32_t j = tid & 1u; j < ch; j += 2)
        cp_async16(base + cm_off(ar, j, ch), rp + kEpc * j, ok ? 16u : 0u);
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
      cp_async16(base + a_bytes + cm_off(n, j, ch), Bk + (size_t)n * p.c_red + kEpc * j, 16u);
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
    const uint32_t a0 = s0 + (s % kStages) * stage_bytes + wg * 64 * width;
    const uint32_t b0 = s0 + (s % kStages) * stage_bytes + a_bytes;
    wgmma_fence();
    for (uint32_t kk = 0; kk < width / 32; ++kk) {     // one k-step = 32 bytes = 2 core matrices
      const uint64_t da = wgmma_desc(a0 + kk * 256, 128, sbo);
#pragma unroll
      for (int i = 0; i < NT; ++i) {
        const uint64_t db = wgmma_desc(b0 + i * NI * width + kk * 256, 128, sbo);
        if constexpr (kIsTf32<T>) wgmma_tf32<NI, 0, 0>(acc[i], da, db);
        else if constexpr (kIsE5M2<T>) wgmma_e5m2e4m3<NI>(acc[i], da, db);
        else if constexpr (kIsFp8<T>) wgmma_e4m3<NI>(acc[i], da, db);
        else wgmma<NI, kIsBf16<T>, 0, 0>(acc[i], da, db);
      }
    }
    wgmma_commit();
    wgmma_wait<1>();
  }
  wgmma_wait<0>();
  float a_s = 1.f;
  if constexpr (kIsFp8<T>) a_s = __ldg(p.a_scale);
  float q_inv = 0.f;
  if constexpr (Q) q_inv = __ldg(q_scale + 1);

  const uint32_t g = lane >> 2, t = lane & 3;
  const uint32_t rbase = row0 + wg * 64 + (warp & 3) * 16 + g;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const uint32_t r = rbase + 8 * h;
    if (r >= p.n_rows) continue;
    const uint32_t orow = p.slot_row != nullptr ? (uint32_t)__ldg(p.slot_row + r) : r;
#pragma unroll
    for (int i = 0; i < NT; ++i)
#pragma unroll
      for (int j = 0; j < NI / 8; ++j) {
        const uint32_t col = col0 + i * NI + 8 * j + 2 * t;
        float v0 = acc[i][4 * j + 2 * h], v1 = acc[i][4 * j + 2 * h + 1];
        if constexpr (kIsFp8<T>) {
          v0 *= a_s;
          v1 *= a_s;
        }
        if constexpr (kIsE5M2<T>) {         // the fp8 dgrad: times the weight scale of column col
          const float2 sc = *reinterpret_cast<const float2 *>(p.scale + col);
          v0 *= sc.x;
          v1 *= sc.y;
        }
        if constexpr (EPI) {
          // plain loads, ordered after the previous pair's store: the compiler then cannot hoist
          // the loads of the whole tile ahead of the stores (which spills the widest tiles)
          const float2 sc = *reinterpret_cast<const float2 *>(p.scale + col);
          const float2 sh = *reinterpret_cast<const float2 *>(p.shift + col);
          v0 = fmaf(v0, sc.x, sh.x);
          v1 = fmaf(v1, sc.y, sh.y);
          if (p.res != nullptr) {
            const size_t e2 = ((size_t)orow * p.out_ld + col) / 2;     // the pair's index
            float2 rv;
            if (kIsTf32<T> || p.out_f32) rv = reinterpret_cast<const float2 *>(p.res)[e2];
            else if constexpr (!kIsTf32<T>)
              rv = unpack2<TO>(reinterpret_cast<const uint32_t *>(p.res)[e2]);
            v0 += rv.x;
            v1 += rv.y;
          }
          if (p.relu) {
            v0 = fmaxf(v0, 0.f);
            v1 = fmaxf(v1, 0.f);
          }
        }
        if (kIsTf32<T> || p.out_f32) {
          *reinterpret_cast<float2 *>(reinterpret_cast<float *>(p.out) + (size_t)orow * p.out_ld + col) =
              make_float2(v0, v1);
        } else if constexpr (!kIsTf32<T>) {
          const uint32_t packed = pack2<TO>(v0, v1);
          *reinterpret_cast<uint32_t *>(reinterpret_cast<TO *>(p.out) + (size_t)orow * p.out_ld + col) =
              packed;
          if constexpr (Q) {                  // the stored values, not the fp32 ones
            const float2 r = unpack2<TO>(packed);
            v0 = r.x;
            v1 = r.y;
          }
        }
        if constexpr (Q)
          *reinterpret_cast<uint16_t *>(q + (size_t)orow * p.out_ld + col) =
              e4m3x2_satfinite(__fmul_rn(v0, q_inv), __fmul_rn(v1, q_inv));
      }
  }
}

template <typename T, int NI, int NT, bool EPI, typename TO = T>
__global__ void __launch_bounds__(kThreads, 1) k_conv_wg(const FwdParams p) {
  conv_wg<T, NI, NT, EPI, TO, false>(p, nullptr, nullptr);
}

// The forward with its shadow (bf16 / fp16 / e4m3 operands, always with the epilogue).  The shadow
// rides in a parameter block of its own, so FwdParams and the kernels above keep their layout.
struct FwdQParams {
  FwdParams f;
  uint8_t *q;             // [n_rows, out_ld] e4m3, at this launch's column 0
  const float *q_scale;   // device fp32 [2]: (scale, inv) of the consumer
};

template <typename T, int NI, int NT, typename TO>
__global__ void __launch_bounds__(kThreads, 1) k_conv_wg_q(const FwdQParams p) {
  conv_wg<T, NI, NT, true, TO, true>(p.f, p.q, p.q_scale);
}

// =====================================================================================
// wgrad:  dW[k][ci][co] += sum over (input row i, output row o) pairs of offset k of
//         In[i][ci] * dOut[o][co]
// GEMM view: D[M = ci][N = co] over the reduction axis "pair"; a stage = 64 pairs.  One unit =
// (offset k, 128 input channels, a share of the pairs), run by one CTA, or in pair mode by one CTA
// per column slice when k has over twice the mean pairs (k_wgrad_wg).  With one share per
// offset it stores its sums into dW; otherwise share s stores into partial[s] and
// launch_split_sum adds the shares in order, so the result does not depend on the order in which
// CTAs finish, nor on the column slicing.  The pairs come from
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
  uint32_t col_slices;     // pair mode, k_wgrad_wg: NT = heavy offsets in column slices (below)
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

// One (offset k, channel tile, share) unit of k_wgrad_wg over the NI * NT output columns col0..:
// NT wgmma instructions of N = NI columns each.  An output element's sum is the same sequence of
// m64nNIk16 instructions on the same operands whichever columns the CTA covers, so a unit cut into
// column slices gives the same bits as the whole unit.
template <typename T, int NI, int NT>
__device__ __forceinline__ void wgrad_unit(const WgParams &p, uint32_t k, uint32_t col0) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t s0 = smem_u32(align1k(smem_raw));
  const uint32_t tid = threadIdx.x, wg = tid >> 7, warp = tid >> 5, lane = tid & 31;
  const uint32_t ci0 = blockIdx.y * tc::kWgChannels;
  constexpr uint32_t kChA = tc::kWgChannels / 8;                    // 16 chunks per A row
  constexpr uint32_t a_bytes = tc::kWgRows * tc::kWgChannels * 2;
  constexpr uint32_t chB = NI * NT / 8, stage_bytes = a_bytes + tc::kWgRows * NI * NT * 2;
  const uint32_t n_chunks = p.pin != nullptr ? p.n_chunks : 1u;
  const T *In = reinterpret_cast<const T *>(p.in);
  const T *G = reinterpret_cast<const T *>(p.gout);

  uint32_t n_st = 0;
  for (uint32_t c = 0; c < n_chunks; ++c) {
    uint32_t lo, hi;
    wg_range(p, k, c, lo, hi);
    n_st += (hi - lo + tc::kWgRows - 1) / tc::kWgRows;
  }
  // Thread tid copies tile row ar = tid / 4 of both operands, chunks (tid & 3) + 4m.  Its two
  // index words per stage are loaded a stage before the copies that use them (fetch), so that no
  // copy waits on a global load: the loads of stage s + 3 are in flight over stage s's MMAs and
  // the next barrier.
  const uint32_t ar = tid >> 2;
  // index cursor: the next stage to fetch is [pos, min(pos + 64, end)) of chunk wc
  uint32_t wc = 0, pos = 0, end = 0;
  auto open = [&]() {
    for (; wc < n_chunks; ++wc) {
      wg_range(p, k, wc, pos, end);
      if (pos < end) return;
    }
  };
  open();
  // row ar of the next stage: src = input row (unused in stem mode), o = dOut row; -1 past the end
  struct Words { int32_t src, o; };
  auto fetch = [&]() {
    Words w{-1, -1};
    const uint32_t r = pos + ar;
    if (r < end) {
      if (p.pin != nullptr) {
        w.src = __ldg(p.pin + r);
        w.o = __ldg(p.pout + r);
      } else {
        if (p.stem_K == 0) w.src = __ldg(p.nbr + (size_t)k * p.n_out + r);
        w.o = (int32_t)r;
      }
    }
    pos += tc::kWgRows;
    if (pos >= end) { ++wc; open(); }
    return w;
  };
  // chunk j = j0 + 4m of row ar lies at cm_off(ar, j0, chunks) + 512 m
  const uint32_t j0 = tid & 3u;
  auto copy = [&](uint32_t s, Words w) {
    const uint32_t base = s0 + (s % kStages) * stage_bytes;
    if (p.stem_K == 0) {
      const bool ok = w.src >= 0 && (uint32_t)w.src < p.n_in;
      const T *rp = In + (size_t)(ok ? w.src : 0) * p.c_in + ci0 + 8 * j0;
      const uint32_t dst = base + cm_off(ar, j0, kChA);
#pragma unroll
      for (uint32_t m = 0; m < 4; ++m) {
        const bool okj = ok && ci0 + 8 * (j0 + 4 * m) < p.c_in;
        cp_async16(dst + 512 * m, okj ? rp + 32 * m : In, okj ? 16u : 0u);
      }
    } else {
      // chunk j = virtual channels ci0 + 8j..: offsets kk = (ci0 + 8j) / 4 + {0, 1}, 8 bytes each.
      // The table is walked by pointer steps (one offset, then seven), which keeps the compiler
      // from holding the eight 64-bit offsets kk * n_out in registers across the loop.
      const uint32_t kk0 = ci0 / 4 + 2 * j0;
      const int32_t *tp = p.nbr + (size_t)kk0 * p.n_out + (w.o >= 0 ? w.o : 0);
      const uint32_t dst = base + cm_off(ar, j0, kChA);
#pragma unroll
      for (uint32_t m = 0; m < 4; ++m) {
#pragma unroll
        for (uint32_t h = 0; h < 2; ++h) {
          const int32_t src = (w.o >= 0 && kk0 + 8 * m + h < p.stem_K) ? __ldg(tp) : -1;
          const bool ok = src >= 0 && (uint32_t)src < p.n_in;
          cp_async8(dst + 512 * m + 8 * h, In + (size_t)(ok ? src : 0) * 4, ok ? 8u : 0u);
          tp += (size_t)(h == 0 ? 1 : 7) * p.n_out;
        }
      }
    }
    const bool ok = w.o >= 0 && (uint32_t)w.o < p.n_out;
    const T *gp = G + (size_t)(ok ? w.o : 0) * p.c_out + col0 + 8 * j0;
    const uint32_t dst = base + a_bytes + cm_off(ar, j0, chB);
#pragma unroll
    for (uint32_t m = 0; m < (chB + 3) / 4; ++m)
      if (j0 + 4 * m < chB) cp_async16(dst + 512 * m, gp + 32 * m, ok ? 16u : 0u);
  };

  float acc[NT][NI / 2];
#pragma unroll
  for (int i = 0; i < NT; ++i)
#pragma unroll
    for (int q = 0; q < NI / 2; ++q) acc[i][q] = 0.f;

  Words first[kStages - 2];
#pragma unroll
  for (uint32_t s = 0; s < kStages - 2; ++s)
    if (s < n_st) first[s] = fetch();
#pragma unroll
  for (uint32_t s = 0; s < kStages - 2; ++s) {
    if (s < n_st) copy(s, first[s]);
    cp_async_commit();
  }
  Words next{-1, -1};                   // stage s + 2's words at the top of iteration s
  if (kStages - 2 < n_st) next = fetch();
  // (a warpgroup whose 64 channels lie past c_in multiplies the zero-filled half of the tile:
  // branching around wgmma would serialise the instructions of the whole kernel)
  for (uint32_t s = 0; s < n_st; ++s) {
    cp_async_wait<kStages - 3>();
    fence_proxy_async();
    __syncthreads();
    if (s + kStages - 2 < n_st) {       // into the slot of stage s - 2
      copy(s + kStages - 2, next);
      if (s + kStages - 1 < n_st) next = fetch();
    }
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
        *reinterpret_cast<float2 *>(dWk + (size_t)ci * p.c_out + col0 + i * NI + 8 * j + 2 * t) =
            make_float2(acc[i][4 * j + 2 * h], acc[i][4 * j + 2 * h + 1]);
      }
  }
}

// 64-pair stages of offset k, over all row chunks of the pair lists
__device__ __forceinline__ uint32_t wg_offset_stages(const WgParams &p, uint32_t k) {
  uint32_t s = 0;
  for (uint32_t c = 0; c < p.n_chunks; ++c)
    s += ((uint32_t)(__ldg(p.seg + (size_t)c * p.K + k + 1) - __ldg(p.seg + (size_t)c * p.K + k)) +
          tc::kWgRows - 1) / tc::kWgRows;
  return s;
}

// Pair mode with col_slices = NT: blockIdx.z = k * NT + j.  An offset with more than twice the
// mean stages per offset (the centre offset of a stride-1 map has 3.2x) runs each of its units as
// NT CTAs of NI columns (slice j); the others as one CTA of all columns (j = 0, the rest exit).
// The sums are those of the unsliced grid, bit for bit; only the longest CTAs get shorter.  (A
// slice gathers the whole input tile for a part of the columns, and the extra CTAs can spill into
// a second wave: below twice the mean that costs more than it saves.)
// (tiles of up to 128 columns fit two CTAs per SM in shared memory: keep the registers for two)
template <typename T, int NI, int NT>
__global__ void __launch_bounds__(kThreads, NI * NT <= 128 ? 2 : 1) k_wgrad_wg(const WgParams p) {
  if constexpr (NT > 1) {
    if (p.col_slices == NT) {
      const uint32_t k = blockIdx.z / NT, j = blockIdx.z % NT;
      // total stages: every warp adds the segments lane-strided, the same sum in every warp
      const uint32_t lane = threadIdx.x & 31, n_seg = p.n_chunks * p.K;
      uint32_t t = 0;
      for (uint32_t i = lane; i < n_seg; i += 32)
        t += ((uint32_t)(__ldg(p.seg + i + 1) - __ldg(p.seg + i)) + tc::kWgRows - 1) / tc::kWgRows;
#pragma unroll
      for (int d = 16; d > 0; d >>= 1) t += __shfl_xor_sync(0xffffffffu, t, d);
      if ((uint64_t)wg_offset_stages(p, k) * p.K > 2ull * t) {
        wgrad_unit<T, NI, 1>(p, k, j * NI);
      } else if (j == 0) {
        wgrad_unit<T, NI, NT>(p, k, 0);
      }
      return;
    }
  }
  wgrad_unit<T, NI, NT>(p, blockIdx.z, 0);
}

// TF32 wgrad.  wgmma reads tf32 operands K-major only, and both wgrad operands are gathered
// MN-major (a pair's channels are contiguous), so this kernel multiplies with the warp-level
// mma.sync.m16n8k8 instead, whose fragments are plain 32-bit shared-memory loads of any layout.
// Same CTAs (offset, 128 input channels, share), shares (wg_range) and stores as k_wgrad_wg; a
// share is walked in stages of kWgRowsTf32 pairs.  Stage = In [32 pairs][128 + pad channels] and
// dOut [32 pairs][c_out + pad], row-major.  Warp w owns channels 32 (w & 3).. (two 16-row M tiles)
// and output columns (w >> 2) * c_out / 2.. (NB 8-column N tiles): NB = c_out / 16.
template <int NB>
__global__ void __launch_bounds__(kThreads, 1) k_wgrad_tf32(const WgParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  float *sm = reinterpret_cast<float *>(align1k(smem_raw));
  constexpr uint32_t R = tc::kWgRowsTf32, SA = tc::kWgChannels + tc::kWgPadTf32;
  const uint32_t tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const uint32_t k = blockIdx.z, ci0 = blockIdx.y * tc::kWgChannels;
  const uint32_t SB = p.c_out + tc::kWgPadTf32;
  constexpr uint32_t chB = 4 * NB;      // 16-byte chunks of a dOut row (c_out = 16 NB)
  const uint32_t stage_floats = R * (SA + SB);
  const uint32_t n_chunks = p.pin != nullptr ? p.n_chunks : 1u;
  const float *In = reinterpret_cast<const float *>(p.in);
  const float *G = reinterpret_cast<const float *>(p.gout);

  uint32_t n_st = 0;
  for (uint32_t c = 0; c < n_chunks; ++c) {
    uint32_t lo, hi;
    wg_range(p, k, c, lo, hi);
    n_st += (hi - lo + R - 1) / R;
  }
  // as in wgrad_unit: thread tid copies row ar = tid / 8 of both operands, chunks (tid & 7) + 8m
  // of 4 channels, from index words fetched a stage ahead
  const uint32_t ar = tid >> 3;
  uint32_t wc = 0, pos = 0, end = 0;
  auto open = [&]() {
    for (; wc < n_chunks; ++wc) {
      wg_range(p, k, wc, pos, end);
      if (pos < end) return;
    }
  };
  open();
  struct Words { int32_t src, o; };
  auto fetch = [&]() {
    Words w{-1, -1};
    const uint32_t r = pos + ar;
    if (r < end) {
      if (p.pin != nullptr) {
        w.src = __ldg(p.pin + r);
        w.o = __ldg(p.pout + r);
      } else {
        w.src = __ldg(p.nbr + (size_t)k * p.n_out + r);
        w.o = (int32_t)r;
      }
    }
    pos += R;
    if (pos >= end) { ++wc; open(); }
    return w;
  };
  auto copy = [&](uint32_t s, Words w) {
    const uint32_t base = smem_u32(sm + (s % kStages) * stage_floats);
    const bool ok = w.src >= 0 && (uint32_t)w.src < p.n_in;
    const float *rp = In + (size_t)(ok ? w.src : 0) * p.c_in + ci0;
#pragma unroll
    for (uint32_t m = 0; m < 4; ++m) {
      const uint32_t j = (tid & 7u) + 8 * m;
      const bool okj = ok && ci0 + 4 * j < p.c_in;
      cp_async16(base + (ar * SA + 4 * j) * 4, okj ? rp + 4 * j : In, okj ? 16u : 0u);
    }
    const bool okr = w.o >= 0 && (uint32_t)w.o < p.n_out;
    const float *gp = G + (size_t)(okr ? w.o : 0) * p.c_out;
#pragma unroll
    for (uint32_t m = 0; m < (chB + 7) / 8; ++m) {
      const uint32_t j = (tid & 7u) + 8 * m;
      if (j < chB) cp_async16(base + (R * SA + ar * SB + 4 * j) * 4, gp + 4 * j, okr ? 16u : 0u);
    }
  };

  float acc[2][NB][4];
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int ni = 0; ni < NB; ++ni)
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[mi][ni][q] = 0.f;

  Words first[kStages - 2];
#pragma unroll
  for (uint32_t s = 0; s < kStages - 2; ++s)
    if (s < n_st) first[s] = fetch();
#pragma unroll
  for (uint32_t s = 0; s < kStages - 2; ++s) {
    if (s < n_st) copy(s, first[s]);
    cp_async_commit();
  }
  Words next{-1, -1};                   // stage s + 2's words at the top of iteration s
  if (kStages - 2 < n_st) next = fetch();
  const uint32_t g = lane >> 2, t = lane & 3;
  const uint32_t m0 = (warp & 3) * 32, n0 = (warp >> 2) * NB * 8;
  for (uint32_t s = 0; s < n_st; ++s) {
    cp_async_wait<kStages - 3>();
    __syncthreads();                    // stage s landed everywhere; stage s - 2 is no longer read
    if (s + kStages - 2 < n_st) {
      copy(s + kStages - 2, next);
      if (s + kStages - 1 < n_st) next = fetch();
    }
    cp_async_commit();
    const uint32_t *sA = reinterpret_cast<const uint32_t *>(sm + (s % kStages) * stage_floats);
    const uint32_t *sB = sA + R * SA;
    // (the widest tiles keep 128 accumulators: unrolled k-steps would spill them)
#pragma unroll(NB > 12 ? 1 : 4)
    for (uint32_t kk = 0; kk < R; kk += 8) {
      // A[m = channel][k = pair] = In stage [pair][channel]; B[k = pair][n = column] = dOut stage
      uint32_t a[2][4];
#pragma unroll
      for (int mi = 0; mi < 2; ++mi) {
        const uint32_t *pa = sA + (kk + t) * SA + m0 + 16 * mi + g;
        a[mi][0] = pa[0]; a[mi][1] = pa[8]; a[mi][2] = pa[4 * SA]; a[mi][3] = pa[4 * SA + 8];
      }
#pragma unroll
      for (int ni = 0; ni < NB; ++ni) {   // B fragments one N tile at a time (register budget)
        const uint32_t *pb = sB + (kk + t) * SB + n0 + 8 * ni + g;
        const uint32_t b[2] = {pb[0], pb[4 * SB]};
        mma_tf32_16x8x8(acc[0][ni], a[0], b);
        mma_tf32_16x8x8(acc[1][ni], a[1], b);
      }
    }
  }

  const size_t dw_elems = (size_t)p.K * p.c_in * p.c_out;   // every element written by one CTA
  float *dWk = (p.n_splits > 1 ? p.partial + blockIdx.x * dw_elems : p.dW) + (size_t)k * p.c_in * p.c_out;
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const uint32_t ci = ci0 + m0 + 16 * mi + g + 8 * h;
      if (ci >= p.c_in) continue;
#pragma unroll
      for (int ni = 0; ni < NB; ++ni)
        *reinterpret_cast<float2 *>(dWk + (size_t)ci * p.c_out + n0 + 8 * ni + 2 * t) =
            make_float2(acc[mi][ni][2 * h], acc[mi][ni][2 * h + 1]);
    }
}


// ---- weight packing ----------------------------------------------------------------------------
// Per-optimizer-step weight packing: fp32 master W[k][ci][co] -> the operand type in the two
// operand-B layouts of the wgmma kernels, in one pass:
//   Wc [k][ci][co]  dgrad operand B            Wt [k][co][ci]  forward operand B
// bf16 / fp16: rounded to nearest even; TF32 (T = float): rounded to the nearest tf32 value, ties
// away from zero (cvt.rna), and kept in fp32 words, so that the forward and the dgrad multiply the
// same matrix.  One CTA packs the 32 x 32 tile (k, ci0.., co0..).
template <typename T>
__device__ __forceinline__ T to_operand(float v) {
  if constexpr (kIsTf32<T>) return tf32_rna(v); else return from_f32<T>(v);
}

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
      Wc[base + (size_t)(ci0 + i) * c_out + co0 + tx] = to_operand<T>(v);
    }
  __syncthreads();
  for (uint32_t i = ty; i < 32; i += 8)
    if (co0 + i < c_out && ci0 + tx < c_in)
      Wt[base + (size_t)(co0 + i) * c_in + ci0 + tx] = to_operand<T>(tile[tx][i]);
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
  else if (dtype == MEB200_TF32)
    k_pack_w_batched<float><<<total_tiles, 256, 0, stream>>>(jobs_dev, n_jobs);
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
  else if (dtype == MEB200_TF32)
    k_pack_w<float><<<grid, 256, 0, stream>>>(W, (float *)w_cast, (float *)w_t, c_in, c_out);
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

template <typename T, int NI, int NT, bool EPI, typename TO>
static int launch_fwd(const FwdParams &p, uint32_t slices, cudaStream_t stream) {
  auto kern = k_conv_wg<T, NI, NT, EPI, TO>;
  MEB_BIG_SMEM(kern);
  const dim3 grid(cdiv(p.n_rows, tc::kFwdRows), slices);
  kern<<<grid, kThreads, tc::fwd_ring_bytes(p.bk * sizeof(T), p.c_cols), stream>>>(p);
  count_tc_launch();
  MEB_LAUNCH_OK();
  return MEB200_OK;
}
template <typename T, bool EPI, typename TO = T>
static int dispatch_fwd(const FwdParams &p, uint32_t slices, cudaStream_t stream) {
#define MEB_L(NI, NT) launch_fwd<T, NI, NT, EPI, TO>(p, slices, stream)
  MEB_COLS_DISPATCH(p.c_cols, MEB_L)
#undef MEB_L
  set_error("conv tc: %u output columns per launch", p.c_cols);
  return MEB200_ERR_UNSUPPORTED;
}
template <typename T, int NI, int NT, typename TO>
static int launch_fwd_q(const FwdQParams &p, uint32_t slices, cudaStream_t stream) {
  auto kern = k_conv_wg_q<T, NI, NT, TO>;
  MEB_BIG_SMEM(kern);
  const dim3 grid(cdiv(p.f.n_rows, tc::kFwdRows), slices);
  kern<<<grid, kThreads, tc::fwd_ring_bytes(p.f.bk * sizeof(T), p.f.c_cols), stream>>>(p);
  count_tc_launch();
  MEB_LAUNCH_OK();
  return MEB200_OK;
}
template <typename T, typename TO = T>
static int dispatch_fwd_q(const FwdQParams &p, uint32_t slices, cudaStream_t stream) {
#define MEB_L(NI, NT) launch_fwd_q<T, NI, NT, TO>(p, slices, stream)
  MEB_COLS_DISPATCH(p.f.c_cols, MEB_L)
#undef MEB_L
  set_error("conv tc: %u output columns per launch", p.f.c_cols);
  return MEB200_ERR_UNSUPPORTED;
}
// p.c_cols = all the launch's columns (<= 256): the launch runs them in the chooser's slices.
// shadow (q, q_scale) given: the _q kernels (16-bit or e4m3 operands, with the epilogue).
static int run_fwd(int dtype, FwdParams p, cudaStream_t stream, int out_dtype = MEB200_F32,
                   const Shadow *shadow = nullptr) {
  const uint32_t cols = p.c_cols;
  p.c_cols = tc::fwd_col_slice(p.n_rows, cols, (uint32_t)num_sms());
  const uint32_t slices = cols / p.c_cols;
  if (shadow != nullptr) {
    const FwdQParams qp{p, shadow->q, shadow->q_scale};
    if (dtype == kOperandE4M3)
      return out_dtype == MEB200_F16 ? dispatch_fwd_q<__nv_fp8_e4m3, __half>(qp, slices, stream)
                                     : dispatch_fwd_q<__nv_fp8_e4m3, __nv_bfloat16>(qp, slices, stream);
    return dtype == MEB200_BF16 ? dispatch_fwd_q<__nv_bfloat16>(qp, slices, stream)
                                : dispatch_fwd_q<__half>(qp, slices, stream);
  }
  if (dtype == kOperandE5M2E4M3) {    // the fp8 dgrad: column scales, no epilogue, no shadow
    return out_dtype == MEB200_F16 ? dispatch_fwd<__nv_fp8_e5m2, false, __half>(p, slices, stream)
                                   : dispatch_fwd<__nv_fp8_e5m2, false, __nv_bfloat16>(p, slices, stream);
  }
  if (dtype == kOperandE4M3) {        // always with the epilogue; fp32 output through out_f32
    return out_dtype == MEB200_F16 ? dispatch_fwd<__nv_fp8_e4m3, true, __half>(p, slices, stream)
                                   : dispatch_fwd<__nv_fp8_e4m3, true, __nv_bfloat16>(p, slices, stream);
  }
  if (p.scale != nullptr) {
    if (dtype == MEB200_TF32) return dispatch_fwd<float, true>(p, slices, stream);
    return dtype == MEB200_BF16 ? dispatch_fwd<__nv_bfloat16, true>(p, slices, stream)
                                : dispatch_fwd<__half, true>(p, slices, stream);
  }
  if (dtype == MEB200_TF32) return dispatch_fwd<float, false>(p, slices, stream);
  return dtype == MEB200_BF16 ? dispatch_fwd<__nv_bfloat16, false>(p, slices, stream)
                              : dispatch_fwd<__half, false>(p, slices, stream);
}

// the epilogue's pointers at output column n0 (out_esz: bytes of an output element)
static void set_epilogue(FwdParams &p, const meb200_conv_epilogue *epi, uint32_t n0, size_t out_esz) {
  if (epi == nullptr) return;
  p.scale = epi->scale + n0;
  p.shift = epi->shift != nullptr ? epi->shift + n0 : nullptr;     // (the fp8 dgrad has none)
  p.res = epi->residual != nullptr ? reinterpret_cast<const uint8_t *>(epi->residual) + n0 * out_esz
                                   : nullptr;
  p.relu = epi->relu != 0;
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
template <int NB>
static int launch_wgrad_tf32(const WgParams &p, dim3 grid, cudaStream_t stream) {
  auto kern = k_wgrad_tf32<NB>;
  MEB_BIG_SMEM(kern);
  kern<<<grid, kThreads, tc::wgrad_tf32_smem_bytes(p.c_out), stream>>>(p);
  count_tc_launch();
  MEB_LAUNCH_OK();
  return MEB200_OK;
}
static int dispatch_wgrad_tf32(const WgParams &p, dim3 grid, cudaStream_t stream) {
  switch (p.c_out / 16) {
#define MEB_L(NB) case NB: return launch_wgrad_tf32<NB>(p, grid, stream);
    MEB_L(1) MEB_L(2) MEB_L(3) MEB_L(4) MEB_L(5) MEB_L(6) MEB_L(7) MEB_L(8)
    MEB_L(9) MEB_L(10) MEB_L(11) MEB_L(12) MEB_L(13) MEB_L(14) MEB_L(15) MEB_L(16)
#undef MEB_L
    default: break;
  }
  set_error("wgrad tc: %u output channels", p.c_out);
  return MEB200_ERR_UNSUPPORTED;
}
// wgmma instructions (NT of MEB_COLS_DISPATCH) per row of a k_wgrad_wg tile of c_out columns
static uint32_t wgrad_col_instructions(uint32_t c_out) {
#define MEB_NT(NI, NT) NT
  MEB_COLS_DISPATCH(c_out, MEB_NT)
#undef MEB_NT
  return 1;
}
static uint32_t wgrad_planned_splits(uint32_t c_in, uint32_t K, uint32_t est_stages) {
  return tc::wgrad_splits(est_stages, K, cdiv(c_in, tc::kWgChannels), (uint32_t)num_sms());
}

uint64_t conv_wgrad_workspace_bytes(uint32_t c_in, uint32_t c_out, uint32_t K, uint32_t n_out) {
  const uint32_t splits = wgrad_planned_splits(c_in, K, cdiv(n_out, tc::kWgRows));
  return splits > 1 ? (uint64_t)splits * K * c_in * c_out * sizeof(float) : 0;
}

// grid = (row splits, 128-channel tiles of c_in, offsets x column slices).  The splits are what
// the workspace holds of the planned ones (one split: no workspace, the CTAs store into dW
// directly); column slices only change which CTA computes which columns (k_wgrad_wg).
static int run_wgrad(int dtype, WgParams p, uint32_t K_grid, uint32_t est_stages, void *workspace,
                     uint64_t workspace_bytes, cudaStream_t stream) {
  const uint32_t m_tiles = cdiv(p.c_in, tc::kWgChannels);
  const size_t dw_elems = (size_t)K_grid * p.c_in * p.c_out;
  p.n_splits = workspace_splits(wgrad_planned_splits(p.c_in, K_grid, est_stages), workspace,
                                workspace_bytes, dw_elems * sizeof(float));
  p.partial = p.n_splits > 1 ? reinterpret_cast<float *>(workspace) : nullptr;
  // pair mode on the 16-bit kernel: room for the column slices of the heavy offsets
  p.col_slices = p.pin != nullptr && dtype != MEB200_TF32 ? wgrad_col_instructions(p.c_out) : 1;
  const dim3 grid(p.n_splits, m_tiles, K_grid * p.col_slices);
  const int rc = dtype == MEB200_TF32   ? dispatch_wgrad_tf32(p, grid, stream)
                 : dtype == MEB200_BF16 ? dispatch_wgrad<__nv_bfloat16>(p, grid, stream)
                                        : dispatch_wgrad<__half>(p, grid, stream);
  if (rc != MEB200_OK || p.n_splits == 1) return rc;
  return launch_split_sum(p.partial, p.dW, dw_elems, p.n_splits, stream);
}

// ---- forward / dgrad ----------------------------------------------------------------------------
static uint32_t operand_bytes(int dtype) {
  return dtype == MEB200_TF32 ? 4 : (dtype == kOperandE4M3 || dtype == kOperandE5M2E4M3 ? 1 : 2);
}

bool conv_fp8_supported(uint32_t c_in, uint32_t c_out) {
  return c_in >= 32 && c_in % 32 == 0 && c_out % 16 == 0 && c_out >= 16 && c_out <= 1024;
}

bool conv_tc_supported(int dtype, uint32_t c_reduce, uint32_t c_cols) {
  if (dtype != MEB200_BF16 && dtype != MEB200_F16 && dtype != MEB200_TF32) return false;
  if (tc::fwd_stage_bytes(c_reduce, operand_bytes(dtype)) == 0) return false;
  return c_cols % 16 == 0 && c_cols >= 16 && c_cols <= 1024;
}

static_assert(tc::kFwdRows == kOrderTileRows, "a tile order's tiles are the kernel's row tiles");

int conv_forward_tc(const void *A, int dtype, uint32_t n_a, uint32_t c_reduce, const void *B,
                    uint32_t K, uint32_t c_cols, const int32_t *nbr, const int32_t *order,
                    uint32_t n_rows, void *out, int out_dtype, const meb200_conv_epilogue *epi,
                    cudaStream_t stream, const float *a_scale, const Shadow *shadow) {
  if (n_rows == 0) return MEB200_OK;
  const bool fp8 = dtype == kOperandE4M3 || dtype == kOperandE5M2E4M3;
  MEB_CHECK_ARG(fp8 ? conv_fp8_supported(c_reduce, c_cols) && epi != nullptr && a_scale != nullptr
                    : conv_tc_supported(dtype, c_reduce, c_cols),
                "shape not supported by tc path");
  MEB_CHECK_ARG(shadow == nullptr || (epi != nullptr && dtype != MEB200_TF32 &&
                                       dtype != kOperandE5M2E4M3),
                "shadow: 16-bit or e4m3 operands with an epilogue");
  if (!aligned(16, A, B)) {
    set_error("conv tc: operands must be 16-byte aligned");
    return MEB200_ERR_UNSUPPORTED;
  }
  const uint8_t *Wb = reinterpret_cast<const uint8_t *>(B);
  const bool ordered = order != nullptr && K <= kMaxOrderK;
  // one launch per <= 256 output columns
  const size_t out_esz = out_dtype == MEB200_F32 ? 4 : 2, esz = operand_bytes(dtype);
  for (uint32_t n0 = 0; n0 < c_cols; n0 += tc::kMaxCols) {
    FwdParams p{};
    p.A = A; p.B = Wb + (size_t)n0 * c_reduce * esz; p.nbr = ordered ? order : nbr;
    if (ordered) {
      p.slot_row = order + (size_t)K * n_rows;
      p.tile_mask = reinterpret_cast<const uint32_t *>(order + (size_t)(K + 1) * n_rows);
    }
    p.out = reinterpret_cast<uint8_t *>(out) + (size_t)n0 * out_esz;
    p.b_k_stride = (uint64_t)c_cols * c_reduce;
    p.c_red = c_reduce; p.c_cols = c_cols - n0 < tc::kMaxCols ? c_cols - n0 : tc::kMaxCols;
    p.K = K; p.n_rows = n_rows; p.n_a = n_a; p.out_ld = c_cols;
    p.bk = tc::fwd_stage_bytes(c_reduce, esz) / esz; p.out_f32 = out_dtype == MEB200_F32;
    set_epilogue(p, epi, n0, out_esz);
    p.a_scale = a_scale;
    Shadow sh{};
    if (shadow != nullptr) sh = Shadow{shadow->q + n0, shadow->q_scale};
    const int rc = run_fwd(dtype, p, stream, out_dtype, shadow != nullptr ? &sh : nullptr);
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
                         const meb200_conv_epilogue *epi, cudaStream_t stream,
                         const Shadow *shadow) {
  if (n_rows == 0) return MEB200_OK;
  MEB_CHECK_ARG(conv_stem_tc_supported(dtype, K, c_cols), "stem forward: K=%u c_out=%u", K, c_cols);
  MEB_CHECK_ARG(shadow == nullptr || epi != nullptr, "shadow: the epilogue is required");
  if (!aligned(8, A4) || !aligned(16, Wv)) {
    set_error("stem forward: operands must be 8 / 16-byte aligned");
    return MEB200_ERR_UNSUPPORTED;
  }
  FwdParams p{};
  p.A = A4; p.B = Wv; p.nbr = nbr; p.out = out;
  p.c_red = stem_virtual(K); p.c_cols = c_cols; p.K = 1; p.n_rows = n_rows; p.n_a = kNoLimit;
  p.out_ld = c_cols; p.bk = tc::fwd_bk(p.c_red); p.out_f32 = out_dtype == MEB200_F32;
  p.stem_K = K;
  set_epilogue(p, epi, 0, out_dtype == MEB200_F32 ? 4 : 2);
  return run_fwd(dtype, p, stream, out_dtype, shadow);
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
  if (dtype != MEB200_BF16 && dtype != MEB200_F16 && dtype != MEB200_TF32) return false;
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
