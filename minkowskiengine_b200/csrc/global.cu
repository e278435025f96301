// Per-cloud (origin) grouping, segmented reduction and broadcast: the two primitives behind global
// pooling, broadcast operations and instance normalisation.
//
// Reference semantics: the origin map of coordinate_map_cpu.hpp:492-513 / 724-783, global pooling
// in src/global_pooling_cpu.cpp (NonzeroAvgPooling / MaxPooling kernels over the origin map) and
// broadcast in src/broadcast_kernel.hpp.  The reference reduces with per-batch index_select or a
// serial loop; here the rows of every cloud are grouped once per coordinate map (a stable counting
// sort, no atomics that decide an order), and every reduction walks fixed row tiles of a segment:
// each tile stores fp32 partials, a second pass adds the tiles in tile order.  Results are
// therefore bit-identical run to run, whatever order the CTAs run in.
#include <float.h>

#include <atomic>

#include <cub/block/block_scan.cuh>

#include "common.cuh"

namespace meb200 {

constexpr uint32_t kSegTile = MEB200_SEGMENT_TILE_ROWS;   // rows per reduction tile
constexpr uint32_t kGroupTile = 1024;                      // rows per counting-sort tile (one warp)
constexpr uint32_t kMaxSegments = 12288;                   // B ints of shared memory per warp tile

// ---- grouping ------------------------------------------------------------------------------
// row_seg[i] = origin row of (batch(i), 0, ..., 0), or -1 when the origin map lacks that batch
template <int NC>
__global__ void __launch_bounds__(256)
k_origin_lookup(const int32_t *__restrict__ coords, uint32_t n, const int32_t *__restrict__ origin,
                const uint32_t *__restrict__ table, uint32_t mask, int32_t *__restrict__ row_seg) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int32_t key[NC];
#pragma unroll
  for (int j = 0; j < NC; ++j) key[j] = 0;
  key[0] = __ldg(coords + (size_t)i * NC);
  row_seg[i] = table_find<NC>(origin, table, mask, key);
}

// The same for the float points of a tensor field, batch index lroundf(field[i, 0]).  A batch
// value that is not finite or outside int32 gets -1 and sets *bad (when bad != NULL).
template <int NC>
__global__ void __launch_bounds__(256)
k_field_origin_lookup(const float *__restrict__ field, uint32_t n,
                      const int32_t *__restrict__ origin, const uint32_t *__restrict__ table,
                      uint32_t mask, int32_t *__restrict__ row_seg, uint32_t *__restrict__ bad) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  bool ok = true;
  int32_t key[NC];
#pragma unroll
  for (int j = 0; j < NC; ++j) key[j] = 0;
  key[0] = quantize_batch(__ldg(field + (size_t)i * NC), &ok);
  row_seg[i] = ok ? table_find<NC>(origin, table, mask, key) : -1;
  if (!ok && bad != nullptr) atomicOr(bad, 1u);   // a flag, not a sum: any order, same word
}

// Origin candidates of a field: row i = (lroundf(field[i, 0]), 0, ..., 0), *bad as above.
template <int NC>
__global__ void __launch_bounds__(256)
k_field_origin_coords(const float *__restrict__ field, uint32_t n, int32_t *__restrict__ out,
                      uint32_t *__restrict__ bad) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  bool ok = true;
  int32_t c[NC];
#pragma unroll
  for (int j = 1; j < NC; ++j) c[j] = 0;
  c[0] = quantize_batch(__ldg(field + (size_t)i * NC), &ok);
  store_coord<NC>(out, i, c);
  if (!ok) atomicOr(bad, 1u);
}

// counts[s * n_tiles + t] = rows of segment s in group tile t (shared-memory integer counters:
// the totals do not depend on the order of the increments)
__global__ void __launch_bounds__(32)
k_group_count(const int32_t *__restrict__ row_seg, uint32_t n, uint32_t B, uint32_t n_tiles,
              int32_t *__restrict__ counts) {
  extern __shared__ int32_t cnt[];
  for (uint32_t s = threadIdx.x; s < B; s += 32) cnt[s] = 0;
  __syncwarp();
  uint32_t begin = blockIdx.x * kGroupTile, end = min(n, begin + kGroupTile);
  for (uint32_t i = begin + threadIdx.x; i < end; i += 32) {
    int32_t s = row_seg[i];
    if (s >= 0) atomicAdd(cnt + s, 1);
  }
  __syncwarp();
  for (uint32_t s = threadIdx.x; s < B; s += 32) counts[(size_t)s * n_tiles + blockIdx.x] = cnt[s];
}

// exclusive scan of counts (segment-major) in place; seg_start[s] = first position of segment s,
// tile_start[s] = first reduction tile of segment s (kSegTile rows per tile)
__global__ void __launch_bounds__(1024)
k_group_scan(int32_t *__restrict__ counts, uint32_t total, uint32_t B, uint32_t n_tiles,
             int32_t *__restrict__ seg_start, int32_t *__restrict__ tile_start) {
  using Scan = cub::BlockScan<int32_t, 1024>;
  __shared__ typename Scan::TempStorage tmp;
  __shared__ int32_t carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (uint32_t base = 0; base < total; base += 1024) {
    uint32_t i = base + threadIdx.x;
    int32_t v = i < total ? counts[i] : 0, ex, agg;
    Scan(tmp).ExclusiveSum(v, ex, agg);
    int32_t c = carry;
    if (i < total) counts[i] = c + ex;
    __syncthreads();
    if (threadIdx.x == 0) carry = c + agg;
    __syncthreads();
  }
  for (uint32_t s = threadIdx.x; s < B; s += 1024) seg_start[s] = n_tiles ? counts[(size_t)s * n_tiles] : 0;
  if (threadIdx.x == 0) seg_start[B] = carry;
  __syncthreads();
  if (threadIdx.x == 0) {
    int32_t t = 0;
    for (uint32_t s = 0; s < B; ++s) {
      tile_start[s] = t;
      t += (int32_t)((seg_start[s + 1] - seg_start[s] + kSegTile - 1) / kSegTile);
    }
    tile_start[B] = t;
  }
}

// stable scatter: the rows of one group tile, 32 at a time in ascending order; lanes holding the
// same segment are ranked by lane (__match_any_sync), so a segment lists its rows in row order
__global__ void __launch_bounds__(32)
k_group_scatter(const int32_t *__restrict__ row_seg, uint32_t n, uint32_t B, uint32_t n_tiles,
                const int32_t *__restrict__ offsets, int32_t *__restrict__ order) {
  extern __shared__ int32_t base[];
  for (uint32_t s = threadIdx.x; s < B; s += 32) base[s] = offsets[(size_t)s * n_tiles + blockIdx.x];
  __syncwarp();
  uint32_t lane = threadIdx.x, lt = (1u << lane) - 1u;
  uint32_t begin = blockIdx.x * kGroupTile, end = min(n, begin + kGroupTile);
  for (uint32_t r0 = begin; r0 < end; r0 += 32) {
    uint32_t i = r0 + lane;
    int32_t s = i < end ? row_seg[i] : -2;
    uint32_t peers = __match_any_sync(0xFFFFFFFFu, s);
    if (s >= 0) {
      int32_t b = base[s];
      order[b + __popc(peers & lt)] = (int32_t)i;
    }
    __syncwarp();
    if (s >= 0 && (peers & lt) == 0) base[s] += __popc(peers);
    __syncwarp();
  }
}

// ---- feature vectors -------------------------------------------------------------------------
template <typename T, int V> struct VecIO;
template <typename T> struct VecIO<T, 1> {
  static __device__ __forceinline__ void load(const T *p, float (&f)[1]) { f[0] = to_f32<T>(*p); }
  static __device__ __forceinline__ void store(T *p, const float (&f)[1]) { *p = from_f32<T>(f[0]); }
};
template <> struct VecIO<float, 4> {
  static __device__ __forceinline__ void load(const float *p, float (&f)[4]) {
    float4 v = *reinterpret_cast<const float4 *>(p);
    f[0] = v.x; f[1] = v.y; f[2] = v.z; f[3] = v.w;
  }
  static __device__ __forceinline__ void store(float *p, const float (&f)[4]) {
    *reinterpret_cast<float4 *>(p) = make_float4(f[0], f[1], f[2], f[3]);
  }
};
template <> struct VecIO<__nv_bfloat16, 4> {
  static __device__ __forceinline__ void load(const __nv_bfloat16 *p, float (&f)[4]) {
    uint2 v = *reinterpret_cast<const uint2 *>(p);
    float2 a = __bfloat1622float2(*reinterpret_cast<__nv_bfloat162 *>(&v.x));
    float2 b = __bfloat1622float2(*reinterpret_cast<__nv_bfloat162 *>(&v.y));
    f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y;
  }
  static __device__ __forceinline__ void store(__nv_bfloat16 *p, const float (&f)[4]) {
    __nv_bfloat162 a = __floats2bfloat162_rn(f[0], f[1]), b = __floats2bfloat162_rn(f[2], f[3]);
    uint2 v;
    v.x = *reinterpret_cast<uint32_t *>(&a);
    v.y = *reinterpret_cast<uint32_t *>(&b);
    *reinterpret_cast<uint2 *>(p) = v;
  }
};
template <> struct VecIO<__half, 4> {
  static __device__ __forceinline__ void load(const __half *p, float (&f)[4]) {
    uint2 v = *reinterpret_cast<const uint2 *>(p);
    float2 a = __half22float2(*reinterpret_cast<__half2 *>(&v.x));
    float2 b = __half22float2(*reinterpret_cast<__half2 *>(&v.y));
    f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y;
  }
  static __device__ __forceinline__ void store(__half *p, const float (&f)[4]) {
    __half2 a = __floats2half2_rn(f[0], f[1]), b = __floats2half2_rn(f[2], f[3]);
    uint2 v;
    v.x = *reinterpret_cast<uint32_t *>(&a);
    v.y = *reinterpret_cast<uint32_t *>(&b);
    *reinterpret_cast<uint2 *>(p) = v;
  }
};

// ---- segmented reduction ---------------------------------------------------------------------
// Pass 1: one CTA per (segment, tile of kSegTile rows).  Thread (r, cv) of the CTA owns column
// vector cv (V channels) and rows r, r + RP, r + 2 RP, ... of the tile in ascending order; the RP
// row lanes are then combined in shared memory in lane order and the tile's fp32 partial (and, for
// MAX, the row of the maximum) goes to the workspace.
template <typename T, int V, int MODE, bool PROD>
__global__ void __launch_bounds__(256)
k_seg_reduce_tiles(const T *__restrict__ a, const T *__restrict__ b, uint32_t C,
                   const int32_t *__restrict__ order, const int32_t *__restrict__ seg_start,
                   const int32_t *__restrict__ tile_start, uint32_t B, uint32_t tpr,
                   float *__restrict__ part, int32_t *__restrict__ part_row) {
  extern __shared__ float red[];          // [rp][C] sums / maxima, then (MAX) [rp][C] rows
  uint32_t tile = blockIdx.x;
  if (tile >= (uint32_t)__ldg(tile_start + B)) return;
  uint32_t lo = 0, hi = B;                // segment s with tile_start[s] <= tile < tile_start[s+1]
  while (hi - lo > 1) {
    uint32_t mid = (lo + hi) >> 1;
    if ((uint32_t)__ldg(tile_start + mid) <= tile) lo = mid; else hi = mid;
  }
  uint32_t s = lo;
  uint32_t p0 = __ldg(seg_start + s) + (tile - __ldg(tile_start + s)) * kSegTile;
  uint32_t p1 = min(p0 + kSegTile, (uint32_t)__ldg(seg_start + s + 1));
  uint32_t rp = blockDim.x / tpr, r = threadIdx.x / tpr, cv0 = threadIdx.x % tpr;
  uint32_t CV = C / V;
  int32_t *red_row = reinterpret_cast<int32_t *>(red + (size_t)rp * C);
  for (uint32_t cv = cv0; cv < CV; cv += tpr) {
    float acc[V];
    int32_t row[V];
#pragma unroll
    for (int j = 0; j < V; ++j) { acc[j] = MODE == MEB200_SEG_MAX ? -FLT_MAX : 0.f; row[j] = -1; }
    uint32_t p = p0 + r;
#pragma unroll 4
    for (; p < p1; p += rp) {
      int32_t i = __ldg(order + p);
      float x[V];
      VecIO<T, V>::load(a + (size_t)i * C + cv * V, x);
      if (PROD) {
        float y[V];
        VecIO<T, V>::load(b + (size_t)i * C + cv * V, y);
#pragma unroll
        for (int j = 0; j < V; ++j) x[j] *= y[j];
      }
#pragma unroll
      for (int j = 0; j < V; ++j) {
        if (MODE == MEB200_SEG_MAX) {
          if (row[j] < 0 || x[j] > acc[j]) { acc[j] = x[j]; row[j] = i; }   // rows ascend: first max wins
        } else {
          acc[j] += x[j];
        }
      }
    }
#pragma unroll
    for (int j = 0; j < V; ++j) {
      red[(size_t)r * C + cv * V + j] = acc[j];
      if (MODE == MEB200_SEG_MAX) red_row[(size_t)r * C + cv * V + j] = row[j];
    }
  }
  __syncthreads();
  for (uint32_t c = threadIdx.x; c < C; c += blockDim.x) {
    float v = red[c];
    int32_t w = MODE == MEB200_SEG_MAX ? red_row[c] : 0;
    for (uint32_t q = 1; q < rp; ++q) {
      float u = red[(size_t)q * C + c];
      if (MODE == MEB200_SEG_MAX) {
        int32_t uw = red_row[(size_t)q * C + c];
        if (uw >= 0 && (w < 0 || u > v || (u == v && uw < w))) { v = u; w = uw; }
      } else {
        v += u;
      }
    }
    part[(size_t)tile * C + c] = v;
    if (MODE == MEB200_SEG_MAX) part_row[(size_t)tile * C + c] = w;
  }
}

// Pass 2: out[s, c] from the tiles of segment s, added (or compared) in tile order.
template <int MODE>
__global__ void __launch_bounds__(256)
k_seg_reduce_finish(const float *__restrict__ part, const int32_t *__restrict__ part_row,
                    const int32_t *__restrict__ seg_start, const int32_t *__restrict__ tile_start,
                    uint32_t B, uint32_t C, float *__restrict__ out, void *__restrict__ aux) {
  uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (uint64_t)B * C) return;
  uint32_t s = (uint32_t)(t / C), c = (uint32_t)(t % C);
  int32_t t0 = __ldg(tile_start + s), t1 = __ldg(tile_start + s + 1);
  int32_t cnt = __ldg(seg_start + s + 1) - __ldg(seg_start + s);
  if (MODE == MEB200_SEG_MAX) {
    float v = 0.f;
    int32_t w = -1;
    for (int32_t k = t0; k < t1; ++k) {
      float u = part[(size_t)k * C + c];
      int32_t uw = part_row[(size_t)k * C + c];
      if (w < 0 || u > v) { v = u; w = uw; }          // tiles ascend in row order: ties keep the first
    }
    out[t] = v;
    if (aux) reinterpret_cast<int32_t *>(aux)[t] = w < 0 ? -1 : w * (int32_t)C + (int32_t)c;
  } else {
    float v = 0.f;
    for (int32_t k = t0; k < t1; ++k) v += part[(size_t)k * C + c];
    if (MODE == MEB200_SEG_AVG && cnt > 0) v /= (float)cnt;
    out[t] = v;
    if (aux && c == 0) reinterpret_cast<float *>(aux)[s] = (float)cnt;
  }
}

// ---- broadcast -------------------------------------------------------------------------------
// out[i, c] = x[i, c] op g[row_seg[i], c]; MAXGRAD: g[b, c] where argmax[b, c] == i*C + c, else 0.
template <typename T, typename TO, int V, int OP>
__global__ void __launch_bounds__(256)
k_broadcast(const T *__restrict__ x, const float *__restrict__ g, const int32_t *__restrict__ argmax,
            const int32_t *__restrict__ row_seg, uint32_t n, uint32_t C, TO *__restrict__ out) {
  uint32_t CV = C / V;
  uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (uint64_t)n * CV) return;
  uint32_t i = (uint32_t)(t / CV), c = (uint32_t)(t % CV) * V;
  int32_t s = __ldg(row_seg + i);
  float y[V];
  if (s < 0) {                         // row outside every segment (not produced by a valid grouping)
#pragma unroll
    for (int j = 0; j < V; ++j) y[j] = 0.f;
  } else {
    float gv[V];
    if constexpr (V == 4) {
      float4 q = __ldg(reinterpret_cast<const float4 *>(g + (size_t)s * C + c));
      gv[0] = q.x; gv[1] = q.y; gv[2] = q.z; gv[3] = q.w;
    } else {
#pragma unroll
      for (int j = 0; j < V; ++j) gv[j] = __ldg(g + (size_t)s * C + c + j);
    }
    if (OP == MEB200_BCAST_COPY) {
#pragma unroll
      for (int j = 0; j < V; ++j) y[j] = gv[j];
    } else if (OP == MEB200_BCAST_MAXGRAD) {
#pragma unroll
      for (int j = 0; j < V; ++j) {
        int32_t flat = (int32_t)(i * C + c + j);
        y[j] = __ldg(argmax + (size_t)s * C + c + j) == flat ? gv[j] : 0.f;
      }
    } else {
      float xv[V];
      VecIO<T, V>::load(x + (size_t)i * C + c, xv);
#pragma unroll
      for (int j = 0; j < V; ++j) y[j] = OP == MEB200_BCAST_ADD ? xv[j] + gv[j] : xv[j] * gv[j];
    }
  }
  VecIO<TO, V>::store(out + (size_t)i * C + c, y);
}

// out[i, c] = x[i, c] * g[s, c] + z[i, c] * h[s, c] + k[s, c], s = row_seg[i] (z / h and k optional)
template <typename T, int V>
__global__ void __launch_bounds__(256)
k_broadcast_fma(const T *__restrict__ x, const T *__restrict__ z, const float *__restrict__ g,
                const float *__restrict__ h, const float *__restrict__ k,
                const int32_t *__restrict__ row_seg, uint32_t n, uint32_t C, T *__restrict__ out) {
  uint32_t CV = C / V;
  uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (uint64_t)n * CV) return;
  uint32_t i = (uint32_t)(t / CV), c = (uint32_t)(t % CV) * V;
  int32_t s = __ldg(row_seg + i);
  float y[V], xv[V], zv[V];
  VecIO<T, V>::load(x + (size_t)i * C + c, xv);
  if (z) VecIO<T, V>::load(z + (size_t)i * C + c, zv);
  size_t o = (size_t)(s < 0 ? 0 : s) * C + c;
#pragma unroll
  for (int j = 0; j < V; ++j) {
    float v = xv[j] * __ldg(g + o + j);
    if (z) v = fmaf(zv[j], __ldg(h + o + j), v);
    if (k) v += __ldg(k + o + j);
    y[j] = s < 0 ? 0.f : v;
  }
  VecIO<T, V>::store(out + (size_t)i * C + c, y);
}

// ---- host dispatch ---------------------------------------------------------------------------
static uint32_t group_tiles(uint32_t n) { return (n + kGroupTile - 1) / kGroupTile; }

static int check_group_args(uint32_t n, const int32_t *origin_coords, const uint32_t *origin_table,
                            uint32_t origin_capacity, uint32_t B, const int32_t *row_seg,
                            const int32_t *order, const int32_t *seg_start,
                            const int32_t *tile_start, const void *scratch) {
  MEB_CHECK_ARG(B >= 1 && B <= kMaxSegments, "B = %u clouds (supported: 1..%u)", B, kMaxSegments);
  MEB_CHECK_ARG(origin_coords && origin_table && seg_start && tile_start, "null buffer");
  MEB_CHECK_ARG(n == 0 || (row_seg && order && scratch), "null buffer");
  MEB_CHECK_ARG(origin_capacity && (origin_capacity & (origin_capacity - 1)) == 0,
                "capacity %u is not a power of two", origin_capacity);
  return MEB200_OK;
}

// The counting sort of the n rows by their row_seg (written by a lookup): counts per group tile,
// the scan, the stable scatter.  Shared by the grouping of a coordinate map and of a field.
static int group_rows(const int32_t *row_seg, uint32_t n, uint32_t B, int32_t *order,
                      int32_t *seg_start, int32_t *tile_start, void *scratch, cudaStream_t s) {
  uint32_t nt = group_tiles(n);
  int32_t *counts = (int32_t *)scratch;
  if (n > 0) {
    k_group_count<<<nt, 32, B * sizeof(int32_t), s>>>(row_seg, n, B, nt, counts);
    MEB_LAUNCH_OK();
  }
  k_group_scan<<<1, 1024, 0, s>>>(counts, nt * B, B, nt, seg_start, tile_start);
  MEB_LAUNCH_OK();
  if (n > 0) {
    k_group_scatter<<<nt, 32, B * sizeof(int32_t), s>>>(row_seg, n, B, nt, counts, order);
    MEB_LAUNCH_OK();
  }
  return MEB200_OK;
}

// The combine of k_seg_reduce_tiles holds [rp][C] values (and, for MAX, rows): at most 8 * 8192
// bytes, for MAX over C > 6144 channels on one row lane.  A launch above the default 48 KB needs
// the kernel opted in on the current device, which is done once per instantiation and device.
constexpr size_t kSegMaxSmem = 8 * 8192;

template <typename T, int V, int MODE, bool PROD>
static int seg_reduce_smem_opt_in(size_t smem) {
  if (smem <= 48 * 1024) return MEB200_OK;
  static std::atomic<uint32_t> done{0};   // bit d: device d opted in
  int dev = 0;
  MEB_CUDA(cudaGetDevice(&dev));
  uint32_t bit = dev < 32 ? 1u << dev : 0u;
  if (done.load() & bit) return MEB200_OK;
  MEB_CUDA(cudaFuncSetAttribute(k_seg_reduce_tiles<T, V, MODE, PROD>,
                                cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSegMaxSmem));
  done.fetch_or(bit);
  return MEB200_OK;
}

template <typename T, int V, int MODE>
static int seg_reduce_launch(const void *a, const void *b, uint32_t C, const int32_t *order,
                             const int32_t *seg_start, const int32_t *tile_start, uint32_t B,
                             uint32_t max_tiles, float *part, int32_t *part_row, cudaStream_t st) {
  uint32_t CV = C / V, tpr = 1;
  while (tpr * 2 <= CV && tpr * 2 <= 256) tpr *= 2;     // threads per row: a power of two <= 256
  uint32_t rp = 256 / tpr;
  size_t smem = (size_t)rp * C * (MODE == MEB200_SEG_MAX ? 8 : 4);
  int rc;
  if (b) {
    if ((rc = seg_reduce_smem_opt_in<T, V, MODE, true>(smem)) != MEB200_OK) return rc;
    k_seg_reduce_tiles<T, V, MODE, true><<<max_tiles, 256, smem, st>>>(
        (const T *)a, (const T *)b, C, order, seg_start, tile_start, B, tpr, part, part_row);
  } else {
    if ((rc = seg_reduce_smem_opt_in<T, V, MODE, false>(smem)) != MEB200_OK) return rc;
    k_seg_reduce_tiles<T, V, MODE, false><<<max_tiles, 256, smem, st>>>(
        (const T *)a, nullptr, C, order, seg_start, tile_start, B, tpr, part, part_row);
  }
  return MEB200_OK;
}

template <typename T>
static int seg_reduce_t(const void *a, const void *b, uint32_t C, const int32_t *order,
                        const int32_t *seg_start, const int32_t *tile_start, uint32_t B,
                        uint32_t max_tiles, int mode, float *part, int32_t *part_row,
                        cudaStream_t st) {
  bool v4 = C % 4 == 0 && aligned(4 * sizeof(T), a, b);
  int rc = MEB200_OK;
#define MEB_SEG(MODE)                                                                           \
  if (v4) rc = seg_reduce_launch<T, 4, MODE>(a, b, C, order, seg_start, tile_start, B, max_tiles, \
                                             part, part_row, st);                               \
  else rc = seg_reduce_launch<T, 1, MODE>(a, b, C, order, seg_start, tile_start, B, max_tiles,  \
                                          part, part_row, st);
  switch (mode) {
    case MEB200_SEG_SUM: MEB_SEG(MEB200_SEG_SUM); break;
    case MEB200_SEG_AVG: MEB_SEG(MEB200_SEG_AVG); break;
    case MEB200_SEG_MAX: MEB_SEG(MEB200_SEG_MAX); break;
  }
#undef MEB_SEG
  if (rc != MEB200_OK) return rc;
  MEB_LAUNCH_OK();
  return MEB200_OK;
}

// The broadcasts take 4 channels per thread in every dtype (8-byte accesses in bf16 / fp16).
template <typename T, typename TO, int V>
static int bcast_launch(const void *x, const float *g, const int32_t *argmax,
                        const int32_t *row_seg, uint32_t n, uint32_t C, int op, void *out,
                        cudaStream_t st) {
  unsigned blocks = cdiv((uint64_t)n * (C / V), 256);
  switch (op) {
    case MEB200_BCAST_ADD:
      k_broadcast<T, TO, V, MEB200_BCAST_ADD><<<blocks, 256, 0, st>>>((const T *)x, g, argmax, row_seg, n, C, (TO *)out);
      break;
    case MEB200_BCAST_MUL:
      k_broadcast<T, TO, V, MEB200_BCAST_MUL><<<blocks, 256, 0, st>>>((const T *)x, g, argmax, row_seg, n, C, (TO *)out);
      break;
    case MEB200_BCAST_COPY:
      k_broadcast<T, TO, V, MEB200_BCAST_COPY><<<blocks, 256, 0, st>>>((const T *)x, g, argmax, row_seg, n, C, (TO *)out);
      break;
    default:
      k_broadcast<T, TO, V, MEB200_BCAST_MAXGRAD><<<blocks, 256, 0, st>>>((const T *)x, g, argmax, row_seg, n, C, (TO *)out);
  }
  MEB_LAUNCH_OK();
  return MEB200_OK;
}

template <typename T, int V>
static int fma_launch(const void *x, const void *z, const float *g, const float *h, const float *k,
                      const int32_t *row_seg, uint32_t n, uint32_t C, void *out, cudaStream_t st) {
  k_broadcast_fma<T, V><<<cdiv((uint64_t)n * (C / V), 256), 256, 0, st>>>(
      (const T *)x, (const T *)z, g, h, k, row_seg, n, C, (T *)out);
  MEB_LAUNCH_OK();
  return MEB200_OK;
}

}  // namespace meb200

using namespace meb200;

extern "C" {

int meb200_broadcast_fma(const void *x, const void *z, int dtype, const float *g, const float *h,
                         const float *k, const int32_t *row_seg, uint32_t n, uint32_t C, void *out,
                         void *stream) {
  if (n == 0 || C == 0) return MEB200_OK;
  MEB_CHECK_ARG(x && g && row_seg && out, "null buffer");
  MEB_CHECK_ARG((z == nullptr) == (h == nullptr), "z and h go together");
  cudaStream_t s = (cudaStream_t)stream;
  MEB_DISPATCH_DTYPE(dtype,
    if (C % 4 == 0 && aligned(4 * sizeof(T), x, z, out))
      return fma_launch<T, 4>(x, z, g, h, k, row_seg, n, C, out, s);
    return fma_launch<T, 1>(x, z, g, h, k, row_seg, n, C, out, s));
}

uint64_t meb200_origin_group_scratch_bytes(uint32_t n, uint32_t B) {
  return ((uint64_t)group_tiles(n) * B + 1) * sizeof(int32_t);
}

int meb200_origin_group(const int32_t *coords, uint32_t n, uint32_t ncols,
                        const int32_t *origin_coords, const uint32_t *origin_table,
                        uint32_t origin_capacity, uint32_t B, int32_t *row_seg, int32_t *order,
                        int32_t *seg_start, int32_t *tile_start, void *scratch, void *stream) {
  int rc = check_group_args(n, origin_coords, origin_table, origin_capacity, B, row_seg, order,
                            seg_start, tile_start, scratch);
  if (rc != MEB200_OK) return rc;
  MEB_CHECK_ARG(n == 0 || coords, "null buffer");
  cudaStream_t s = (cudaStream_t)stream;
  if (n > 0) {
    MEB_DISPATCH_NCOLS(ncols, (k_origin_lookup<NC><<<cdiv(n, 256), 256, 0, s>>>(
                                  coords, n, origin_coords, origin_table, origin_capacity - 1,
                                  row_seg)));
    MEB_LAUNCH_OK();
  }
  return group_rows(row_seg, n, B, order, seg_start, tile_start, scratch, s);
}

int meb200_field_origin_group(const float *field, uint32_t n, uint32_t ncols,
                              const int32_t *origin_coords, const uint32_t *origin_table,
                              uint32_t origin_capacity, uint32_t B, int32_t *row_seg,
                              int32_t *order, int32_t *seg_start, int32_t *tile_start,
                              uint32_t *d_bad, void *scratch, void *stream) {
  int rc = check_group_args(n, origin_coords, origin_table, origin_capacity, B, row_seg, order,
                            seg_start, tile_start, scratch);
  if (rc != MEB200_OK) return rc;
  MEB_CHECK_ARG(n == 0 || field, "null buffer");
  cudaStream_t s = (cudaStream_t)stream;
  if (d_bad != nullptr) MEB_CUDA(cudaMemsetAsync(d_bad, 0, 4, s));
  if (n > 0) {
    MEB_DISPATCH_NCOLS(ncols, (k_field_origin_lookup<NC><<<cdiv(n, 256), 256, 0, s>>>(
                                  field, n, origin_coords, origin_table, origin_capacity - 1,
                                  row_seg, d_bad)));
    MEB_LAUNCH_OK();
  }
  return group_rows(row_seg, n, B, order, seg_start, tile_start, scratch, s);
}

int meb200_field_origin_insert(const float *field, uint32_t n, uint32_t ncols, int32_t *ocoords,
                               uint32_t *table, uint32_t capacity, int32_t *unique_coords,
                               int64_t *unique_index, int64_t *inverse_map, void *scratch,
                               uint32_t *h_num_unique, void *stream) {
  MEB_CHECK_ARG(h_num_unique != nullptr, "h_num_unique");
  cudaStream_t s = (cudaStream_t)stream;
  if (n > 0) {
    MEB_CHECK_ARG(field && ocoords && scratch, "null buffer");
    uint32_t *bad = insert_flag_word(scratch, n);
    MEB_CUDA(cudaMemsetAsync(bad, 0, 4, s));
    MEB_DISPATCH_NCOLS(ncols, (k_field_origin_coords<NC><<<cdiv(n, 256), 256, 0, s>>>(
                                  field, n, ocoords, bad)));
    MEB_LAUNCH_OK();
  }
  uint32_t h[2] = {0, 0};
  int rc = insert_and_map(ocoords, nullptr, n, ncols, table, capacity, unique_coords,
                          unique_index, inverse_map, scratch, h, n > 0 ? 2 : 1, s);
  if (rc != MEB200_OK) return rc;
  *h_num_unique = h[0];
  if (h[1] != 0) {
    set_error("a field batch coordinate is not finite, or lies outside int32");
    return MEB200_ERR_DOMAIN;
  }
  return MEB200_OK;
}

uint32_t meb200_segment_max_tiles(uint32_t n, uint32_t B) {
  return (n + kSegTile - 1) / kSegTile + B;
}

uint64_t meb200_segment_workspace_bytes(uint32_t n, uint32_t C, uint32_t B) {
  // fp32 partials + int32 rows (MAX) per (tile, channel)
  return (uint64_t)meb200_segment_max_tiles(n, B) * C * 8;
}

int meb200_segment_reduce(const void *a, const void *b, int dtype, uint32_t n, uint32_t C,
                          const int32_t *order, const int32_t *seg_start,
                          const int32_t *tile_start, uint32_t B, int mode, float *out, void *aux,
                          void *workspace, uint64_t workspace_bytes, void *stream) {
  if (B == 0 || C == 0) return MEB200_OK;
  MEB_CHECK_ARG(mode == MEB200_SEG_SUM || mode == MEB200_SEG_AVG || mode == MEB200_SEG_MAX,
                "mode %d is not a segment reduction", mode);
  MEB_CHECK_ARG(mode != MEB200_SEG_MAX || b == nullptr, "MAX takes no second operand");
  MEB_CHECK_ARG(out && seg_start && tile_start, "null buffer");
  MEB_CHECK_ARG(n == 0 || (a && order), "null buffer");
  MEB_CHECK_ARG(C <= 8192, "C = %u channels (supported: <= 8192)", C);
  MEB_CHECK_ARG(mode != MEB200_SEG_MAX || (uint64_t)n * C < 0x7FFFFFFFull,
                "max_index is int32: n*C too large");
  uint32_t max_tiles = meb200_segment_max_tiles(n, B);
  MEB_CHECK_ARG(workspace && workspace_bytes >= meb200_segment_workspace_bytes(n, C, B) &&
                    ((uintptr_t)workspace & 15) == 0,
                "workspace: %llu bytes needed, 16-byte aligned",
                (unsigned long long)meb200_segment_workspace_bytes(n, C, B));
  cudaStream_t s = (cudaStream_t)stream;
  float *part = (float *)workspace;
  int32_t *part_row = (int32_t *)(part + (size_t)max_tiles * C);
  int rc = MEB200_OK;
  if (n > 0) {
    MEB_DISPATCH_DTYPE(dtype, rc = seg_reduce_t<T>(a, b, C, order, seg_start, tile_start, B,
                                                   max_tiles, mode, part, part_row, s));
    if (rc != MEB200_OK) return rc;
  }
  unsigned blocks = cdiv((uint64_t)B * C, 256);
  switch (mode) {
    case MEB200_SEG_SUM: k_seg_reduce_finish<MEB200_SEG_SUM><<<blocks, 256, 0, s>>>(part, part_row, seg_start, tile_start, B, C, out, aux); break;
    case MEB200_SEG_AVG: k_seg_reduce_finish<MEB200_SEG_AVG><<<blocks, 256, 0, s>>>(part, part_row, seg_start, tile_start, B, C, out, aux); break;
    default: k_seg_reduce_finish<MEB200_SEG_MAX><<<blocks, 256, 0, s>>>(part, part_row, seg_start, tile_start, B, C, out, aux); break;
  }
  MEB_LAUNCH_OK();
  return MEB200_OK;
}

int meb200_broadcast(const void *x, int dtype, const float *g, const int32_t *argmax,
                     const int32_t *row_seg, uint32_t n, uint32_t C, int op, void *out,
                     int out_dtype, void *stream) {
  if (n == 0 || C == 0) return MEB200_OK;
  MEB_CHECK_ARG(op == MEB200_BCAST_ADD || op == MEB200_BCAST_MUL || op == MEB200_BCAST_COPY ||
                    op == MEB200_BCAST_MAXGRAD, "op %d is not a broadcast operation", op);
  MEB_CHECK_ARG(g && row_seg && out, "null buffer");
  MEB_CHECK_ARG(x || op == MEB200_BCAST_COPY || op == MEB200_BCAST_MAXGRAD, "null x");
  MEB_CHECK_ARG(argmax || op != MEB200_BCAST_MAXGRAD, "null argmax");
  MEB_CHECK_ARG(out_dtype == dtype || out_dtype == MEB200_F32,
                "out_dtype %d must be the feature dtype %d or F32", out_dtype, dtype);
  cudaStream_t s = (cudaStream_t)stream;
  MEB_DISPATCH_DTYPE_OUT(dtype, out_dtype,
    if (C % 4 == 0 && aligned(4 * sizeof(T), x) && aligned(16, g) && aligned(4 * sizeof(TO), out))
      return bcast_launch<T, TO, 4>(x, g, argmax, row_seg, n, C, op, out, s);
    return bcast_launch<T, TO, 1>(x, g, argmax, row_seg, n, C, op, out, s));
}

}
