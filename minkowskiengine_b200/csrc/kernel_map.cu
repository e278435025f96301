// Kernel-map construction: per-offset in/out row pairs as k-major neighbour tables.
//
// Replaces the reference's direct_kernel_map + remove_if + sort_by_key decomposition
// (src/coordinate_map_gpu.cu:1479-1542,1697-1733, src/kernel_map.cuh:313-405) and the CPU
// loop it mirrors (src/coordinate_map_cpu.hpp:569-670).  One thread per (offset k, row x)
// with x fastest: coordinate loads and table writes are coalesced, each probe is one
// hash-table sector + one coordinate sector.  The result is written directly in the
// layout the convolution kernels consume — x_nbr[k][x] (stationary side) and
// y_nbr[k][y] (its transpose, used by dgrad / transposed convolution) — so there is no
// compaction, no sort and no host synchronisation on this path, and the pair order is
// deterministic.  The reference's per-offset pair lists are recoverable as the
// non-negative entries of row k (that is what CoordinateManager.kernel_map() returns).
#include "common.cuh"

namespace meb200 {

template <int NC>
__global__ void __launch_bounds__(256)
k_kernel_map(const int32_t *__restrict__ x_coords, uint32_t nx,
             const int32_t *__restrict__ y_coords, uint32_t ny,
             const uint32_t *__restrict__ y_table, uint32_t mask,
             const int32_t *__restrict__ offsets, uint32_t K, int32_t *__restrict__ x_nbr,
             int32_t *__restrict__ y_nbr, uint32_t *__restrict__ num_pairs) {
  uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  bool active = t < (uint64_t)nx * K;
  int32_t y = -1;
  if (active) {
    uint32_t k = (uint32_t)(t / nx), x = (uint32_t)(t % nx);
    int32_t key[NC];
    load_coord<NC>(x_coords, x, key);
#pragma unroll
    for (int j = 1; j < NC; ++j) key[j] += __ldg(offsets + (size_t)k * (NC - 1) + (j - 1));
    y = table_find<NC>(y_coords, y_table, mask, key);
    x_nbr[t] = y;
    if (y >= 0 && y_nbr != nullptr) y_nbr[(size_t)k * ny + y] = (int32_t)x;
  }
  if (num_pairs != nullptr) {
    unsigned hits = __popc(__ballot_sync(0xffffffffu, y >= 0));
    if ((threadIdx.x & 31) == 0 && hits) atomicAdd(num_pairs, hits);
  }
}

// ---- compacted per-offset pair lists (the reference's own kernel-map representation:
//      gpu_kernel_map in_maps / out_maps, src/kernel_map.cuh:48-429) --------------------------
// The dense neighbour table is what the output-stationary forward/dgrad kernels want; the wgrad
// kernel reduces over PAIRS, so it wants them compacted: for every offset k the valid
// (other row, table row) pairs in table-row order, each offset's segment padded with (-1, -1)
// to a multiple of `stage` entries.  The table rows are cut into CHUNKS (row ranges) and the
// list is ordered (chunk, offset): a consumer that walks it keeps one chunk's rows of both
// operands L2-resident across the K offsets (offset-major over the whole map re-read both
// feature matrices from HBM once per offset: 2.4 GB against 0.39 GB algorithmic on the largest
// layer).  Three small deterministic passes (count, scan, fill), no atomics, no host
// synchronisation; capacity is the caller's upper bound K*n + K*stage*chunks.
constexpr uint32_t kPairChunk = 2048;   // table entries per block: 256 threads x 8 consecutive

__device__ __forceinline__ void load8(const int32_t *__restrict__ row_k, uint32_t r0, uint32_t n,
                                      int32_t (&v)[8]) {
  if (r0 + 8 <= n && ((reinterpret_cast<uintptr_t>(row_k + r0) & 15) == 0)) {
    const int4 a = __ldg(reinterpret_cast<const int4 *>(row_k + r0));
    const int4 b = __ldg(reinterpret_cast<const int4 *>(row_k + r0) + 1);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
  } else {
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = (r0 + j < n) ? __ldg(row_k + r0 + j) : -1;
  }
}

// exclusive prefix of `c` over the 256 threads of the block; *total = block sum
__device__ __forceinline__ uint32_t block_excl_scan_256(uint32_t c, uint32_t *total) {
  __shared__ uint32_t warp_sums[8];
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t incl = c;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t t = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= (uint32_t)d) incl += t;
  }
  if (lane == 31) warp_sums[warp] = incl;
  __syncthreads();
  uint32_t base = 0, sum = 0;
#pragma unroll
  for (int w = 0; w < 8; ++w) {
    const uint32_t ws = warp_sums[w];
    if ((uint32_t)w < warp) base += ws;
    sum += ws;
  }
  *total = sum;
  return base + incl - c;
}

__global__ void __launch_bounds__(256)
k_pair_count(const int32_t *__restrict__ nbr, uint32_t n, uint32_t nchunks,
             uint32_t *__restrict__ cnt) {
  const uint32_t chunk = blockIdx.x, k = blockIdx.y;
  int32_t v[8];
  load8(nbr + (size_t)k * n, chunk * kPairChunk + threadIdx.x * 8, n, v);
  uint32_t c = 0;
#pragma unroll
  for (int j = 0; j < 8; ++j) c += v[j] >= 0;
  uint32_t total;
  block_excl_scan_256(c, &total);
  if (threadIdx.x == 0) cnt[(size_t)k * nchunks + chunk] = total;
}

// one block: for every (row chunk c, offset k) segment the exclusive scan of its block counts
// (a warp per offset), then the padded segment starts in (c, k) order
// (seg_start[s+1] - seg_start[s] = roundup(count_s, stage), s = c*K + k)
__global__ void __launch_bounds__(1024)
k_pair_scan(uint32_t *__restrict__ cnt /* in: counts, out: exclusive offsets within the segment */,
            uint32_t K, uint32_t nblocks, uint32_t bpc /* blocks per chunk */, uint32_t n_chunks,
            uint32_t stage, int32_t *__restrict__ seg_start, uint32_t *__restrict__ seg_count) {
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (uint32_t k = warp; k < K; k += 32) {
    for (uint32_t c = 0; c < n_chunks; ++c) {
      const uint32_t b0 = c * bpc, b1 = min(b0 + bpc, nblocks);
      uint32_t running = 0;
      for (uint32_t base = b0; base < b1; base += 32) {
        const uint32_t i = base + lane;
        const uint32_t v = i < b1 ? cnt[(size_t)k * nblocks + i] : 0u;
        uint32_t incl = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
          const uint32_t t = __shfl_up_sync(0xffffffffu, incl, d);
          if (lane >= (uint32_t)d) incl += t;
        }
        if (i < b1) cnt[(size_t)k * nblocks + i] = running + incl - v;
        running += __shfl_sync(0xffffffffu, incl, 31);
      }
      if (lane == 0) seg_count[(size_t)c * K + k] = running;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t pos = 0;
    const uint32_t n_seg = n_chunks * K;
    for (uint32_t sgm = 0; sgm < n_seg; ++sgm) {
      seg_start[sgm] = (int32_t)pos;
      pos += (seg_count[sgm] + stage - 1) / stage * stage;
    }
    seg_start[n_seg] = (int32_t)pos;
  }
}

__global__ void __launch_bounds__(256)
k_pair_fill(const int32_t *__restrict__ nbr, uint32_t n, uint32_t nblocks, uint32_t bpc, uint32_t K,
            const uint32_t *__restrict__ block_off, const int32_t *__restrict__ seg_start,
            const uint32_t *__restrict__ seg_count, int32_t *__restrict__ pairs_other,
            int32_t *__restrict__ pairs_row) {
  const uint32_t blk = blockIdx.x, k = blockIdx.y;
  const uint32_t c = blk / bpc, sgm = c * K + k;
  const uint32_t r0 = blk * kPairChunk + threadIdx.x * 8;
  int32_t v[8];
  load8(nbr + (size_t)k * n, r0, n, v);
  uint32_t cn = 0;
#pragma unroll
  for (int j = 0; j < 8; ++j) cn += v[j] >= 0;
  uint32_t total;
  uint32_t pos = (uint32_t)seg_start[sgm] + block_off[(size_t)k * nblocks + blk] +
                 block_excl_scan_256(cn, &total);
#pragma unroll
  for (int j = 0; j < 8; ++j)
    if (v[j] >= 0) {
      pairs_other[pos] = v[j];
      pairs_row[pos] = (int32_t)(r0 + j);
      ++pos;
    }
  if (blk == min((c + 1) * bpc, nblocks) - 1) {   // pad the segment to a whole number of stages
    const uint32_t beg = (uint32_t)seg_start[sgm] + seg_count[sgm], end = (uint32_t)seg_start[sgm + 1];
    for (uint32_t i = beg + threadIdx.x; i < end; i += 256) {
      pairs_other[i] = -1;
      pairs_row[i] = -1;
    }
  }
}

// ---- tile order of a neighbour table (K <= 32) -------------------------------------------------
// The forward / dgrad kernel gives every 128-row tile the stages of every offset.  Rows are
// numbered by first occurrence, which on real clouds is a random order, so every tile reaches
// nearly every offset and a stage whose rows all miss its offset still costs its copies and MMAs.
// Sorting the rows by their neighbour mask (bit k = nbr[k][r] >= 0) packs rows that miss the same
// offsets into the same tiles; the kernel then runs only the offsets of its tile's mask.  The
// order is one int32 buffer of (K + 1) n + ceil(n / 128) words:
//   table  [K][n]  nbr[k][slot_row[s]] at [k][s]   (k-major: the kernel's index reads stay coalesced)
//   slot_row [n]   the row at slot s: rows stably sorted by mask (ties keep row order)
//   tile_mask [ceil(n / 128)]  the OR of the masks of the tile's rows
// The sort is an LSD radix sort over 8-bit digits of the mask (ceil(K / 8) passes), each pass a
// stable counting sort: per-tile digit counts, a scan per digit, a ranked scatter.  No atomics;
// the result does not depend on the order CTAs run in.
constexpr uint32_t kSortBins = 256;     // 8-bit digits
constexpr uint32_t kSortTile = 2048;    // rows per counting-sort tile (one 256-thread block)

__global__ void __launch_bounds__(256)
k_row_mask(const int32_t *__restrict__ nbr, uint32_t K, uint32_t n, uint32_t *__restrict__ mask) {
  const uint32_t r = blockIdx.x * 256 + threadIdx.x;
  if (r >= n) return;
  uint32_t m = 0;
  for (uint32_t k = 0; k < K; ++k) m |= (uint32_t)(__ldg(nbr + (size_t)k * n + r) >= 0) << k;
  mask[r] = m;
}

// digit of the row at position i of the pass's input order (src == NULL: row i)
__device__ __forceinline__ uint32_t sort_digit(const uint32_t *__restrict__ mask,
                                               const int32_t *__restrict__ src, uint32_t i,
                                               uint32_t shift, int32_t &row) {
  row = src != nullptr ? __ldg(src + i) : (int32_t)i;
  return (__ldg(mask + row) >> shift) & (kSortBins - 1);
}

// cnt[d * n_tiles + t] = rows of sort tile t whose digit is d.  Each warp counts its rows per digit
// (one lane per group of equal digits adds the group's size), then the 8 warps' counts are added.
__global__ void __launch_bounds__(256)
k_sort_count(const uint32_t *__restrict__ mask, const int32_t *__restrict__ src, uint32_t n,
             uint32_t shift, uint32_t n_tiles, uint32_t *__restrict__ cnt) {
  __shared__ uint32_t wcnt[8][kSortBins];
  const uint32_t tid = threadIdx.x, warp = tid >> 5, lt = (1u << (tid & 31)) - 1u;
#pragma unroll
  for (int w = 0; w < 8; ++w) wcnt[w][tid] = 0;
  __syncthreads();
  const uint32_t end = min(n, (blockIdx.x + 1) * kSortTile);
  for (uint32_t r0 = blockIdx.x * kSortTile; r0 < end; r0 += 256) {
    const uint32_t i = r0 + tid;
    int32_t row;
    const uint32_t d = i < end ? sort_digit(mask, src, i, shift, row) : kSortBins;
    const uint32_t peers = __match_any_sync(0xffffffffu, d);
    if (d < kSortBins && (peers & lt) == 0) wcnt[warp][d] += __popc(peers);
    __syncwarp();
  }
  __syncthreads();
  uint32_t c = 0;
#pragma unroll
  for (int w = 0; w < 8; ++w) c += wcnt[w][tid];
  cnt[(size_t)tid * n_tiles + blockIdx.x] = c;
}

// one warp per digit d: cnt[d][.] -> exclusive offsets within the digit, total[d] = its rows
__global__ void __launch_bounds__(32)
k_sort_scan(uint32_t *__restrict__ cnt, uint32_t n_tiles, uint32_t *__restrict__ total) {
  const uint32_t lane = threadIdx.x, d = blockIdx.x;
  uint32_t *row = cnt + (size_t)d * n_tiles;
  uint32_t running = 0;
  for (uint32_t base = 0; base < n_tiles; base += 32) {
    const uint32_t i = base + lane;
    const uint32_t v = i < n_tiles ? row[i] : 0u;
    uint32_t incl = v;
#pragma unroll
    for (int s = 1; s < 32; s <<= 1) {
      const uint32_t t = __shfl_up_sync(0xffffffffu, incl, s);
      if (lane >= (uint32_t)s) incl += t;
    }
    if (i < n_tiles) row[i] = running + incl - v;
    running += __shfl_sync(0xffffffffu, incl, 31);
  }
  if (lane == 0) total[d] = running;
}

// Stable scatter of one sort tile, 256 rows per round in ascending order: a row's position is its
// digit's base + the rows of that digit in earlier warps of the round + its rank among the lanes
// of its warp with the same digit (__match_any_sync).
__global__ void __launch_bounds__(256)
k_sort_scatter(const uint32_t *__restrict__ mask, const int32_t *__restrict__ src, uint32_t n,
               uint32_t shift, uint32_t n_tiles, const uint32_t *__restrict__ cnt,
               const uint32_t *__restrict__ total, int32_t *__restrict__ dst) {
  __shared__ uint32_t base[kSortBins];
  __shared__ uint32_t wcnt[8][kSortBins];
  const uint32_t tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, lt = (1u << lane) - 1u;
  uint32_t digit_total;
  const uint32_t digit_base = block_excl_scan_256(__ldg(total + tid), &digit_total);
  base[tid] = digit_base + __ldg(cnt + (size_t)tid * n_tiles + blockIdx.x);
#pragma unroll
  for (int w = 0; w < 8; ++w) wcnt[w][tid] = 0;
  __syncthreads();
  const uint32_t begin = blockIdx.x * kSortTile, end = min(n, begin + kSortTile);
  for (uint32_t r0 = begin; r0 < end; r0 += 256) {
    const uint32_t i = r0 + tid;
    int32_t row = -1;
    const uint32_t d = i < end ? sort_digit(mask, src, i, shift, row) : kSortBins;
    const uint32_t peers = __match_any_sync(0xffffffffu, d);
    if (d < kSortBins && (peers & lt) == 0) wcnt[warp][d] = __popc(peers);
    __syncthreads();
    if (d < kSortBins) {
      uint32_t pos = base[d] + __popc(peers & lt);
      for (uint32_t w = 0; w < warp; ++w) pos += wcnt[w][d];
      dst[pos] = row;
    }
    __syncthreads();
    uint32_t round = 0;
#pragma unroll
    for (int w = 0; w < 8; ++w) { round += wcnt[w][tid]; wcnt[w][tid] = 0; }
    base[tid] += round;
    __syncthreads();
  }
}

// One block per 128-slot tile: its mask and its slots of the table in slot order.
__global__ void __launch_bounds__(128)
k_order_finish(const int32_t *__restrict__ nbr, uint32_t K, uint32_t n,
               const uint32_t *__restrict__ mask, int32_t *__restrict__ order) {
  __shared__ uint32_t wor[4];
  const uint32_t s = blockIdx.x * 128 + threadIdx.x;
  const int32_t *slot_row = order + (size_t)K * n;
  uint32_t *tile_mask = reinterpret_cast<uint32_t *>(order + (size_t)(K + 1) * n);
  const int32_t row = s < n ? __ldg(slot_row + s) : -1;
  const uint32_t m = __reduce_or_sync(0xffffffffu, row >= 0 ? __ldg(mask + row) : 0u);
  if ((threadIdx.x & 31) == 0) wor[threadIdx.x >> 5] = m;
  if (row >= 0)
    for (uint32_t k = 0; k < K; ++k) order[(size_t)k * n + s] = __ldg(nbr + (size_t)k * n + row);
  __syncthreads();
  if (threadIdx.x == 0) tile_mask[blockIdx.x] = wor[0] | wor[1] | wor[2] | wor[3];
}

static int build_tile_order(const int32_t *nbr, uint32_t K, uint32_t n, int32_t *order,
                            void *scratch, cudaStream_t stream) {
  if (n == 0) return MEB200_OK;
  const uint32_t n_tiles = cdiv(n, kSortTile);
  uint32_t *mask = reinterpret_cast<uint32_t *>(scratch);
  int32_t *tmp = reinterpret_cast<int32_t *>(mask + n);
  uint32_t *cnt = reinterpret_cast<uint32_t *>(tmp + n);
  uint32_t *total = cnt + (size_t)kSortBins * n_tiles;
  int32_t *slot_row = order + (size_t)K * n;
  k_row_mask<<<cdiv(n, 256), 256, 0, stream>>>(nbr, K, n, mask);
  MEB_LAUNCH_OK();
  const uint32_t passes = cdiv(K, 8);
  const int32_t *src = nullptr;
  for (uint32_t p = 0; p < passes; ++p) {
    int32_t *dst = (passes - 1 - p) % 2 == 0 ? slot_row : tmp;   // the last pass ends in slot_row
    k_sort_count<<<n_tiles, 256, 0, stream>>>(mask, src, n, 8 * p, n_tiles, cnt);
    MEB_LAUNCH_OK();
    k_sort_scan<<<kSortBins, 32, 0, stream>>>(cnt, n_tiles, total);
    MEB_LAUNCH_OK();
    k_sort_scatter<<<n_tiles, 256, 0, stream>>>(mask, src, n, 8 * p, n_tiles, cnt, total, dst);
    MEB_LAUNCH_OK();
    src = dst;
  }
  k_order_finish<<<cdiv(n, kOrderTileRows), 128, 0, stream>>>(nbr, K, n, mask, order);
  MEB_LAUNCH_OK();
  return MEB200_OK;
}

}  // namespace meb200

using namespace meb200;

extern "C" int meb200_kernel_map(const int32_t *x_coords, uint32_t nx, const int32_t *y_coords,
                                 uint32_t ny, const uint32_t *y_table, uint32_t y_capacity,
                                 uint32_t ncols, const int32_t *offsets, uint32_t K,
                                 int32_t *x_nbr, int32_t *y_nbr, uint32_t *d_num_pairs,
                                 int32_t *x_order, int32_t *y_order, void *order_scratch,
                                 void *stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  MEB_CHECK_ARG(y_capacity >= 2 && (y_capacity & (y_capacity - 1)) == 0, "capacity=%u",
                y_capacity);
  if (K == 0) return MEB200_OK;
  MEB_CHECK_ARG((x_order == nullptr && y_order == nullptr) ||
                    (K <= kMaxOrderK && order_scratch != nullptr &&
                     (y_order == nullptr || ny == 0 || y_nbr)),
                "tile orders need K <= %u (K=%u), scratch and their table", kMaxOrderK, K);
  if (nx > 0) {
    MEB_CHECK_ARG(x_coords && y_table && offsets && x_nbr, "null buffer");
    MEB_CHECK_ARG(ny == 0 || y_coords != nullptr, "y_coords");
    uint64_t total = (uint64_t)nx * K;
    MEB_CHECK_ARG(total < (1ull << 40), "nx*K too large");
    MEB_DISPATCH_NCOLS(ncols, k_kernel_map<NC><<<cdiv(total, 256), 256, 0, stream>>>(
                                  x_coords, nx, y_coords, ny, y_table, y_capacity - 1, offsets, K,
                                  x_nbr, y_nbr, d_num_pairs));
    MEB_LAUNCH_OK();
  }
  // with nx = 0 the caller's y_nbr is all -1: its order is still built (the identity, every tile
  // mask empty), since a forward or dgrad over the y rows reads it
  if (x_order != nullptr) {
    const int rc = build_tile_order(x_nbr, K, nx, x_order, order_scratch, stream);
    if (rc != MEB200_OK) return rc;
  }
  if (y_order != nullptr) return build_tile_order(y_nbr, K, ny, y_order, order_scratch, stream);
  return MEB200_OK;
}


extern "C" uint32_t meb200_pair_list_chunks(uint32_t n_rows, uint32_t chunk_rows) {
  if (chunk_rows == 0 || n_rows == 0) return 1;
  const uint32_t bpc = (chunk_rows + kPairChunk - 1) / kPairChunk;
  const uint32_t nblocks = (n_rows + kPairChunk - 1) / kPairChunk;
  return (nblocks + bpc - 1) / bpc;
}

extern "C" uint64_t meb200_pair_list_scratch_bytes(uint32_t K, uint32_t n_rows, uint32_t chunk_rows) {
  const uint64_t nblocks = (n_rows + kPairChunk - 1) / kPairChunk;
  return (K * nblocks + (uint64_t)K * meb200_pair_list_chunks(n_rows, chunk_rows)) * sizeof(uint32_t) + 256;
}

extern "C" uint64_t meb200_pair_list_capacity(uint32_t K, uint32_t n_rows, uint32_t stage,
                                              uint32_t chunk_rows) {
  return (uint64_t)K * n_rows + (uint64_t)K * stage * meb200_pair_list_chunks(n_rows, chunk_rows);
}

extern "C" int meb200_kernel_map_pairs(const int32_t *nbr, uint32_t K, uint32_t n_rows,
                                       uint32_t stage, uint32_t chunk_rows, int32_t *pairs_other,
                                       int32_t *pairs_row, int32_t *seg_start, void *scratch,
                                       void *stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  MEB_CHECK_ARG(K > 0 && K <= 65535 && stage > 0, "K=%u stage=%u", K, stage);
  MEB_CHECK_ARG(seg_start != nullptr, "seg_start");
  const uint32_t n_chunks = meb200_pair_list_chunks(n_rows, chunk_rows);
  MEB_CHECK_ARG(meb200_pair_list_capacity(K, n_rows, stage, chunk_rows) < (1ull << 31),
                "pair list too long");
  if (n_rows == 0) {
    MEB_CUDA(cudaMemsetAsync(seg_start, 0, ((size_t)K + 1) * sizeof(int32_t), stream));
    return MEB200_OK;
  }
  MEB_CHECK_ARG(nbr && pairs_other && pairs_row && scratch, "null buffer");
  const uint32_t nblocks = (n_rows + kPairChunk - 1) / kPairChunk;
  const uint32_t bpc = chunk_rows == 0 ? nblocks : (chunk_rows + kPairChunk - 1) / kPairChunk;
  uint32_t *cnt = reinterpret_cast<uint32_t *>(scratch);
  uint32_t *seg_count = cnt + (size_t)K * nblocks;
  dim3 grid(nblocks, K);
  k_pair_count<<<grid, 256, 0, stream>>>(nbr, n_rows, nblocks, cnt);
  MEB_LAUNCH_OK();
  k_pair_scan<<<1, 1024, 0, stream>>>(cnt, K, nblocks, bpc, n_chunks, stage, seg_start, seg_count);
  MEB_LAUNCH_OK();
  k_pair_fill<<<grid, 256, 0, stream>>>(nbr, n_rows, nblocks, bpc, K, cnt, seg_start, seg_count,
                                        pairs_other, pairs_row);
  MEB_LAUNCH_OK();
  return MEB200_OK;
}
