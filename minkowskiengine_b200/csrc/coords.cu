// Coordinate hashing: deduplicating insert, strided / region candidate generation, find.
//
// Replaces (does not port) the reference's cuDF-map based CoordinateMapGPU
// (src/coordinate_map_gpu.cu:70-96,196-278,366-483,502-607).  Design (DESIGN.md §3):
//   * the table holds 4-byte ROW INDICES only; keys are compared against the int32
//     coordinate rows themselves (16 B vector load for D=3), so a probe touches one
//     table sector and one coordinate sector, both L2-resident at these sizes;
//   * duplicates resolve deterministically to the smallest row (atomicMin on the slot),
//     which reproduces the CPU reference's "first occurrence wins, numbered by rank of
//     first occurrence" (coordinate_map_cpu.hpp:353-380) bit for bit;
//   * compaction is a two-kernel count/fill scan — no thrust, no sort, no host round
//     trip except the single read of the unique count the caller needs to size tensors.
#include "common.cuh"

namespace meb200 {

constexpr int kScanThreads = 256;
constexpr int kScanItems = 8;
constexpr int kScanTile = kScanThreads * kScanItems;

struct InsertScratch {
  uint32_t *slot_of;     // [n]
  uint32_t *rank_of;     // [n]
  uint32_t *block_sums;  // [nblocks]
  uint32_t *ticket;      // [1]
  uint32_t *total;       // [1]
};

static inline uint32_t scan_blocks(uint32_t n) { return n == 0 ? 1 : cdiv(n, kScanTile); }

static InsertScratch carve(void *scratch, uint32_t n) {
  InsertScratch s;
  uint32_t *p = reinterpret_cast<uint32_t *>(scratch);
  s.slot_of = p;
  s.rank_of = p + n;
  s.block_sums = p + 2 * (size_t)n;
  s.ticket = s.block_sums + scan_blocks(n);
  s.total = s.ticket + 1;
  return s;
}

template <int NC>
__global__ void __launch_bounds__(256)
k_insert(const int32_t *__restrict__ coords, const uint8_t *__restrict__ valid,
         const uint32_t *__restrict__ d_n, uint32_t n, uint32_t *__restrict__ table, uint32_t mask,
         uint32_t *__restrict__ slot_of) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  // d_n: the number of meaningful rows lives on the device (a map enqueued before its parent's
  // size reached the host); rows past it take no part
  if ((valid != nullptr && valid[i] == 0) || (d_n != nullptr && i >= *d_n)) {
    slot_of[i] = kEmpty;
    return;
  }
  int32_t key[NC];
  load_coord<NC>(coords, i, key);
  uint32_t h = hash_coord<NC>(key) & mask;
  while (true) {
    uint32_t cur = *reinterpret_cast<volatile uint32_t *>(table + h);
    if (cur == kEmpty) {
      cur = atomicCAS(table + h, kEmpty, i);
      if (cur == kEmpty) break;  // claimed an empty slot
    }
    // slot owned by row `cur` (a slot never changes key once claimed)
    int32_t other[NC];
    load_coord<NC>(coords, cur, other);
    if (coord_eq<NC>(other, key)) {
      atomicMin(table + h, i);  // first occurrence wins
      break;
    }
    h = (h + 1) & mask;
  }
  slot_of[i] = h;
}

__device__ __forceinline__ bool is_winner(const uint32_t *__restrict__ table,
                                          const uint32_t *__restrict__ slot_of, uint32_t i) {
  uint32_t s = slot_of[i];
  return s != kEmpty && table[s] == i;
}

// Pass 1: winners per tile; the last block to finish scans the tile sums.
__global__ void __launch_bounds__(kScanThreads)
k_count(const uint32_t *__restrict__ table, const uint32_t *__restrict__ slot_of, uint32_t n,
        uint32_t *__restrict__ block_sums, uint32_t *__restrict__ ticket,
        uint32_t *__restrict__ total) {
  __shared__ uint32_t s_warp[kScanThreads / 32];
  __shared__ bool s_last;
  uint32_t base = blockIdx.x * kScanTile + threadIdx.x * kScanItems;
  uint32_t c = 0;
#pragma unroll
  for (int j = 0; j < kScanItems; ++j) {
    uint32_t i = base + j;
    if (i < n) c += is_winner(table, slot_of, i) ? 1u : 0u;
  }
  for (int o = 16; o > 0; o >>= 1) c += __shfl_down_sync(0xffffffffu, c, o);
  if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t t = 0;
    for (int w = 0; w < kScanThreads / 32; ++w) t += s_warp[w];
    block_sums[blockIdx.x] = t;
    __threadfence();
    s_last = (atomicAdd(ticket, 1u) == gridDim.x - 1);
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  // exclusive scan of block_sums[0..gridDim.x) by this block
  __shared__ uint32_t s_part[kScanThreads];
  uint32_t nb = gridDim.x;
  uint32_t per = (nb + kScanThreads - 1) / kScanThreads;
  uint32_t lo = threadIdx.x * per, hi = min(lo + per, nb);
  uint32_t sum = 0;
  for (uint32_t b = lo; b < hi; ++b) sum += *reinterpret_cast<volatile uint32_t *>(block_sums + b);
  s_part[threadIdx.x] = sum;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t run = 0;
    for (int t = 0; t < kScanThreads; ++t) {
      uint32_t v = s_part[t];
      s_part[t] = run;
      run += v;
    }
    *total = run;
  }
  __syncthreads();
  uint32_t run = s_part[threadIdx.x];
  for (uint32_t b = lo; b < hi; ++b) {
    uint32_t v = block_sums[b];
    block_sums[b] = run;
    run += v;
  }
}

// Pass 2: ranks of the winners, compacted coordinates and the unique_index list.
template <int NC>
__global__ void __launch_bounds__(kScanThreads)
k_fill(const int32_t *__restrict__ coords, const uint32_t *__restrict__ table,
       const uint32_t *__restrict__ slot_of, uint32_t n,
       const uint32_t *__restrict__ block_offsets, uint32_t *__restrict__ rank_of,
       int32_t *__restrict__ unique_coords, int64_t *__restrict__ unique_index) {
  __shared__ uint32_t s_warp[kScanThreads / 32];
  uint32_t base = blockIdx.x * kScanTile + threadIdx.x * kScanItems;
  uint32_t flags = 0, c = 0;
#pragma unroll
  for (int j = 0; j < kScanItems; ++j) {
    uint32_t i = base + j;
    if (i < n && is_winner(table, slot_of, i)) {
      flags |= 1u << j;
      ++c;
    }
  }
  // block-wide exclusive scan of c
  uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t incl = c;
  for (int o = 1; o < 32; o <<= 1) {
    uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= (uint32_t)o) incl += v;
  }
  if (lane == 31) s_warp[warp] = incl;
  __syncthreads();
  uint32_t warp_off = 0;
  for (uint32_t w = 0; w < warp; ++w) warp_off += s_warp[w];
  uint32_t rank = block_offsets[blockIdx.x] + warp_off + incl - c;
#pragma unroll
  for (int j = 0; j < kScanItems; ++j) {
    if (flags & (1u << j)) {
      uint32_t i = base + j;
      rank_of[i] = rank;
      unique_index[rank] = (int64_t)i;
      int32_t key[NC];
      load_coord<NC>(coords, i, key);
      store_coord<NC>(unique_coords, rank, key);
      ++rank;
    }
  }
}

__global__ void __launch_bounds__(256)
k_inverse(const uint32_t *__restrict__ table, const uint32_t *__restrict__ slot_of,
          const uint32_t *__restrict__ rank_of, uint32_t n, int64_t *__restrict__ inverse_map) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint32_t s = slot_of[i];
  inverse_map[i] = (s == kEmpty) ? -1 : (int64_t)rank_of[table[s]];
}

// Insert of rows known to be distinct (table rebuild over the compacted coordinates).
template <int NC>
__global__ void __launch_bounds__(256)
k_insert_unique(const int32_t *__restrict__ coords, uint32_t n, uint32_t *__restrict__ table,
                uint32_t mask) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int32_t key[NC];
  load_coord<NC>(coords, i, key);
  uint32_t h = hash_coord<NC>(key) & mask;
  while (atomicCAS(table + h, kEmpty, i) != kEmpty) h = (h + 1) & mask;
}

__device__ __forceinline__ int32_t floor_div(int32_t a, int32_t b) {
  int32_t q = a / b, r = a % b;
  return (r != 0 && ((r < 0) != (b < 0))) ? q - 1 : q;
}

template <int NC>
__global__ void __launch_bounds__(256)
k_stride_coords(const int32_t *__restrict__ coords, uint32_t n, IntVec ts,
                int32_t *__restrict__ out) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int32_t c[NC];
  load_coord<NC>(coords, i, c);
#pragma unroll
  for (int j = 1; j < NC; ++j) c[j] = floor_div(c[j], ts.v[j - 1]) * ts.v[j - 1];
  store_coord<NC>(out, i, c);
}

template <int NC>
__global__ void __launch_bounds__(256)
k_region_coords(const int32_t *__restrict__ coords, uint32_t n,
                const int32_t *__restrict__ offsets, uint32_t K, IntVec ts, int aligned_only,
                int32_t *__restrict__ out, uint8_t *__restrict__ valid) {
  uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (uint64_t)n * K) return;
  uint32_t i = (uint32_t)(t / K), k = (uint32_t)(t % K);
  int32_t c[NC];
  load_coord<NC>(coords, i, c);
  bool ok = true;
#pragma unroll
  for (int j = 1; j < NC; ++j) {
    c[j] += __ldg(offsets + (size_t)k * (NC - 1) + (j - 1));
    if (aligned_only) ok &= (c[j] % ts.v[j - 1] == 0);
  }
  store_coord<NC>(out, (uint32_t)t, c);
  valid[t] = ok ? 1 : 0;
}

template <int NC>
__global__ void __launch_bounds__(256)
k_find(const int32_t *__restrict__ map_coords, const uint32_t *__restrict__ table, uint32_t mask,
       const int32_t *__restrict__ query, uint32_t nq, int32_t *__restrict__ result) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nq) return;
  int32_t key[NC];
  load_coord<NC>(query, i, key);
  result[i] = table_find<NC>(map_coords, table, mask, key);
}

uint32_t *insert_flag_word(void *scratch, uint32_t n) { return carve(scratch, n).total + 1; }

// Enqueues the insert of n > 0 candidate rows; the unique count is left in the scratch
// (carve(scratch, n).total).  d_n: the number of meaningful rows when it lives on the device.
static int enqueue_insert(const int32_t *coords, const uint8_t *valid, const uint32_t *d_n,
                          uint32_t n, uint32_t ncols, uint32_t *table, uint32_t capacity,
                          int32_t *unique_coords, int64_t *unique_index, int64_t *inverse_map,
                          void *scratch, cudaStream_t stream) {
  int rc = check_table(table, capacity, n);
  if (rc != MEB200_OK) return rc;
  MEB_CHECK_ARG(coords && unique_coords && unique_index && inverse_map && scratch, "null buffer");
  MEB_CUDA(cudaMemsetAsync(table, 0xFF, (size_t)capacity * 4, stream));
  InsertScratch s = carve(scratch, n);
  uint32_t nb = scan_blocks(n);
  MEB_CUDA(cudaMemsetAsync(s.ticket, 0, 8, stream));
  uint32_t mask = capacity - 1;
  MEB_DISPATCH_NCOLS(ncols, k_insert<NC><<<cdiv(n, 256), 256, 0, stream>>>(
                                coords, valid, d_n, n, table, mask, s.slot_of));
  MEB_LAUNCH_OK();
  k_count<<<nb, kScanThreads, 0, stream>>>(table, s.slot_of, n, s.block_sums, s.ticket, s.total);
  MEB_LAUNCH_OK();
  MEB_DISPATCH_NCOLS(ncols, k_fill<NC><<<nb, kScanThreads, 0, stream>>>(
                                coords, table, s.slot_of, n, s.block_sums, s.rank_of,
                                unique_coords, unique_index));
  MEB_LAUNCH_OK();
  k_inverse<<<cdiv(n, 256), 256, 0, stream>>>(table, s.slot_of, s.rank_of, n, inverse_map);
  MEB_LAUNCH_OK();
  return MEB200_OK;
}

// Table over m rows known to be distinct.
static int build_table(const int32_t *coords, uint32_t m, uint32_t ncols, uint32_t *table,
                       uint32_t capacity, cudaStream_t stream) {
  int rc = check_table(table, capacity, m);
  if (rc != MEB200_OK) return rc;
  MEB_CUDA(cudaMemsetAsync(table, 0xFF, (size_t)capacity * 4, stream));
  if (m == 0) return MEB200_OK;
  MEB_CHECK_ARG(coords != nullptr, "null coordinates");
  MEB_DISPATCH_NCOLS(ncols, k_insert_unique<NC><<<cdiv(m, 256), 256, 0, stream>>>(
                                coords, m, table, capacity - 1));
  MEB_LAUNCH_OK();
  return MEB200_OK;
}

int insert_and_map(const int32_t *coords, const uint8_t *valid, uint32_t n, uint32_t ncols,
                   uint32_t *table, uint32_t capacity, int32_t *unique_coords,
                   int64_t *unique_index, int64_t *inverse_map, void *scratch,
                   uint32_t *h_num_unique, uint32_t h_words, cudaStream_t stream) {
  MEB_CHECK_ARG(h_num_unique != nullptr, "h_num_unique");
  if (n == 0) {
    int rc = build_table(nullptr, 0, ncols, table, capacity, stream);
    if (rc == MEB200_OK) *h_num_unique = 0;
    return rc;
  }
  int rc = enqueue_insert(coords, valid, nullptr, n, ncols, table, capacity, unique_coords,
                          unique_index, inverse_map, scratch, stream);
  if (rc != MEB200_OK) return rc;
  MEB_CUDA(cudaMemcpyAsync(h_num_unique, carve(scratch, n).total, 4 * h_words,
                           cudaMemcpyDeviceToHost, stream));
  MEB_CUDA(cudaStreamSynchronize(stream));
  uint32_t m = *h_num_unique;
  // duplicates or masked rows: rebuild the table over the compacted rows
  return m != n ? build_table(unique_coords, m, ncols, table, capacity, stream) : MEB200_OK;
}

}  // namespace meb200

using namespace meb200;

extern "C" {

uint32_t meb200_hash_capacity(uint32_t n) {
  uint64_t want = (uint64_t)n * 3u;
  uint64_t cap = 1024;
  while (cap < want) cap <<= 1;
  return (uint32_t)(cap > 0x80000000ull ? 0x80000000ull : cap);
}

uint64_t meb200_insert_scratch_bytes(uint32_t n) {
  return 4ull * (2ull * n + scan_blocks(n) + 8);
}

int meb200_insert_and_map(const int32_t *coords, const uint8_t *valid, uint32_t n,
                          uint32_t ncols, uint32_t *table, uint32_t capacity,
                          int32_t *unique_coords, int64_t *unique_index, int64_t *inverse_map,
                          void *scratch, uint32_t *h_num_unique, void *stream_) {
  return meb200::insert_and_map(coords, valid, n, ncols, table, capacity, unique_coords,
                                unique_index, inverse_map, scratch, h_num_unique, 1,
                                (cudaStream_t)stream_);
}

int meb200_insert_and_map_enqueue(const int32_t *coords, const uint8_t *valid,
                                  const uint32_t *d_n, uint32_t n, uint32_t ncols,
                                  uint32_t *table, uint32_t capacity, int32_t *unique_coords,
                                  int64_t *unique_index, int64_t *inverse_map, void *scratch,
                                  uint32_t *d_num_unique, void *stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  MEB_CHECK_ARG(d_num_unique != nullptr && n > 0, "enqueue: count pointer / empty input");
  int rc = enqueue_insert(coords, valid, d_n, n, ncols, table, capacity, unique_coords,
                          unique_index, inverse_map, scratch, stream);
  if (rc != MEB200_OK) return rc;
  MEB_CUDA(cudaMemcpyAsync(d_num_unique, carve(scratch, n).total, 4, cudaMemcpyDeviceToDevice,
                           stream));
  return MEB200_OK;
}

int meb200_map_build_table(const int32_t *unique_coords, uint32_t m, uint32_t ncols,
                           uint32_t *table, uint32_t capacity, void *stream_) {
  return build_table(unique_coords, m, ncols, table, capacity, (cudaStream_t)stream_);
}

int meb200_stride_coords(const int32_t *coords, uint32_t n, uint32_t ncols,
                         const int32_t *out_tensor_stride, int32_t *out, void *stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  MEB_CHECK_ARG(ncols >= 2 && ncols <= MEB200_MAX_NCOLS, "ncols=%u", ncols);
  if (n == 0) return MEB200_OK;
  MEB_CHECK_ARG(coords && out, "null buffer");
  IntVec ts;
  int rc = load_strides(out_tensor_stride, ncols, &ts);
  if (rc != MEB200_OK) return rc;
  MEB_DISPATCH_NCOLS(ncols,
                     k_stride_coords<NC><<<cdiv(n, 256), 256, 0, stream>>>(coords, n, ts, out));
  MEB_LAUNCH_OK();
  return MEB200_OK;
}

int meb200_region_coords(const int32_t *coords, uint32_t n, uint32_t ncols,
                         const int32_t *offsets, uint32_t K, const int32_t *out_tensor_stride,
                         int aligned_only, int32_t *out, uint8_t *valid, void *stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  MEB_CHECK_ARG(ncols >= 2 && ncols <= MEB200_MAX_NCOLS, "ncols=%u", ncols);
  if (n == 0 || K == 0) return MEB200_OK;
  MEB_CHECK_ARG(coords && out && valid && offsets, "null buffer");
  MEB_CHECK_ARG((uint64_t)n * K < 0xFFFFFFFFull, "n*K too large");
  IntVec ts;
  int rc = load_strides(out_tensor_stride, ncols, &ts);
  if (rc != MEB200_OK) return rc;
  MEB_DISPATCH_NCOLS(ncols, k_region_coords<NC><<<cdiv((uint64_t)n * K, 256), 256, 0, stream>>>(
                                coords, n, offsets, K, ts, aligned_only, out, valid));
  MEB_LAUNCH_OK();
  return MEB200_OK;
}

int meb200_map_find(const int32_t *map_coords, const uint32_t *table, uint32_t capacity,
                    uint32_t ncols, const int32_t *query, uint32_t nq, int32_t *result,
                    void *stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  MEB_CHECK_ARG(capacity >= 2 && (capacity & (capacity - 1)) == 0, "capacity=%u", capacity);
  if (nq == 0) return MEB200_OK;
  MEB_CHECK_ARG(table && query && result, "null buffer");
  MEB_DISPATCH_NCOLS(ncols, k_find<NC><<<cdiv(nq, 256), 256, 0, stream>>>(
                                map_coords, table, capacity - 1, query, nq, result));
  MEB_LAUNCH_OK();
  return MEB200_OK;
}

}
