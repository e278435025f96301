// The border between sparse tensors and dense torch tensors: feature rows -> dense volume, dense
// volume -> feature rows, and the coordinates of the non-zero cells of a dense volume.
//
// Reference semantics: SparseTensor.dense (MinkowskiSparseTensor.py:460-557), to_sparse
// (MinkowskiOps.py:279-317).  The reference zero-fills the volume and index-assigns the rows into
// it, and finds the non-zero cells with abs().sum() + where() + stack().  Here every kernel is
// stationary over what it writes, so each output element is written exactly once, with no memset
// and no atomics.  Everything is data movement: values travel as raw 2- or 4-byte words, so the
// results are bit-exact in every dtype.
//
// A dense tensor is described by element strides (meb200_dense_desc), so any axis order and any
// strided view is read or written in place; offsets are 64-bit.
#include <type_traits>

#include "common.cuh"

namespace meb200 {

constexpr int kDenseThreads = 256;
constexpr int kTileCells = 128;  // cells per CTA of rows -> dense
constexpr int kChunk = 32;       // channels staged per pass when the channel axis is not innermost

// The raw word a feature element travels as
template <typename T>
using word_t = std::conditional_t<sizeof(T) == 4, uint32_t, uint16_t>;

// Index of cell `cell` (row-major over batch, X1..XD) along every axis -> its element offset
__device__ __forceinline__ int64_t cell_offset(const meb200_dense_desc &d, uint64_t cell,
                                               int32_t *idx) {
  int64_t off = 0;
  for (int j = (int)d.ncols - 1; j >= 0; --j) {
    uint32_t s = d.shape[j];
    uint32_t i = (uint32_t)(cell % s);
    cell /= s;
    idx[j] = (int32_t)i;
    off += (int64_t)i * d.stride[j];
  }
  return off;
}

// V words from p (one 16-byte load when V > 1), or zeros when p is null
template <typename U, int V>
__device__ __forceinline__ void load_words(const U *p, U (&w)[V]) {
  if (p == nullptr) {
#pragma unroll
    for (int e = 0; e < V; ++e) w[e] = 0;
  } else if constexpr (V == 1) {
    w[0] = *p;
  } else {
    static_assert(V * sizeof(U) == 16, "16-byte vectors");
    uint4 v = __ldg(reinterpret_cast<const uint4 *>(p));
    const U *e = reinterpret_cast<const U *>(&v);
#pragma unroll
    for (int j = 0; j < V; ++j) w[j] = e[j];
  }
}

template <typename U, int V>
__device__ __forceinline__ void store_words(U *p, const U (&w)[V]) {
  if constexpr (V == 1) {
    *p = w[0];
  } else {
    uint4 v;
    U *e = reinterpret_cast<U *>(&v);
#pragma unroll
    for (int j = 0; j < V; ++j) e[j] = w[j];
    *reinterpret_cast<uint4 *>(p) = v;
  }
}

// ---- rows -> dense: stationary over the cells ---------------------------------------------------
// A CTA owns kTileCells consecutive cells.  One thread per cell probes the map at
// origin + index * step and leaves the row (or -1) and the cell's offset in shared memory; then the
// CTA writes every channel of every cell.  CLAST (channel stride 1): consecutive threads write
// consecutive channels of a cell, V at a time.  Otherwise the feature rows are read V at a time into
// a shared [cell][channel] tile and written with consecutive threads on consecutive cells, the
// innermost axis of a channel-first volume.
template <typename U, int V, int NC, bool CLAST>
__global__ void __launch_bounds__(kDenseThreads)
k_dense_from_rows(const U *__restrict__ feats, uint32_t C, const int32_t *__restrict__ map_coords,
                  const uint32_t *__restrict__ table, uint32_t mask, meb200_dense_desc d,
                  uint64_t cells, U *__restrict__ dense) {
  __shared__ int32_t s_row[kTileCells];
  __shared__ int64_t s_off[kTileCells];
  __shared__ __align__(16) U s_tile[CLAST ? 1 : kTileCells * (kChunk + 1)];
  uint64_t cell0 = (uint64_t)blockIdx.x * kTileCells;
  uint32_t ncell = (uint32_t)min((uint64_t)kTileCells, cells - cell0);
  if (threadIdx.x < ncell) {
    int32_t key[NC];
    s_off[threadIdx.x] = cell_offset(d, cell0 + threadIdx.x, key);
#pragma unroll
    for (int j = 0; j < NC; ++j) key[j] = d.origin[j] + key[j] * d.step[j];
    s_row[threadIdx.x] = table_find<NC>(map_coords, table, mask, key);
  }
  __syncthreads();
  if constexpr (CLAST) {
    uint32_t CV = C / V;
    for (uint32_t i = threadIdx.x; i < ncell * CV; i += kDenseThreads) {
      uint32_t j = i / CV, c = (i % CV) * V;
      int32_t r = s_row[j];
      U w[V];
      load_words<U, V>(r >= 0 ? feats + (size_t)r * C + c : nullptr, w);
      store_words<U, V>(dense + s_off[j] + c, w);
    }
  } else {
    for (uint32_t c0 = 0; c0 < C; c0 += kChunk) {
      uint32_t cw = min((uint32_t)kChunk, C - c0), CV = cw / V;
      for (uint32_t i = threadIdx.x; i < ncell * CV; i += kDenseThreads) {
        uint32_t j = i / CV, c = (i % CV) * V;
        int32_t r = s_row[j];
        U w[V];
        load_words<U, V>(r >= 0 ? feats + (size_t)r * C + c0 + c : nullptr, w);
#pragma unroll
        for (int e = 0; e < V; ++e) s_tile[j * (kChunk + 1) + c + e] = w[e];
      }
      __syncthreads();
      for (uint32_t i = threadIdx.x; i < cw * kTileCells; i += kDenseThreads) {
        uint32_t c = i / kTileCells, j = i % kTileCells;
        if (j < ncell) dense[s_off[j] + (int64_t)(c0 + c) * d.channel_stride] = s_tile[j * (kChunk + 1) + c];
      }
      __syncthreads();
    }
  }
}

// ---- dense -> rows: stationary over the rows ----------------------------------------------------
// out[r, :] = the cell of coordinate row r, zero when the row lies outside the volume or off the
// step lattice.  dense_vec: the V channels of an access are one aligned 16-byte word of the volume.
template <typename U, int V>
__global__ void __launch_bounds__(kDenseThreads)
k_dense_to_rows(const U *__restrict__ dense, meb200_dense_desc d, bool dense_vec,
                const int32_t *__restrict__ coords, uint32_t n, uint32_t C, U *__restrict__ out) {
  uint32_t CV = C / V;
  uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (uint64_t)n * CV) return;
  uint32_t r = (uint32_t)(t / CV), c = (uint32_t)(t % CV) * V;
  int64_t off = 0;
  bool inside = true;
  for (uint32_t j = 0; j < d.ncols; ++j) {
    int64_t rel = (int64_t)__ldg(coords + (size_t)r * d.ncols + j) - d.origin[j];
    int64_t q = rel / d.step[j];
    inside &= rel >= 0 && rel % d.step[j] == 0 && q < (int64_t)d.shape[j];
    off += q * d.stride[j];
  }
  U w[V];
  if (!inside) {
    load_words<U, V>(nullptr, w);
  } else if (dense_vec) {
    load_words<U, V>(dense + off + c, w);
  } else {
#pragma unroll
    for (int e = 0; e < V; ++e) w[e] = __ldg(dense + off + (int64_t)(c + e) * d.channel_stride);
  }
  store_words<U, V>(out + (size_t)r * C + c, w);
}

// ---- non-zero cells: flag + scan + fill ----------------------------------------------------------
// The insert's compaction (coords.cu) is bound to its winner test and its outputs (ranks, the
// unique_index list, a copy of the winning rows); this one flags cells from the volume and writes
// their indices, so it shares the approach (tile counts, one CTA scans them) and not the code.
constexpr int kNzItems = 8;
constexpr int kNzTile = kDenseThreads * kNzItems;

struct NonzeroScratch {
  uint8_t *flag;         // [tiles * kNzTile]
  uint32_t *block_sums;  // [tiles]
  uint32_t *total;       // [1]
};

static inline uint32_t nz_tiles(uint64_t cells) { return cells == 0 ? 1 : cdiv(cells, kNzTile); }

static NonzeroScratch nz_carve(void *scratch, uint64_t cells) {
  NonzeroScratch s;
  uint32_t tiles = nz_tiles(cells);
  s.flag = reinterpret_cast<uint8_t *>(scratch);
  s.block_sums = reinterpret_cast<uint32_t *>(s.flag + (size_t)tiles * kNzTile);
  s.total = s.block_sums + tiles;
  return s;
}

// Every bit of a word except the sign bit(s): zero for +0 and -0 only, so NaN counts as non-zero,
// as in the reference's abs(x).sum(channel) != 0
template <typename U>
__device__ __forceinline__ uint32_t magnitude_bits(uint32_t packed) {
  return packed & (sizeof(U) == 4 ? 0x7fffffffu : 0x7fff7fffu);
}

// Pass 1: flag[cell] = any channel non-zero; non-zero cells per tile.
template <typename U, int V>
__global__ void __launch_bounds__(kDenseThreads)
k_nonzero_flag(const U *__restrict__ dense, meb200_dense_desc d, bool dense_vec, uint32_t cells,
               NonzeroScratch s) {
  __shared__ uint32_t s_warp[kDenseThreads / 32];
  uint32_t count = 0;
  for (int it = 0; it < kNzItems; ++it) {
    // consecutive threads on consecutive cells: coalesced along the innermost axis of a
    // channel-first volume
    uint32_t cell = blockIdx.x * kNzTile + it * kDenseThreads + threadIdx.x;
    if (cell >= cells) break;
    int32_t idx[MEB200_MAX_NCOLS];
    int64_t off = cell_offset(d, cell, idx);
    uint32_t any = 0;
    if (dense_vec) {
      for (uint32_t c = 0; c < d.channels; c += V) {
        uint4 v = __ldg(reinterpret_cast<const uint4 *>(dense + off + c));
        any |= magnitude_bits<U>(v.x | v.y | v.z | v.w);
      }
    } else {
      for (uint32_t c = 0; c < d.channels; ++c)
        any |= magnitude_bits<U>(__ldg(dense + off + (int64_t)c * d.channel_stride));
    }
    s.flag[cell] = any != 0;
    count += any != 0;
  }
  for (int o = 16; o > 0; o >>= 1) count += __shfl_down_sync(0xffffffffu, count, o);
  if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = count;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t t = 0;
    for (int w = 0; w < kDenseThreads / 32; ++w) t += s_warp[w];
    s.block_sums[blockIdx.x] = t;
  }
}

// One CTA: the tile counts -> exclusive offsets, and the total.
__global__ void __launch_bounds__(kDenseThreads) k_nonzero_scan(uint32_t nb, NonzeroScratch s) {
  __shared__ uint32_t s_part[kDenseThreads];
  uint32_t per = (nb + kDenseThreads - 1) / kDenseThreads;
  uint32_t lo = min(threadIdx.x * per, nb), hi = min(lo + per, nb);
  uint32_t sum = 0;
  for (uint32_t b = lo; b < hi; ++b) sum += s.block_sums[b];
  s_part[threadIdx.x] = sum;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t run = 0;
    for (int t = 0; t < kDenseThreads; ++t) {
      uint32_t v = s_part[t];
      s_part[t] = run;
      run += v;
    }
    *s.total = run;
  }
  __syncthreads();
  uint32_t run = s_part[threadIdx.x];
  for (uint32_t b = lo; b < hi; ++b) {
    uint32_t v = s.block_sums[b];
    s.block_sums[b] = run;
    run += v;
  }
}

// Pass 2: the indices of the flagged cells, in cell order (row-major over batch, X1..XD: the order
// torch.where gives).  A thread owns kNzItems consecutive cells.
__global__ void __launch_bounds__(kDenseThreads)
k_nonzero_fill(meb200_dense_desc d, uint32_t cells, NonzeroScratch s, int32_t *__restrict__ coords) {
  __shared__ uint32_t s_warp[kDenseThreads / 32];
  uint32_t base = blockIdx.x * kNzTile + threadIdx.x * kNzItems;
  uint32_t flags = 0, c = 0;
#pragma unroll
  for (int j = 0; j < kNzItems; ++j) {
    if (base + j < cells && s.flag[base + j]) {
      flags |= 1u << j;
      ++c;
    }
  }
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
  uint32_t rank = s.block_sums[blockIdx.x] + warp_off + incl - c;
#pragma unroll
  for (int j = 0; j < kNzItems; ++j) {
    if (flags & (1u << j)) {
      int32_t idx[MEB200_MAX_NCOLS];
      cell_offset(d, base + j, idx);
      for (uint32_t k = 0; k < d.ncols; ++k) coords[(size_t)rank * d.ncols + k] = idx[k];
      ++rank;
    }
  }
}

// ---- host side -----------------------------------------------------------------------------------
static int check_desc(const meb200_dense_desc *d, uint64_t *cells) {
  MEB_CHECK_ARG(d != nullptr, "null dense descriptor");
  MEB_CHECK_ARG(d->ncols >= 2 && d->ncols <= MEB200_MAX_NCOLS, "ncols=%u", d->ncols);
  uint64_t n = 1;
  for (uint32_t j = 0; j < d->ncols; ++j) {
    MEB_CHECK_ARG(d->step[j] > 0, "step must be positive (column %u: %d)", j, d->step[j]);
    MEB_CHECK_ARG(d->stride[j] >= 0, "negative stride (column %u)", j);
    MEB_CHECK_ARG(d->shape[j] == 0 || n <= UINT64_MAX / d->shape[j], "volume too large");
    n *= d->shape[j];
  }
  MEB_CHECK_ARG(d->channel_stride >= 0, "negative channel stride");
  *cells = n;
  return MEB200_OK;
}

// V channels of a cell are one aligned 16-byte word of the volume: the channel axis is innermost,
// the base is 16-byte aligned and every other stride is a multiple of V
static bool dense_vectorises(const void *dense, const meb200_dense_desc &d, size_t elem) {
  uint32_t V = vec_elems(elem, d.channels);
  if (V == 1 || d.channel_stride != 1 || !aligned(16, (const char *)dense)) return false;
  for (uint32_t j = 0; j < d.ncols; ++j)
    if (d.stride[j] % V != 0) return false;
  return true;
}

template <typename U, int V, bool CLAST>
static int launch_from_rows(const void *feats, const int32_t *map_coords, const uint32_t *table,
                            uint32_t capacity, const meb200_dense_desc &d, uint64_t cells,
                            void *dense, cudaStream_t st) {
  unsigned blocks = cdiv(cells, kTileCells);
  MEB_DISPATCH_NCOLS(d.ncols, k_dense_from_rows<U, V, NC, CLAST><<<blocks, kDenseThreads, 0, st>>>(
                                  (const U *)feats, d.channels, map_coords, table, capacity - 1, d,
                                  cells, (U *)dense));
  return MEB200_OK;
}

}  // namespace meb200

using namespace meb200;

extern "C" {

int meb200_dense_from_rows(const void *feats, int dtype, uint32_t n, const int32_t *map_coords,
                           const uint32_t *table, uint32_t capacity,
                           const meb200_dense_desc *desc, void *dense, void *stream) {
  uint64_t cells;
  int rc = check_desc(desc, &cells);
  if (rc != MEB200_OK) return rc;
  const meb200_dense_desc &d = *desc;
  if (cells == 0 || d.channels == 0) return MEB200_OK;
  rc = check_table(table, capacity, n);
  if (rc != MEB200_OK) return rc;
  MEB_CHECK_ARG(dense && (n == 0 || (feats && map_coords)), "null buffer");
  MEB_CHECK_ARG(cells <= (uint64_t)kTileCells * 0x7fffffffull, "volume too large");
  cudaStream_t s = (cudaStream_t)stream;
  // channel-last writes V channels at once; channel-first only reads the feature rows V at a time
  bool clast = d.channel_stride == 1 && d.channels > 1;
  MEB_DISPATCH_DTYPE(dtype, {
    using U = word_t<T>;
    bool ok = aligned(16, (const char *)feats) && (!clast || dense_vectorises(dense, d, sizeof(T)));
    MEB_DISPATCH_VEC(T, d.channels, ok, {
      rc = clast ? launch_from_rows<U, V, true>(feats, map_coords, table, capacity, d, cells, dense, s)
                 : launch_from_rows<U, V, false>(feats, map_coords, table, capacity, d, cells, dense, s);
    });
  });
  if (rc != MEB200_OK) return rc;
  MEB_LAUNCH_OK();
  return MEB200_OK;
}

int meb200_dense_to_rows(const void *dense, int dtype, const meb200_dense_desc *desc,
                         const int32_t *coords, uint32_t n, void *out, void *stream) {
  uint64_t cells;
  int rc = check_desc(desc, &cells);
  if (rc != MEB200_OK) return rc;
  const meb200_dense_desc &d = *desc;
  if (n == 0 || d.channels == 0) return MEB200_OK;
  MEB_CHECK_ARG(coords && out && (dense || cells == 0), "null buffer");
  cudaStream_t s = (cudaStream_t)stream;
  MEB_DISPATCH_DTYPE(dtype, {
    using U = word_t<T>;
    bool dv = dense_vectorises(dense, d, sizeof(T));
    MEB_DISPATCH_VEC(T, d.channels, aligned(16, (const char *)out), {
      k_dense_to_rows<U, V><<<cdiv((uint64_t)n * (d.channels / V), kDenseThreads), kDenseThreads, 0, s>>>(
          (const U *)dense, d, dv && V > 1, coords, n, d.channels, (U *)out);
    });
  });
  MEB_LAUNCH_OK();
  return MEB200_OK;
}

uint64_t meb200_dense_nonzero_scratch_bytes(uint64_t cells) {
  uint64_t tiles = nz_tiles(cells);
  return tiles * kNzTile + 4ull * (tiles + 2);
}

int meb200_dense_nonzero_count(const void *dense, int dtype, const meb200_dense_desc *desc,
                               void *scratch, uint32_t *h_count, void *stream) {
  uint64_t cells;
  int rc = check_desc(desc, &cells);
  if (rc != MEB200_OK) return rc;
  const meb200_dense_desc &d = *desc;
  MEB_CHECK_ARG(h_count != nullptr, "h_count");
  *h_count = 0;
  if (cells == 0) return MEB200_OK;
  MEB_CHECK_ARG(cells <= 0xFFFFFFFFull - kNzTile, "more cells than a coordinate map has rows");
  MEB_CHECK_ARG(scratch && (dense || d.channels == 0), "null buffer");
  cudaStream_t s = (cudaStream_t)stream;
  NonzeroScratch sc = nz_carve(scratch, cells);
  unsigned tiles = nz_tiles(cells);
  MEB_DISPATCH_DTYPE(dtype, {
    using U = word_t<T>;
    bool dv = dense_vectorises(dense, d, sizeof(T));
    constexpr int V = 16 / sizeof(T);
    k_nonzero_flag<U, V><<<tiles, kDenseThreads, 0, s>>>((const U *)dense, d, dv, (uint32_t)cells, sc);
  });
  MEB_LAUNCH_OK();
  k_nonzero_scan<<<1, kDenseThreads, 0, s>>>(tiles, sc);
  MEB_LAUNCH_OK();
  MEB_CUDA(cudaMemcpyAsync(h_count, sc.total, 4, cudaMemcpyDeviceToHost, s));
  MEB_CUDA(cudaStreamSynchronize(s));
  return MEB200_OK;
}

int meb200_dense_nonzero_coords(const meb200_dense_desc *desc, void *scratch, int32_t *coords,
                                void *stream) {
  uint64_t cells;
  int rc = check_desc(desc, &cells);
  if (rc != MEB200_OK) return rc;
  if (cells == 0) return MEB200_OK;
  MEB_CHECK_ARG(cells <= 0xFFFFFFFFull - kNzTile, "more cells than a coordinate map has rows");
  MEB_CHECK_ARG(scratch && coords, "null buffer");
  k_nonzero_fill<<<nz_tiles(cells), kDenseThreads, 0, (cudaStream_t)stream>>>(
      *desc, (uint32_t)cells, nz_carve(scratch, cells), coords);
  MEB_LAUNCH_OK();
  return MEB200_OK;
}

}
