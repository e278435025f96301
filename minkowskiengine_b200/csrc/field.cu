// Tensor fields: quantisation of float point coordinates to voxels, the reductions from points to
// voxels and back, and multilinear interpolation.
//
// Reference semantics: CoordinateFieldMapCPU::quantize_coordinates (coordinate_map_cpu.hpp:994-1037),
// interpolation_map_weight_kernel (:139-240), MinkowskiTensorField.sparse / SparseTensor.slice, the
// SPMM and direct max-pool functions they call (MinkowskiTensorField.py, src/direct_max_pool.cpp)
// and InterpolationForward/BackwardKernelCPU (src/interpolation_cpu.cpp).  The reference scatters
// into zero-filled outputs; here the points are grouped by voxel once (a stable radix sort) and
// every kernel is stationary over the rows it writes: each output element is written once, in a
// fixed order, with fp32 accumulation and one rounding.
#include <cub/device/device_radix_sort.cuh>

#include "common.cuh"

namespace meb200 {

// Voxel of a field point at stride s, as the reference computes it: float division, floorf, the
// product s * floor in float, then the conversion to int32.  *ok is cleared when the coordinate is
// not finite or the voxel is outside int32.
__device__ __forceinline__ int32_t quantize_axis(float x, int32_t s, bool *ok) {
  float fs = (float)s;
  float v = __fmul_rn(fs, floorf(__fdiv_rn(x, fs)));
  bool in = v >= -2147483648.f && v < 2147483648.f;  // false for NaN and +-inf
  *ok &= in;
  return in ? (int32_t)v : 0;
}

template <int NC>
__global__ void __launch_bounds__(256)
k_quantize_field(const float *__restrict__ field, uint32_t n, IntVec ts, int32_t *__restrict__ out,
                 uint32_t *__restrict__ bad) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float *p = field + (size_t)i * NC;
  bool ok = true;
  int32_t c[NC];
  c[0] = quantize_batch(__ldg(p), &ok);
#pragma unroll
  for (int j = 1; j < NC; ++j) c[j] = quantize_axis(__ldg(p + j), ts.v[j - 1], &ok);
  store_coord<NC>(out, i, c);
  if (!ok && bad != nullptr) atomicOr(bad, 1u);  // a flag, not a sum: any order, same word
}

// ---- grouping by key ----------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_group_keys(const int32_t *__restrict__ keys, uint32_t P, uint32_t M, uint32_t *__restrict__ k_out,
             int32_t *__restrict__ v_out) {
  uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= P) return;
  int32_t k = __ldg(keys + j);
  k_out[j] = (k < 0 || (uint32_t)k >= M) ? M : (uint32_t)k;  // left-out entries sort last
  v_out[j] = (int32_t)j;
}

// start[r] = first sorted position whose key is >= r, for r in [0, M]: one thread per row, a binary
// search over the sorted keys (O(log P) per row, however the keys are spread over the rows).
__global__ void __launch_bounds__(256)
k_group_starts(const uint32_t *__restrict__ sorted, uint32_t P, uint32_t M,
               int32_t *__restrict__ start) {
  uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r > M) return;
  uint32_t lo = 0, hi = P;
  while (lo < hi) {
    uint32_t mid = lo + (hi - lo) / 2;
    if (__ldg(sorted + mid) < r) lo = mid + 1;
    else hi = mid;
  }
  start[r] = (int32_t)lo;
}

static int key_bits(uint32_t M) {
  int b = 1;
  while (b < 32 && (M >> b) != 0) ++b;
  return b;
}

static size_t cub_temp_bytes(uint32_t P, uint32_t M) {
  size_t bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, bytes, (const uint32_t *)nullptr, (uint32_t *)nullptr,
                                  (const int32_t *)nullptr, (int32_t *)nullptr, (int)P, 0,
                                  key_bits(M));
  return bytes;
}

static size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

// ---- points -> voxels ---------------------------------------------------------------------------
template <typename T, int V, int MODE, bool WEIGHTED>
__global__ void __launch_bounds__(256)
k_field_reduce(const T *__restrict__ src, uint32_t C, const int32_t *__restrict__ perm,
               const int32_t *__restrict__ start, uint32_t M, const float *__restrict__ weight,
               const int32_t *__restrict__ src_row, uint32_t src_div, T *__restrict__ out,
               int32_t *__restrict__ argmax) {
  uint32_t CV = C / V;
  uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (uint64_t)M * CV) return;
  uint32_t r = (uint32_t)(t / CV), c = (uint32_t)(t % CV) * V;
  int32_t b = __ldg(start + r), e = __ldg(start + r + 1);
  float acc[V];
  int32_t arg[V];
#pragma unroll
  for (int v = 0; v < V; ++v) {
    acc[v] = 0.f;
    arg[v] = -1;
  }
  for (int32_t j = b; j < e; ++j) {
    uint32_t p = (uint32_t)__ldg(perm + j);
    uint32_t s = src_row != nullptr ? (uint32_t)__ldg(src_row + p) : p / src_div;
    float x[V];
    load_f32<T, V>(src + (size_t)s * C + c, x);
    if (WEIGHTED) {
      float w = __ldg(weight + p);
#pragma unroll
      for (int v = 0; v < V; ++v) x[v] = __fmul_rn(x[v], w);
    }
#pragma unroll
    for (int v = 0; v < V; ++v) {
      if (MODE == MEB200_FIELD_MAX) {
        if (j == b || x[v] > acc[v]) {  // strict: the first point of the voxel wins a tie
          acc[v] = x[v];
          arg[v] = (int32_t)p;
        }
      } else {
        acc[v] = __fadd_rn(acc[v], x[v]);
      }
    }
  }
  if (MODE == MEB200_FIELD_AVG && e > b) {
    float cnt = (float)(e - b);
#pragma unroll
    for (int v = 0; v < V; ++v) acc[v] = __fdiv_rn(acc[v], cnt);
  }
  store_f32<T, V>(out + (size_t)r * C + c, acc);
  if (MODE == MEB200_FIELD_MAX) {
#pragma unroll
    for (int v = 0; v < V; ++v) argmax[(size_t)r * C + c + v] = arg[v];
  }
}

// Status bits of a pair list: 1 = a row outside [0, n_rows), 2 = a column outside [0, n_cols).
__global__ void __launch_bounds__(256)
k_check_pairs(const int32_t *__restrict__ rows, const int32_t *__restrict__ cols, uint32_t P,
              uint32_t n_rows, uint32_t n_cols, uint32_t *__restrict__ bad) {
  uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  uint32_t status = ((uint32_t)__ldg(rows + p) >= n_rows ? 1u : 0u) |
                    ((uint32_t)__ldg(cols + p) >= n_cols ? 2u : 0u);  // negatives wrap past the end
  if (status != 0) atomicOr(bad, status);  // flags, not a sum: any order, same word
}

// The MAX argmax (the winning entry, -1 for none) as the flat index src_row[entry] * C + c of a
// [n_src, C] input.
template <typename I>
__global__ void __launch_bounds__(256)
k_flat_mask(const int32_t *__restrict__ argmax, const int32_t *__restrict__ src_row, uint64_t n,
            uint32_t C, I *__restrict__ mask) {
  uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  int32_t a = __ldg(argmax + t);
  mask[t] = a < 0 ? (I)-1 : (I)__ldg(src_row + a) * (I)C + (I)(t % C);
}

// ---- voxels -> points ---------------------------------------------------------------------------
template <typename T, int V, int MODE>
__global__ void __launch_bounds__(256)
k_field_expand(const T *__restrict__ g, uint32_t M, uint32_t C, const int64_t *__restrict__ inv,
               uint32_t n, const int32_t *__restrict__ start, const int32_t *__restrict__ argmax,
               const int64_t *__restrict__ unique_index, T *__restrict__ out) {
  uint32_t CV = C / V;
  uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (uint64_t)n * CV) return;
  uint32_t i = (uint32_t)(t / CV), c = (uint32_t)(t % CV) * V;
  int64_t r = __ldg(inv + i);
  float x[V];
  if (r < 0 || r >= (int64_t)M) {
#pragma unroll
    for (int v = 0; v < V; ++v) x[v] = 0.f;
  } else {
    load_f32<T, V>(g + (size_t)r * C + c, x);
    if (MODE == MEB200_FIELD_AVG) {
      float inv_cnt = __frcp_rn((float)(__ldg(start + r + 1) - __ldg(start + r)));
#pragma unroll
      for (int v = 0; v < V; ++v) x[v] = __fmul_rn(x[v], inv_cnt);
    } else if (MODE == MEB200_FIELD_MAX) {
#pragma unroll
      for (int v = 0; v < V; ++v)
        if (__ldg(argmax + (size_t)r * C + c + v) != (int32_t)i) x[v] = 0.f;
    } else {  // SUBSAMPLE
      if (__ldg(unique_index + r) != (int64_t)i) {
#pragma unroll
        for (int v = 0; v < V; ++v) x[v] = 0.f;
      }
    }
  }
  store_f32<T, V>(out + (size_t)i * C + c, x);
}

// ---- interpolation ------------------------------------------------------------------------------
template <int NC>
__global__ void __launch_bounds__(256)
k_interp_map(const float *__restrict__ query, uint32_t n, IntVec ts,
             const int32_t *__restrict__ map_coords, const uint32_t *__restrict__ table,
             uint32_t mask, int32_t *__restrict__ rows, float *__restrict__ weights) {
  constexpr uint32_t K = 1u << (NC - 1);
  uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (uint64_t)n * K) return;
  uint32_t q = (uint32_t)(t / K), k = (uint32_t)(t % K);
  const float *p = query + (size_t)q * NC;
  bool ok = true;
  int32_t c[NC];
  float x[NC];
  c[0] = quantize_batch(__ldg(p), &ok);
#pragma unroll
  for (int j = 1; j < NC; ++j) {
    x[j] = __ldg(p + j);
    c[j] = quantize_axis(x[j], ts.v[j - 1], &ok);
    if ((k >> (NC - 1 - j)) & 1u) {  // the upper end of axis j
      int64_t u = (int64_t)c[j] + ts.v[j - 1];
      ok &= u <= 2147483647ll;
      c[j] = (int32_t)u;
    }
  }
  int32_t row = ok ? table_find<NC>(map_coords, table, mask, c) : -1;
  float w = 0.f;
  if (row >= 0) {
    w = 1.f;
#pragma unroll
    for (int j = 1; j < NC; ++j)
      w = __fmul_rn(w, __fsub_rn(1.f, __fdiv_rn(fabsf(__fsub_rn(x[j], (float)c[j])),
                                                (float)ts.v[j - 1])));
  }
  rows[t] = row;
  weights[t] = w;
}

// Splat corners: for point q and corner k, floorf of every column (the batch column included, as
// the reference's create_splat_coordinates floors it) plus 1 on axis j when bit NC-1-j of k is set
// (the corner order of k_interp_map).  Status bits: 1 = a coordinate is not finite or a corner is
// outside int32, 2 = a batch value is not an integer (k_interp_map rounds it, so its corners would
// be missed).
template <int NC>
__global__ void __launch_bounds__(256)
k_splat_coords(const float *__restrict__ field, uint32_t n, int32_t *__restrict__ out,
               uint32_t *__restrict__ bad) {
  constexpr uint32_t K = 1u << (NC - 1);
  uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (uint64_t)n * K) return;
  uint32_t q = (uint32_t)(t / K), k = (uint32_t)(t % K);
  const float *p = field + (size_t)q * NC;
  uint32_t status = 0;
  int32_t c[NC];
#pragma unroll
  for (int j = 0; j < NC; ++j) {
    float x = __ldg(p + j);
    float f = floorf(x);
    int64_t up = (j > 0 && ((k >> (NC - 1 - j)) & 1u)) ? 1 : 0;
    bool in = f >= -2147483648.f && f < 2147483648.f;  // false for NaN and +-inf
    int64_t v = in ? (int64_t)f + up : 0;
    if (!in || v > 2147483647ll) status |= 1u;
    if (j == 0 && in && f != x) status |= 2u;
    c[j] = (int32_t)v;
  }
  store_coord<NC>(out, (uint32_t)t, c);
  if (status != 0) atomicOr(bad, status);  // flags, not a sum: any order, same word
}

template <typename T, int V>
__global__ void __launch_bounds__(256)
k_interp_fwd(const T *__restrict__ F, uint32_t C, const int32_t *__restrict__ rows,
             const float *__restrict__ weights, uint32_t n, uint32_t K, T *__restrict__ out) {
  uint32_t CV = C / V;
  uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (uint64_t)n * CV) return;
  uint32_t q = (uint32_t)(t / CV), c = (uint32_t)(t % CV) * V;
  float acc[V];
#pragma unroll
  for (int v = 0; v < V; ++v) acc[v] = 0.f;
  for (uint32_t k = 0; k < K; ++k) {
    int32_t r = __ldg(rows + (size_t)q * K + k);
    if (r < 0) continue;
    float w = __ldg(weights + (size_t)q * K + k);
    float x[V];
    load_f32<T, V>(F + (size_t)r * C + c, x);
#pragma unroll
    for (int v = 0; v < V; ++v) acc[v] = __fadd_rn(acc[v], __fmul_rn(w, x[v]));
  }
  store_f32<T, V>(out + (size_t)q * C + c, acc);
}

// ---- host dispatch ------------------------------------------------------------------------------
template <typename T, int V>
static void reduce_launch(const void *src, uint32_t C, const int32_t *perm, const int32_t *start,
                          uint32_t M, const float *weight, const int32_t *src_row, uint32_t src_div,
                          int mode, void *out, int32_t *argmax, cudaStream_t st) {
  unsigned blocks = cdiv((uint64_t)M * (C / V), 256);
  const T *s = (const T *)src;
  T *o = (T *)out;
#define MEB_REDUCE(MODE, W)                                                                 \
  k_field_reduce<T, V, MODE, W><<<blocks, 256, 0, st>>>(s, C, perm, start, M, weight, src_row, \
                                                        src_div, o, argmax)
  if (mode == MEB200_FIELD_MAX) {
    MEB_REDUCE(MEB200_FIELD_MAX, false);
  } else if (mode == MEB200_FIELD_AVG) {
    MEB_REDUCE(MEB200_FIELD_AVG, false);
  } else if (weight != nullptr) {
    MEB_REDUCE(MEB200_FIELD_SUM, true);
  } else {
    MEB_REDUCE(MEB200_FIELD_SUM, false);
  }
#undef MEB_REDUCE
}

template <typename T, int V>
static void expand_launch(const void *g, uint32_t M, uint32_t C, const int64_t *inv, uint32_t n,
                          int mode, const int32_t *start, const int32_t *argmax,
                          const int64_t *uidx, void *out, cudaStream_t st) {
  unsigned blocks = cdiv((uint64_t)n * (C / V), 256);
  const T *gg = (const T *)g;
  T *o = (T *)out;
  if (mode == MEB200_FIELD_AVG)
    k_field_expand<T, V, MEB200_FIELD_AVG><<<blocks, 256, 0, st>>>(gg, M, C, inv, n, start, argmax, uidx, o);
  else if (mode == MEB200_FIELD_MAX)
    k_field_expand<T, V, MEB200_FIELD_MAX><<<blocks, 256, 0, st>>>(gg, M, C, inv, n, start, argmax, uidx, o);
  else
    k_field_expand<T, V, MEB200_FIELD_SUBSAMPLE><<<blocks, 256, 0, st>>>(gg, M, C, inv, n, start, argmax, uidx, o);
}

template <typename T, int V>
static void interp_launch(const void *F, uint32_t C, const int32_t *rows, const float *w, uint32_t n,
                          uint32_t K, void *out, cudaStream_t st) {
  k_interp_fwd<T, V><<<cdiv((uint64_t)n * (C / V), 256), 256, 0, st>>>((const T *)F, C, rows, w, n,
                                                                       K, (T *)out);
}

}  // namespace meb200

using namespace meb200;

extern "C" {

int meb200_quantize_field(const float *field, uint32_t n, uint32_t ncols,
                          const int32_t *tensor_stride, int32_t *out, uint32_t *d_bad,
                          void *stream) {
  MEB_CHECK_ARG(ncols >= 2 && ncols <= MEB200_MAX_NCOLS, "ncols=%u", ncols);
  IntVec ts;
  int rc = load_strides(tensor_stride, ncols, &ts);
  if (rc != MEB200_OK) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  if (d_bad != nullptr) MEB_CUDA(cudaMemsetAsync(d_bad, 0, 4, s));
  if (n == 0) return MEB200_OK;
  MEB_CHECK_ARG(field && out, "null buffer");
  MEB_DISPATCH_NCOLS(ncols, k_quantize_field<NC><<<cdiv(n, 256), 256, 0, s>>>(field, n, ts, out,
                                                                              d_bad));
  MEB_LAUNCH_OK();
  return MEB200_OK;
}

int meb200_field_insert_and_map(const float *field, uint32_t n, uint32_t ncols,
                                const int32_t *tensor_stride, int32_t *qcoords, uint32_t *table,
                                uint32_t capacity, int32_t *unique_coords, int64_t *unique_index,
                                int64_t *inverse_map, void *scratch, uint32_t *h_num_unique,
                                void *stream) {
  MEB_CHECK_ARG(h_num_unique != nullptr, "h_num_unique");
  if (n > 0) {
    MEB_CHECK_ARG(scratch != nullptr, "null scratch");
    int rc = meb200_quantize_field(field, n, ncols, tensor_stride, qcoords,
                                   insert_flag_word(scratch, n), stream);
    if (rc != MEB200_OK) return rc;
  }
  uint32_t h[2] = {0, 0};
  int rc = insert_and_map(qcoords, nullptr, n, ncols, table, capacity, unique_coords,
                          unique_index, inverse_map, scratch, h, n > 0 ? 2 : 1,
                          (cudaStream_t)stream);
  if (rc != MEB200_OK) return rc;
  *h_num_unique = h[0];
  if (h[1] != 0) {
    set_error("a field coordinate is not finite, or its voxel lies outside int32");
    return MEB200_ERR_DOMAIN;
  }
  return MEB200_OK;
}

uint64_t meb200_group_by_row_scratch_bytes(uint32_t P, uint32_t M) {
  return 3 * align256(4ull * P) + align256(cub_temp_bytes(P, M));
}

int meb200_group_by_row(const int32_t *keys, uint32_t P, uint32_t M, int32_t *start, int32_t *perm,
                        void *scratch, uint64_t scratch_bytes, void *stream) {
  MEB_CHECK_ARG(start != nullptr, "null start");
  MEB_CHECK_ARG(M < 0x7FFFFFFFu && P < 0x7FFFFFFFu, "too many rows (%u) or entries (%u)", M, P);
  cudaStream_t s = (cudaStream_t)stream;
  if (P > 0) {
    MEB_CHECK_ARG(keys && perm && scratch, "null buffer");
    MEB_CHECK_ARG(scratch_bytes >= meb200_group_by_row_scratch_bytes(P, M),
                  "scratch of %llu bytes, %llu needed", (unsigned long long)scratch_bytes,
                  (unsigned long long)meb200_group_by_row_scratch_bytes(P, M));
    char *p = (char *)scratch;
    uint32_t *k_in = (uint32_t *)p;
    p += align256(4ull * P);
    uint32_t *k_out = (uint32_t *)p;
    p += align256(4ull * P);
    int32_t *v_in = (int32_t *)p;
    p += align256(4ull * P);
    size_t temp = cub_temp_bytes(P, M);
    k_group_keys<<<cdiv(P, 256), 256, 0, s>>>(keys, P, M, k_in, v_in);
    MEB_LAUNCH_OK();
    MEB_CUDA(cub::DeviceRadixSort::SortPairs(p, temp, k_in, k_out, v_in, perm, (int)P, 0,
                                             key_bits(M), s));
    count_launch();
    k_group_starts<<<cdiv((uint64_t)M + 1, 256), 256, 0, s>>>(k_out, P, M, start);
  } else {
    k_group_starts<<<cdiv((uint64_t)M + 1, 256), 256, 0, s>>>(nullptr, 0, M, start);
  }
  MEB_LAUNCH_OK();
  return MEB200_OK;
}

int meb200_field_reduce(const void *src, int dtype, uint32_t n_src, uint32_t C, const int32_t *perm,
                        const int32_t *start, uint32_t M, const float *weight,
                        const int32_t *src_row, uint32_t src_div, int mode, void *out,
                        int32_t *argmax, void *stream) {
  if (M == 0 || C == 0) return MEB200_OK;
  MEB_CHECK_ARG(mode == MEB200_FIELD_SUM || mode == MEB200_FIELD_AVG || mode == MEB200_FIELD_MAX,
                "mode %d is not a reduction", mode);
  MEB_CHECK_ARG(start && out && (perm || n_src == 0) && (src || n_src == 0), "null buffer");
  MEB_CHECK_ARG(src_div >= 1, "src_div must be positive");
  MEB_CHECK_ARG(mode != MEB200_FIELD_MAX || argmax != nullptr, "MAX needs argmax");
  MEB_CHECK_ARG(weight == nullptr || mode == MEB200_FIELD_SUM, "weights are for SUM only");
  cudaStream_t s = (cudaStream_t)stream;
  MEB_DISPATCH_DTYPE(dtype, MEB_DISPATCH_VEC(T, C, aligned(16, src, out),
                                             reduce_launch<T, V>(src, C, perm, start, M, weight,
                                                                 src_row, src_div, mode, out,
                                                                 argmax, s)));
  MEB_LAUNCH_OK();
  return MEB200_OK;
}

int meb200_check_pairs(const int32_t *rows, const int32_t *cols, uint32_t P, uint32_t n_rows,
                       uint32_t n_cols, uint32_t *d_status, void *stream) {
  if (P == 0) return MEB200_OK;
  MEB_CHECK_ARG(rows && cols && d_status, "null buffer");
  cudaStream_t s = (cudaStream_t)stream;
  MEB_CUDA(cudaMemsetAsync(d_status, 0, 4, s));
  k_check_pairs<<<cdiv(P, 256), 256, 0, s>>>(rows, cols, P, n_rows, n_cols, d_status);
  MEB_LAUNCH_OK();
  uint32_t h = 0;
  MEB_CUDA(cudaMemcpyAsync(&h, d_status, 4, cudaMemcpyDeviceToHost, s));
  MEB_CUDA(cudaStreamSynchronize(s));
  MEB_CHECK_ARG((h & 1u) == 0, "a row index is outside [0, %u)", n_rows);
  MEB_CHECK_ARG((h & 2u) == 0, "a column index is outside [0, %u)", n_cols);
  return MEB200_OK;
}

int meb200_flat_mask(const int32_t *argmax, const int32_t *src_row, uint32_t M, uint32_t C,
                     uint32_t n_src, int index_bits, void *mask, void *stream) {
  MEB_CHECK_ARG(index_bits == 32 || index_bits == 64, "index_bits=%d", index_bits);
  uint64_t flat = (uint64_t)n_src * C;  // the largest index is flat - 1
  MEB_CHECK_ARG(index_bits == 64 || flat <= 0x80000000ull,
                "the flat mask n_src * C = %llu does not fit int32", (unsigned long long)flat);
  uint64_t n = (uint64_t)M * C;
  if (n == 0) return MEB200_OK;
  MEB_CHECK_ARG(argmax && src_row && mask, "null buffer");
  cudaStream_t s = (cudaStream_t)stream;
  if (index_bits == 32)
    k_flat_mask<int32_t><<<cdiv(n, 256), 256, 0, s>>>(argmax, src_row, n, C, (int32_t *)mask);
  else
    k_flat_mask<int64_t><<<cdiv(n, 256), 256, 0, s>>>(argmax, src_row, n, C, (int64_t *)mask);
  MEB_LAUNCH_OK();
  return MEB200_OK;
}

int meb200_field_expand(const void *g, int dtype, uint32_t M, uint32_t C, const int64_t *inv,
                        uint32_t n, int mode, const int32_t *start, const int32_t *argmax,
                        const int64_t *unique_index, void *out, void *stream) {
  if (n == 0 || C == 0) return MEB200_OK;
  MEB_CHECK_ARG(inv && out && (g || M == 0), "null buffer");
  MEB_CHECK_ARG((mode == MEB200_FIELD_AVG && start) || (mode == MEB200_FIELD_MAX && argmax) ||
                    (mode == MEB200_FIELD_SUBSAMPLE && unique_index),
                "mode %d without its table", mode);
  cudaStream_t s = (cudaStream_t)stream;
  MEB_DISPATCH_DTYPE(dtype, MEB_DISPATCH_VEC(T, C, aligned(16, g, out),
                                             expand_launch<T, V>(g, M, C, inv, n, mode, start,
                                                                 argmax, unique_index, out, s)));
  MEB_LAUNCH_OK();
  return MEB200_OK;
}

int meb200_interp_map(const float *query, uint32_t n, uint32_t ncols, const int32_t *tensor_stride,
                      const int32_t *map_coords, const uint32_t *table, uint32_t capacity,
                      int32_t *rows, float *weights, void *stream) {
  MEB_CHECK_ARG(ncols >= 2 && ncols <= MEB200_MAX_NCOLS, "ncols=%u", ncols);
  IntVec ts;
  int rc = load_strides(tensor_stride, ncols, &ts);
  if (rc != MEB200_OK) return rc;
  MEB_CHECK_ARG(capacity >= 2 && (capacity & (capacity - 1)) == 0, "capacity=%u", capacity);
  if (n == 0) return MEB200_OK;
  MEB_CHECK_ARG(query && table && rows && weights, "null buffer");
  uint64_t total = (uint64_t)n << (ncols - 1);
  MEB_CHECK_ARG(total < 0xFFFFFFFFull, "n * 2^D too large");
  cudaStream_t s = (cudaStream_t)stream;
  MEB_DISPATCH_NCOLS(ncols, k_interp_map<NC><<<cdiv(total, 256), 256, 0, s>>>(
                                query, n, ts, map_coords, table, capacity - 1, rows, weights));
  MEB_LAUNCH_OK();
  return MEB200_OK;
}

int meb200_splat_coords(const float *field, uint32_t n, uint32_t ncols, int32_t *out,
                        uint32_t *d_bad, void *stream) {
  MEB_CHECK_ARG(ncols >= 2 && ncols <= MEB200_MAX_NCOLS, "ncols=%u", ncols);
  MEB_CHECK_ARG(d_bad != nullptr, "null status word");
  cudaStream_t s = (cudaStream_t)stream;
  MEB_CUDA(cudaMemsetAsync(d_bad, 0, 4, s));
  if (n == 0) return MEB200_OK;
  MEB_CHECK_ARG(field && out, "null buffer");
  uint64_t total = (uint64_t)n << (ncols - 1);
  MEB_CHECK_ARG(total < 0xFFFFFFFFull, "n * 2^D too large");
  MEB_DISPATCH_NCOLS(ncols, k_splat_coords<NC><<<cdiv(total, 256), 256, 0, s>>>(field, n, out,
                                                                                d_bad));
  MEB_LAUNCH_OK();
  return MEB200_OK;
}

int meb200_interp_forward(const void *F, int dtype, uint32_t M, uint32_t C, const int32_t *rows,
                          const float *weights, uint32_t n, uint32_t K, void *out, void *stream) {
  if (n == 0 || C == 0) return MEB200_OK;
  MEB_CHECK_ARG(rows && weights && out && (F || M == 0), "null buffer");
  cudaStream_t s = (cudaStream_t)stream;
  MEB_DISPATCH_DTYPE(dtype, MEB_DISPATCH_VEC(T, C, aligned(16, F, out),
                                             interp_launch<T, V>(F, C, rows, weights, n, K, out, s)));
  MEB_LAUNCH_OK();
  return MEB200_OK;
}

}
