// Shared host/device helpers for the meb200 kernels (sm_90a only).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/meb200.h"

namespace meb200 {

constexpr uint32_t kEmpty = 0xFFFFFFFFu;

// ---- error plumbing ---------------------------------------------------------------
void set_error(const char *fmt, ...);
void count_launch(unsigned n = 1);
void count_tc_launch();
uint64_t tc_launches();

void set_arg_error(const char *file, int line, const char *cond, const char *fmt, ...);

// MEB_CHECK_ARG(cond, "message with %u", value): message arguments are formatted first, the
// location and the failed condition are prepended by set_arg_error.
#define MEB_CHECK_ARG(cond, ...)                                                         \
  do {                                                                                   \
    if (!(cond)) {                                                                       \
      ::meb200::set_arg_error(__FILE__, __LINE__, #cond, __VA_ARGS__);                   \
      return MEB200_ERR_INVALID;                                                         \
    }                                                                                    \
  } while (0)

#define MEB_CUDA(call)                                                                   \
  do {                                                                                   \
    cudaError_t e__ = (call);                                                            \
    if (e__ != cudaSuccess) {                                                            \
      ::meb200::set_error("%s:%d CUDA error %d (%s) in %s", __FILE__, __LINE__,          \
                          (int)e__, cudaGetErrorString(e__), #call);                     \
      return MEB200_ERR_CUDA;                                                            \
    }                                                                                    \
  } while (0)

// Launch-check: catches bad configurations immediately; execution errors surface at the
// caller's next synchronisation, as with any stream-ordered API.
#define MEB_LAUNCH_OK()                                                                  \
  do {                                                                                   \
    ::meb200::count_launch();                                                            \
    MEB_CUDA(cudaGetLastError());                                                        \
  } while (0)

inline unsigned cdiv(uint64_t a, uint64_t b) { return (unsigned)((a + b - 1) / b); }

int num_sms();

// The deduplicating insert behind meb200_insert_and_map (coords.cu).  Its one blocking read copies
// h_words words to the host: the unique count, and with h_words = 2 the word beside it in the
// scratch (insert_flag_word), which kernels enqueued before the insert may set.
int insert_and_map(const int32_t *coords, const uint8_t *valid, uint32_t n, uint32_t ncols,
                   uint32_t *table, uint32_t capacity, int32_t *unique_coords,
                   int64_t *unique_index, int64_t *inverse_map, void *scratch,
                   uint32_t *h_num_unique, uint32_t h_words, cudaStream_t stream);
uint32_t *insert_flag_word(void *scratch, uint32_t n);

// ---- coordinate rows ---------------------------------------------------------------
struct IntVec {  // small by-value parameter block (tensor strides, etc.)
  int32_t v[MEB200_MAX_NCOLS];
};

template <int NC>
struct Coord {
  int32_t c[NC];
};

// Loads one [ncols] row; NC is the compile-time row width.
template <int NC>
__device__ __forceinline__ void load_coord(const int32_t *__restrict__ base, uint32_t row,
                                           int32_t (&c)[NC]) {
  if constexpr (NC == 4) {
    int4 v = __ldg(reinterpret_cast<const int4 *>(base) + row);
    c[0] = v.x; c[1] = v.y; c[2] = v.z; c[3] = v.w;
  } else if constexpr (NC == 2) {
    int2 v = __ldg(reinterpret_cast<const int2 *>(base) + row);
    c[0] = v.x; c[1] = v.y;
  } else {
#pragma unroll
    for (int j = 0; j < NC; ++j) c[j] = __ldg(base + (size_t)row * NC + j);
  }
}

template <int NC>
__device__ __forceinline__ void store_coord(int32_t *__restrict__ base, uint32_t row,
                                            const int32_t (&c)[NC]) {
  if constexpr (NC == 4) {
    reinterpret_cast<int4 *>(base)[row] = make_int4(c[0], c[1], c[2], c[3]);
  } else if constexpr (NC == 2) {
    reinterpret_cast<int2 *>(base)[row] = make_int2(c[0], c[1]);
  } else {
#pragma unroll
    for (int j = 0; j < NC; ++j) base[(size_t)row * NC + j] = c[j];
  }
}

template <int NC>
__device__ __forceinline__ bool coord_eq(const int32_t (&a)[NC], const int32_t (&b)[NC]) {
  bool eq = true;
#pragma unroll
  for (int j = 0; j < NC; ++j) eq &= (a[j] == b[j]);
  return eq;
}

__device__ __forceinline__ uint32_t rotl32(uint32_t x, int r) {
  return (x << r) | (x >> (32 - r));
}

// MurmurHash3_x86_32 over the NC int32 words of a coordinate row, seed 0 — the same
// function the reference hashes coordinates with (src/coordinate.hpp:276-349).
template <int NC>
__device__ __forceinline__ uint32_t hash_coord(const int32_t (&c)[NC]) {
  uint32_t h = 0u;
#pragma unroll
  for (int j = 0; j < NC; ++j) {
    uint32_t k = (uint32_t)c[j];
    k *= 0xcc9e2d51u;
    k = rotl32(k, 15);
    k *= 0x1b873593u;
    h ^= k;
    h = rotl32(h, 13);
    h = h * 5u + 0xe6546b64u;
  }
  h ^= (uint32_t)(NC * 4);
  h ^= h >> 16;
  h *= 0x85ebca6bu;
  h ^= h >> 13;
  h *= 0xc2b2ae35u;
  h ^= h >> 16;
  return h;
}

// Lookup in an open-addressing table of row indices; keys live in `coords`.
template <int NC>
__device__ __forceinline__ int32_t table_find(const int32_t *__restrict__ coords,
                                              const uint32_t *__restrict__ table,
                                              uint32_t mask, const int32_t (&key)[NC]) {
  uint32_t h = hash_coord<NC>(key) & mask;
  while (true) {
    uint32_t cur = __ldg(table + h);
    if (cur == kEmpty) return -1;
    int32_t other[NC];
    load_coord<NC>(coords, cur, other);
    if (coord_eq<NC>(other, key)) return (int32_t)cur;
    h = (h + 1) & mask;
  }
}

// Dispatch a templated-on-NC body over the runtime column count.
#define MEB_DISPATCH_NCOLS(ncols, ...)                                                   \
  switch (ncols) {                                                                       \
    case 2: { constexpr int NC = 2; __VA_ARGS__; } break;                                \
    case 3: { constexpr int NC = 3; __VA_ARGS__; } break;                                \
    case 4: { constexpr int NC = 4; __VA_ARGS__; } break;                                \
    case 5: { constexpr int NC = 5; __VA_ARGS__; } break;                                \
    case 6: { constexpr int NC = 6; __VA_ARGS__; } break;                                \
    case 7: { constexpr int NC = 7; __VA_ARGS__; } break;                                \
    case 8: { constexpr int NC = 8; __VA_ARGS__; } break;                                \
    default:                                                                             \
      ::meb200::set_error("unsupported coordinate width %u (need 2..8)", (unsigned)ncols); \
      return MEB200_ERR_INVALID;                                                         \
  }

// ---- feature element types --------------------------------------------------------
template <typename T> __device__ __forceinline__ float to_f32(T v);
template <> __device__ __forceinline__ float to_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f32<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }
template <> __device__ __forceinline__ float to_f32<__half>(__half v) { return __half2float(v); }

template <typename T> __device__ __forceinline__ T from_f32(float v);
template <> __device__ __forceinline__ float from_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ __nv_bfloat16 from_f32<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }
template <> __device__ __forceinline__ __half from_f32<__half>(float v) { return __float2half_rn(v); }

inline size_t dtype_size(int dt) { return dt == MEB200_F32 ? 4 : 2; }

// Every pointer is a multiple of `bytes` (a null pointer is)
template <typename... P>
inline bool aligned(size_t bytes, const P *...p) {
  return ((reinterpret_cast<uintptr_t>(p) % bytes == 0) && ...);
}

// Elements of elem_bytes each per 16-byte vector when a row of C of them is a whole number of
// such vectors, otherwise 1
inline uint32_t vec_elems(size_t elem_bytes, uint32_t C) {
  return C * elem_bytes % 16 == 0 ? (uint32_t)(16 / elem_bytes) : 1u;
}

// Dispatch a body templated on the feature type T over the runtime dtype.
#define MEB_DISPATCH_DTYPE(dtype, ...)                                                   \
  switch (dtype) {                                                                       \
    case MEB200_F32: { using T = float; __VA_ARGS__; } break;                            \
    case MEB200_BF16: { using T = __nv_bfloat16; __VA_ARGS__; } break;                   \
    case MEB200_F16: { using T = __half; __VA_ARGS__; } break;                           \
    default:                                                                             \
      ::meb200::set_error("unsupported dtype %d", (int)(dtype));                         \
      return MEB200_ERR_UNSUPPORTED;                                                     \
  }

// The same over (input dtype, output dtype), binding T and TO: a feature dtype to itself, or
// bf16 / fp16 to fp32.
#define MEB_DISPATCH_DTYPE_OUT(dtype, out_dtype, ...)                                    \
  if ((out_dtype) == (dtype)) {                                                          \
    MEB_DISPATCH_DTYPE(dtype, using TO = T; __VA_ARGS__);                                \
  } else if ((out_dtype) == MEB200_F32 && (dtype) == MEB200_BF16) {                      \
    using T = __nv_bfloat16; using TO = float; __VA_ARGS__;                              \
  } else if ((out_dtype) == MEB200_F32 && (dtype) == MEB200_F16) {                       \
    using T = __half; using TO = float; __VA_ARGS__;                                     \
  } else {                                                                               \
    ::meb200::set_error("unsupported dtypes in=%d out=%d", (int)(dtype), (int)(out_dtype)); \
    return MEB200_ERR_UNSUPPORTED;                                                       \
  }

// Dispatch a body templated on V, the elements of T per access, over a row of C elements:
// V = 16 / sizeof(T) when the row is a whole number of 16-byte vectors and `is_aligned` (the
// pointers the kernel vectorises are 16-byte aligned), V = 1 otherwise.
#define MEB_DISPATCH_VEC(T, C, is_aligned, ...)                                          \
  if (::meb200::vec_elems(sizeof(T), C) > 1 && (is_aligned)) {                           \
    constexpr int V = 16 / sizeof(T); __VA_ARGS__;                                       \
  } else {                                                                               \
    constexpr int V = 1; __VA_ARGS__;                                                    \
  }

// ---- deterministic split reduction -------------------------------------------------------
// A weight gradient reduced over row splits stores each split's partial sums in its own slot of
// the caller's workspace, then launch_split_sum adds the slots in split order: no atomics, so
// results are bit-identical run to run.  With one split the kernel writes dW directly.

// Splits to run of the `planned` ones, with slots of slot_bytes: as many as the workspace holds,
// at least one; one when the workspace is null or not 16-byte aligned.
uint32_t workspace_splits(uint32_t planned, const void *workspace, uint64_t workspace_bytes,
                          uint64_t slot_bytes);

// dW[i] = part[i] + part[n + i] + ... + part[(splits - 1) n + i], added in that order
int launch_split_sum(const float *part, float *dW, size_t n, uint32_t splits, cudaStream_t stream);

// V elements of T per access: 16 bytes when V = 16 / sizeof(T), one element when V = 1
template <typename T, int V>
__device__ __forceinline__ void load_f32(const T *p, float (&f)[V]) {
  if constexpr (V == 1) {
    f[0] = to_f32<T>(*p);
  } else {
    static_assert(V * sizeof(T) == 16, "16-byte vectors");
    uint4 v = __ldg(reinterpret_cast<const uint4 *>(p));
    const T *e = reinterpret_cast<const T *>(&v);
#pragma unroll
    for (int j = 0; j < V; ++j) f[j] = to_f32<T>(e[j]);
  }
}

template <typename T, int V>
__device__ __forceinline__ void store_f32(T *p, const float (&f)[V]) {
  if constexpr (V == 1) {
    *p = from_f32<T>(f[0]);
  } else {
    uint4 v;
    T *e = reinterpret_cast<T *>(&v);
#pragma unroll
    for (int j = 0; j < V; ++j) e[j] = from_f32<T>(f[j]);
    *reinterpret_cast<uint4 *>(p) = v;
  }
}

}  // namespace meb200
