// Row gather and the union fold: the feature side of pruning, MinkowskiUnion and arithmetic between
// sparse tensors on different coordinate maps.
//
// Reference semantics: PruningForwardKernelCPU / PruningBackwardKernelCPU (src/pruning_cpu.cpp),
// MinkowskiUnionFunction (MinkowskiUnion.py:50-82) and the different-key branch of
// Tensor._binary_functor (MinkowskiTensor.py:522-540).  The reference writes through index_add /
// index assignment into zero-filled outputs; here every kernel is stationary over the rows it
// writes, so each output element is written exactly once, with no memset and no atomics, and the
// results are bit-identical run to run.  Arithmetic is fp32 with one rounding to the output dtype.
#include "common.cuh"

namespace meb200 {

template <int OP>
__device__ __forceinline__ float fold_op(float a, float b) {
  if (OP == MEB200_UNION_ADD) return a + b;
  if (OP == MEB200_UNION_SUB) return a - b;
  if (OP == MEB200_UNION_MUL) return a * b;
  return a / b;
}

// ---- row gather: out[j, :] = idx[j] >= 0 ? src[idx[j], :] : 0 (a copy: W is the access word) ------
template <typename W>
__global__ void __launch_bounds__(256)
k_gather_rows(const W *__restrict__ src, uint32_t n_src, uint32_t CW, const int64_t *__restrict__ idx,
              uint32_t n_out, W *__restrict__ out) {
  uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (uint64_t)n_out * CW) return;
  uint32_t j = (uint32_t)(t / CW), c = (uint32_t)(t % CW);
  int64_t r = __ldg(idx + j);
  W v{};
  if (r >= 0 && r < (int64_t)n_src) v = __ldg(src + (size_t)r * CW + c);
  out[(size_t)j * CW + c] = v;
}

// ---- union fold, forward: stationary over union rows u, inputs in order -------------------------
//   acc = 0; for i with src[i, u] >= 0: acc = (i == 0) ? x_i : op(acc, x_i)
template <typename T, int V, int OP>
__global__ void __launch_bounds__(256)
k_union_fold(const T *const *__restrict__ inputs, uint32_t N, const int32_t *__restrict__ src,
             uint32_t M, uint32_t C, T *__restrict__ out) {
  uint32_t CV = C / V;
  uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (uint64_t)M * CV) return;
  uint32_t u = (uint32_t)(t / CV), c = (uint32_t)(t % CV) * V;
  float acc[V];
#pragma unroll
  for (int j = 0; j < V; ++j) acc[j] = 0.f;
  for (uint32_t i = 0; i < N; ++i) {
    int32_t r = __ldg(src + (size_t)i * M + u);
    if (r < 0) continue;
    float x[V];
    load_f32<T, V>(inputs[i] + (size_t)r * C + c, x);
#pragma unroll
    for (int j = 0; j < V; ++j) acc[j] = i == 0 ? x[j] : fold_op<OP>(acc[j], x[j]);
  }
  store_f32<T, V>(out + (size_t)u * C + c, acc);
}

// ---- union fold, backward: stationary over the rows r of input i, u = u_i[r] ---------------------
//   ADD: g   SUB: i == 0 ? g : -g
//   MUL: g * prod_{j != i present} x_j, 0 when i > 0 and input 0 lacks u (0 * x_i * ...)
//   DIV: i == 0: g / x_1 / x_2 ...;  i > 0: -g * (out / x_i)  (torch's a / b backward for N = 2)
template <typename T, int V, int OP>
__global__ void __launch_bounds__(256)
k_union_fold_bwd(const T *const *__restrict__ inputs, uint32_t N, const int32_t *__restrict__ src,
                 uint32_t M, uint32_t C, const T *__restrict__ g, uint32_t i,
                 const int64_t *__restrict__ u_i, uint32_t n_i, T *__restrict__ grad) {
  uint32_t CV = C / V;
  uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (uint64_t)n_i * CV) return;
  uint32_t r = (uint32_t)(t / CV), c = (uint32_t)(t % CV) * V;
  uint32_t u = (uint32_t)__ldg(u_i + r);
  float y[V];
  load_f32<T, V>(g + (size_t)u * C + c, y);
  if (OP == MEB200_UNION_SUB) {
    if (i > 0) {
#pragma unroll
      for (int j = 0; j < V; ++j) y[j] = -y[j];
    }
  } else if (OP == MEB200_UNION_MUL) {
    if (i > 0 && __ldg(src + u) < 0) {
#pragma unroll
      for (int j = 0; j < V; ++j) y[j] = 0.f;
    } else {
      float p[V];
#pragma unroll
      for (int j = 0; j < V; ++j) p[j] = 1.f;
      for (uint32_t k = 0; k < N; ++k) {
        int32_t rk = __ldg(src + (size_t)k * M + u);
        if (k == i || rk < 0) continue;
        float x[V];
        load_f32<T, V>(inputs[k] + (size_t)rk * C + c, x);
#pragma unroll
        for (int j = 0; j < V; ++j) p[j] *= x[j];
      }
#pragma unroll
      for (int j = 0; j < V; ++j) y[j] *= p[j];
    }
  } else if (OP == MEB200_UNION_DIV) {
    if (i == 0) {
      for (uint32_t k = 1; k < N; ++k) {
        int32_t rk = __ldg(src + (size_t)k * M + u);
        if (rk < 0) continue;
        float x[V];
        load_f32<T, V>(inputs[k] + (size_t)rk * C + c, x);
#pragma unroll
        for (int j = 0; j < V; ++j) y[j] /= x[j];
      }
    } else {
      float acc[V], xi[V];
#pragma unroll
      for (int j = 0; j < V; ++j) acc[j] = 0.f;
      for (uint32_t k = 0; k < N; ++k) {
        int32_t rk = __ldg(src + (size_t)k * M + u);
        if (rk < 0) continue;
        float x[V];
        load_f32<T, V>(inputs[k] + (size_t)rk * C + c, x);
#pragma unroll
        for (int j = 0; j < V; ++j) {
          acc[j] = k == 0 ? x[j] : acc[j] / x[j];
          if (k == i) xi[j] = x[j];
        }
      }
#pragma unroll
      for (int j = 0; j < V; ++j) y[j] = -y[j] * (acc[j] / xi[j]);
    }
  }
  store_f32<T, V>(grad + (size_t)r * C + c, y);
}

// ---- host dispatch ---------------------------------------------------------------------------
template <typename T, int V>
static void fold_launch(const void *const *inputs, uint32_t N, const int32_t *src, uint32_t M,
                        uint32_t C, int op, void *out, cudaStream_t st) {
  unsigned blocks = cdiv((uint64_t)M * (C / V), 256);
  const T *const *in = (const T *const *)inputs;
  switch (op) {
    case MEB200_UNION_ADD: k_union_fold<T, V, MEB200_UNION_ADD><<<blocks, 256, 0, st>>>(in, N, src, M, C, (T *)out); break;
    case MEB200_UNION_SUB: k_union_fold<T, V, MEB200_UNION_SUB><<<blocks, 256, 0, st>>>(in, N, src, M, C, (T *)out); break;
    case MEB200_UNION_MUL: k_union_fold<T, V, MEB200_UNION_MUL><<<blocks, 256, 0, st>>>(in, N, src, M, C, (T *)out); break;
    default: k_union_fold<T, V, MEB200_UNION_DIV><<<blocks, 256, 0, st>>>(in, N, src, M, C, (T *)out); break;
  }
}

template <typename T, int V>
static void fold_bwd_launch(const void *const *inputs, uint32_t N, const int32_t *src, uint32_t M,
                            uint32_t C, int op, const void *g, uint32_t i, const int64_t *u_i,
                            uint32_t n_i, void *grad, cudaStream_t st) {
  unsigned blocks = cdiv((uint64_t)n_i * (C / V), 256);
  const T *const *in = (const T *const *)inputs;
#define MEB_FOLD_BWD(OP)                                                                           \
  k_union_fold_bwd<T, V, OP><<<blocks, 256, 0, st>>>(in, N, src, M, C, (const T *)g, i, u_i, n_i, \
                                                     (T *)grad)
  switch (op) {
    case MEB200_UNION_ADD: MEB_FOLD_BWD(MEB200_UNION_ADD); break;
    case MEB200_UNION_SUB: MEB_FOLD_BWD(MEB200_UNION_SUB); break;
    case MEB200_UNION_MUL: MEB_FOLD_BWD(MEB200_UNION_MUL); break;
    default: MEB_FOLD_BWD(MEB200_UNION_DIV); break;
  }
#undef MEB_FOLD_BWD
}

}  // namespace meb200

using namespace meb200;

extern "C" {

int meb200_gather_rows(const void *src, int dtype, uint32_t n_src, uint32_t C, const int64_t *idx,
                       uint32_t n_out, void *out, void *stream) {
  if (n_out == 0 || C == 0) return MEB200_OK;
  MEB_CHECK_ARG(dtype == MEB200_F32 || dtype == MEB200_BF16 || dtype == MEB200_F16,
                "unsupported dtype %d", dtype);
  MEB_CHECK_ARG(idx && out && (src || n_src == 0), "null buffer");
  cudaStream_t s = (cudaStream_t)stream;
  size_t row = (size_t)C * dtype_size(dtype);
  if (row % 16 == 0 && aligned(16, src, out)) {
    uint32_t CW = (uint32_t)(row / 16);
    k_gather_rows<uint4><<<cdiv((uint64_t)n_out * CW, 256), 256, 0, s>>>(
        (const uint4 *)src, n_src, CW, idx, n_out, (uint4 *)out);
  } else if (dtype == MEB200_F32) {
    k_gather_rows<uint32_t><<<cdiv((uint64_t)n_out * C, 256), 256, 0, s>>>(
        (const uint32_t *)src, n_src, C, idx, n_out, (uint32_t *)out);
  } else {
    k_gather_rows<uint16_t><<<cdiv((uint64_t)n_out * C, 256), 256, 0, s>>>(
        (const uint16_t *)src, n_src, C, idx, n_out, (uint16_t *)out);
  }
  MEB_LAUNCH_OK();
  return MEB200_OK;
}

int meb200_union_fold_forward(const void *const *inputs, uint32_t N, uint32_t inputs_align,
                              const int32_t *src, uint32_t M, uint32_t C, int dtype, int op,
                              void *out, void *stream) {
  if (M == 0 || C == 0) return MEB200_OK;
  MEB_CHECK_ARG(op >= MEB200_UNION_ADD && op <= MEB200_UNION_DIV, "op %d is not a fold", op);
  MEB_CHECK_ARG(N >= 1 && inputs && src && out, "null buffer");
  cudaStream_t s = (cudaStream_t)stream;
  MEB_DISPATCH_DTYPE(dtype, MEB_DISPATCH_VEC(T, C, inputs_align % 16 == 0 && aligned(16, out),
                                             fold_launch<T, V>(inputs, N, src, M, C, op, out, s)));
  MEB_LAUNCH_OK();
  return MEB200_OK;
}

int meb200_union_fold_backward(const void *const *inputs, uint32_t N, uint32_t inputs_align,
                               const int32_t *src, uint32_t M, uint32_t C, int dtype, int op,
                               const void *grad_out, uint32_t i, const int64_t *u_i, uint32_t n_i,
                               void *grad_i, void *stream) {
  if (n_i == 0 || C == 0) return MEB200_OK;
  MEB_CHECK_ARG(op >= MEB200_UNION_ADD && op <= MEB200_UNION_DIV, "op %d is not a fold", op);
  MEB_CHECK_ARG(i < N, "input %u of %u", i, N);
  MEB_CHECK_ARG(inputs && src && grad_out && u_i && grad_i, "null buffer");
  cudaStream_t s = (cudaStream_t)stream;
  MEB_DISPATCH_DTYPE(dtype,
                     MEB_DISPATCH_VEC(T, C, inputs_align % 16 == 0 && aligned(16, grad_out, grad_i),
                                      fold_bwd_launch<T, V>(inputs, N, src, M, C, op, grad_out, i,
                                                            u_i, n_i, grad_i, s)));
  MEB_LAUNCH_OK();
  return MEB200_OK;
}

}
