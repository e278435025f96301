// Channel-wise (depthwise) sparse convolution over the k-major neighbour tables.
//
// Reference semantics: MinkowskiChannelwiseConvolution.forward
// (MinkowskiEngine/MinkowskiChannelwiseConvolution.py:142-191): out[o] += in[i] * kernel[k] for every
// pair (i, o) of offset k, one torch launch per offset, backward by autograd.  Here:
//   k_chwise_gather   y[r, c] = sum_k W[k, c] * x[nbr[k, r], c]   (forward: nbr = out_nbr;
//                     input gradient: nbr = in_nbr, x = the output gradient, the same W)
//   k_chwise_wgrad    dW[k, c] = sum_o x[out_nbr[k, o], c] * g[o, c]
// Every output element is written once, accumulated in fp32 (one fma per term, ascending k in the
// gather, a fixed row order in the wgrad) and rounded once; no atomics, bit-identical run to run.
#include <algorithm>

#include "common.cuh"

namespace meb200 {

constexpr int CW_SK = 8;       // offsets whose table entries are in flight ahead of the row loads
constexpr int CW_ROWS = 4;     // rows per wgrad thread iteration (independent loads in flight)
constexpr int CW_THREADS = 256;

// V fp32 weights of offset k at channel c: 16-byte loads on the vector path
template <int V>
__device__ __forceinline__ void load_w(const float *__restrict__ p, float (&w)[V]) {
  if constexpr (V == 1) {
    w[0] = __ldg(p);
  } else {
#pragma unroll
    for (int j = 0; j < V / 4; ++j) {
      const float4 q = __ldg(reinterpret_cast<const float4 *>(p) + j);
      w[4 * j + 0] = q.x; w[4 * j + 1] = q.y; w[4 * j + 2] = q.z; w[4 * j + 3] = q.w;
    }
  }
}

// One thread per (row, V-channel vector); consecutive threads take consecutive vectors of a row, so
// a warp reads whole gathered rows.  Offsets are walked in batches of CW_SK: the table entries of
// the NEXT batch and the rows of THIS batch are issued before the FMAs (as k_conv_small_cin_fwd
// does), so a thread has up to 2 * CW_SK independent loads outstanding instead of a dependent
// (index -> row) chain per offset.  W is read through L1: K * C fp32 (up to 700 KB at K = 343,
// C = 512) does not fit shared memory, and a CTA only reads the few vectors of W its rows share.
template <typename T, int V>
__global__ void __launch_bounds__(CW_THREADS)
k_chwise_gather(const T *__restrict__ x, uint32_t C, const float *__restrict__ W,
                const int32_t *__restrict__ nbr, uint32_t K, uint32_t n_rows, T *__restrict__ y) {
  const uint32_t vpr = C / V;
  const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (uint64_t)n_rows * vpr) return;
  const uint32_t r = (uint32_t)(t / vpr), c = (uint32_t)(t % vpr) * V;
  const int32_t *col = nbr + r;
  float acc[V];
#pragma unroll
  for (int j = 0; j < V; ++j) acc[j] = 0.f;
  int32_t idx[CW_SK];
#pragma unroll
  for (int j = 0; j < CW_SK; ++j) idx[j] = (uint32_t)j < K ? __ldg(col + (size_t)j * n_rows) : -1;
  for (uint32_t k0 = 0; k0 < K; k0 += CW_SK) {
    int32_t nxt[CW_SK];
#pragma unroll
    for (int j = 0; j < CW_SK; ++j) {
      const uint32_t kk = k0 + CW_SK + j;
      nxt[j] = kk < K ? __ldg(col + (size_t)kk * n_rows) : -1;
    }
    float xv[CW_SK][V];
#pragma unroll
    for (int j = 0; j < CW_SK; ++j) {
      if (idx[j] >= 0) {
        load_f32<T, V>(x + (size_t)idx[j] * C + c, xv[j]);
      } else {
#pragma unroll
        for (int v = 0; v < V; ++v) xv[j][v] = 0.f;
      }
    }
#pragma unroll
    for (int j = 0; j < CW_SK; ++j) {
      if (idx[j] < 0) continue;
      float w[V];
      load_w<V>(W + (size_t)(k0 + j) * C + c, w);
#pragma unroll
      for (int v = 0; v < V; ++v) acc[v] = fmaf(w[v], xv[j][v], acc[v]);
    }
#pragma unroll
    for (int j = 0; j < CW_SK; ++j) idx[j] = nxt[j];
  }
  store_f32<T, V>(y + (size_t)r * C + c, acc);
}

// CTA <-> (offset k = blockIdx.x, row split = blockIdx.y, channel slab = blockIdx.z); threads are
// (vector lane x < S of the slab, row lane y < R), S * R = CW_THREADS.  Row lane y takes the rows
// r_begin + y, r_begin + y + R, ... of the split in ascending order, CW_ROWS at a time, from the
// dense table column out_nbr[k]: the table the forward reads, so the wgrad needs nothing built for
// it.  The R lanes are then folded in ascending y, and the sum is stored to the split's slot
// part[split][k][c] (dW itself with one split); launch_split_sum adds the slots in split order.
template <typename T, int V>
__global__ void __launch_bounds__(CW_THREADS)
k_chwise_wgrad(const T *__restrict__ x, const T *__restrict__ g, uint32_t C,
               const int32_t *__restrict__ out_nbr, uint32_t K, uint32_t n_out,
               uint32_t rows_per_split, float *__restrict__ part) {
  __shared__ float red[CW_THREADS * V];
  const uint32_t S = blockDim.x, R = blockDim.y;
  const uint32_t k = blockIdx.x, split = blockIdx.y;
  const uint32_t vec = blockIdx.z * S + threadIdx.x;
  const bool live = vec < C / V;
  const uint32_t c = vec * V;
  const uint32_t r_begin = split * rows_per_split;
  const uint32_t r_end = min(r_begin + rows_per_split, n_out);
  const int32_t *col = out_nbr + (size_t)k * n_out;
  float acc[V];
#pragma unroll
  for (int j = 0; j < V; ++j) acc[j] = 0.f;
  if (live) {
    for (uint32_t o0 = r_begin + threadIdx.y; o0 < r_end; o0 += CW_ROWS * R) {
      int32_t idx[CW_ROWS];
#pragma unroll
      for (int u = 0; u < CW_ROWS; ++u) {
        const uint32_t o = o0 + u * R;
        idx[u] = o < r_end ? __ldg(col + o) : -1;
      }
      float xv[CW_ROWS][V], gv[CW_ROWS][V];
#pragma unroll
      for (int u = 0; u < CW_ROWS; ++u) {
        if (idx[u] >= 0) {
          load_f32<T, V>(x + (size_t)idx[u] * C + c, xv[u]);
          load_f32<T, V>(g + (size_t)(o0 + u * R) * C + c, gv[u]);
        }
      }
#pragma unroll
      for (int u = 0; u < CW_ROWS; ++u) {
        if (idx[u] < 0) continue;
#pragma unroll
        for (int v = 0; v < V; ++v) acc[v] = fmaf(xv[u][v], gv[u][v], acc[v]);
      }
    }
  }
  const uint32_t lane = threadIdx.y * S + threadIdx.x;
#pragma unroll
  for (int v = 0; v < V; ++v) red[lane * V + v] = acc[v];
  __syncthreads();
  if (threadIdx.y != 0 || !live) return;
  for (uint32_t ry = 1; ry < R; ++ry) {
#pragma unroll
    for (int v = 0; v < V; ++v) acc[v] += red[(ry * S + threadIdx.x) * V + v];
  }
  float *dst = part + ((size_t)split * K + k) * C + c;
#pragma unroll
  for (int v = 0; v < V; ++v) dst[v] = acc[v];
}

// Vector lanes of one wgrad slab: the row's vectors, rounded up to a power of two, at most 32.
static uint32_t wgrad_slab_lanes(uint32_t vpr) {
  uint32_t s = 1;
  while (s < vpr && s < 32) s *= 2;
  return s;
}

// Row splits k_chwise_wgrad plans: about eight 256-thread CTAs per SM over the grid, each split at
// least 1024 rows.
static uint32_t chwise_wgrad_splits(uint32_t vpr, uint32_t K, uint32_t n_out) {
  const uint64_t slabs = cdiv(vpr, wgrad_slab_lanes(vpr));
  const uint64_t splits = std::max<uint64_t>(1, cdiv(8ull * num_sms(), (uint64_t)K * slabs));
  return (uint32_t)std::min<uint64_t>({splits, cdiv(n_out, 1024), 65535});
}

template <typename T, int V>
static int launch_gather(const void *x, uint32_t C, const float *W, const int32_t *nbr, uint32_t K,
                         uint32_t n_rows, void *y, cudaStream_t stream) {
  const unsigned blocks = cdiv((uint64_t)n_rows * (C / V), CW_THREADS);
  k_chwise_gather<T, V><<<blocks, CW_THREADS, 0, stream>>>((const T *)x, C, W, nbr, K, n_rows,
                                                           (T *)y);
  MEB_LAUNCH_OK();
  return MEB200_OK;
}

template <typename T, int V>
static int launch_wgrad(const void *x, const void *g, uint32_t C, const int32_t *out_nbr,
                        uint32_t K, uint32_t n_out, float *dW, void *workspace,
                        uint64_t workspace_bytes, cudaStream_t stream) {
  const uint32_t vpr = C / V, S = wgrad_slab_lanes(vpr);
  const uint32_t planned = chwise_wgrad_splits(vpr, K, n_out);
  const uint32_t rows = cdiv(n_out, workspace_splits(planned, workspace, workspace_bytes,
                                                     (uint64_t)K * C * sizeof(float)));
  const uint32_t splits = cdiv(n_out, rows);
  float *part = splits > 1 ? reinterpret_cast<float *>(workspace) : dW;
  dim3 grid(K, splits, cdiv(vpr, S)), block(S, CW_THREADS / S);
  k_chwise_wgrad<T, V><<<grid, block, 0, stream>>>((const T *)x, (const T *)g, C, out_nbr, K,
                                                   n_out, rows, part);
  MEB_LAUNCH_OK();
  if (splits == 1) return MEB200_OK;
  return launch_split_sum(part, dW, (size_t)K * C, splits, stream);
}

}  // namespace meb200

using namespace meb200;

extern "C" {

int meb200_chwise_gather(const void *x, int dtype, uint32_t n_x, uint32_t C, const float *W,
                         const int32_t *nbr, uint32_t K, uint32_t n_rows, void *y, void *stream) {
  if (n_rows == 0 || C == 0) return MEB200_OK;
  MEB_CHECK_ARG(K >= 1, "kernel volume %u", K);
  MEB_CHECK_ARG(x != nullptr || n_x == 0, "null x with %u rows", n_x);
  MEB_CHECK_ARG(W && nbr && y, "null buffer");
  cudaStream_t s = (cudaStream_t)stream;
  MEB_DISPATCH_DTYPE(dtype, MEB_DISPATCH_VEC(T, C, aligned(16, x, y, W),
                                             return launch_gather<T, V>(x, C, W, nbr, K, n_rows, y, s)));
}

uint64_t meb200_chwise_wgrad_workspace_bytes(uint32_t n_out, uint32_t C, uint32_t K, int dtype) {
  if (n_out == 0 || C == 0 || K == 0) return 0;
  const uint32_t vpr = C / vec_elems(dtype_size(dtype), C);
  const uint32_t rows = cdiv(n_out, chwise_wgrad_splits(vpr, K, n_out));
  const uint32_t splits = cdiv(n_out, rows);
  return splits > 1 ? (uint64_t)splits * K * C * sizeof(float) : 0;
}

int meb200_chwise_wgrad(const void *x, const void *g, int dtype, uint32_t n_x, uint32_t C,
                        const int32_t *out_nbr, uint32_t K, uint32_t n_out, float *dW,
                        void *workspace, uint64_t workspace_bytes, void *stream) {
  if (C == 0 || K == 0) return MEB200_OK;
  MEB_CHECK_ARG(dW != nullptr, "null dW");
  cudaStream_t s = (cudaStream_t)stream;
  if (n_out == 0) {
    MEB_CUDA(cudaMemsetAsync(dW, 0, (size_t)K * C * sizeof(float), s));
    return MEB200_OK;
  }
  MEB_CHECK_ARG(x != nullptr || n_x == 0, "null x with %u rows", n_x);
  MEB_CHECK_ARG(g && out_nbr, "null buffer");
  MEB_DISPATCH_DTYPE(dtype, MEB_DISPATCH_VEC(T, C, aligned(16, x, g),
                                             return launch_wgrad<T, V>(x, g, C, out_nbr, K, n_out, dW,
                                                                       workspace, workspace_bytes, s)));
}

}
