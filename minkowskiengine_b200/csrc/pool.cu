// Local pooling (sum / avg / max) over the same neighbour tables as the convolution.
//
// Reference semantics: NonzeroAvgPooling{Forward,Backward}KernelCPU
// (src/pooling_avg_kernel.hpp:40-150) and MaxPooling{Forward,Backward}KernelCPU
// (src/pooling_max_kernel.hpp:35-115).  The reference GPU path goes through cuSPARSE
// SpMM + thrust sorts (src/pooling_avg_kernel.cu:127-345, pooling_max_kernel.cu:129-234);
// here each output element is reduced by one thread straight from the k-major table:
// no sort, no temporaries, deterministic, offsets visited in ascending k so max ties
// resolve exactly as the CPU loop does (strict '<', first k wins).
#include <float.h>

#include "common.cuh"

namespace meb200 {

// The lowest finite value of the storage type: what an empty max window holds, as the reference
// CPU kernel fills it (-FLT_MAX would round to -inf in bf16 / fp16).
template <typename T> __device__ __forceinline__ float lowest_finite();
template <> __device__ __forceinline__ float lowest_finite<float>() { return -FLT_MAX; }
template <> __device__ __forceinline__ float lowest_finite<__nv_bfloat16>() {
  return __uint_as_float(0xff7f0000u);   // -0x1.fep+127
}
template <> __device__ __forceinline__ float lowest_finite<__half>() { return -65504.f; }

template <typename T, int MODE>
__global__ void __launch_bounds__(256)
k_pool_fwd(const T *__restrict__ in, uint32_t C, const int32_t *__restrict__ out_nbr, uint32_t K,
           uint32_t n_out, T *__restrict__ out, void *__restrict__ aux) {
  uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (uint64_t)n_out * C) return;
  uint32_t o = (uint32_t)(t / C), c = (uint32_t)(t % C);
  if (MODE == MEB200_POOL_MAX) {
    float best = lowest_finite<T>();
    int32_t arg = -1;
    for (uint32_t k = 0; k < K; ++k) {
      int32_t i = __ldg(out_nbr + (size_t)k * n_out + o);
      if (i < 0) continue;
      float v = to_f32<T>(in[(size_t)i * C + c]);
      if (best < v) {
        best = v;
        arg = i * (int32_t)C + (int32_t)c;
      }
    }
    out[t] = from_f32<T>(best);
    reinterpret_cast<int32_t *>(aux)[t] = arg;
  } else {
    float acc = 0.f;
    uint32_t cnt = 0;
    for (uint32_t k = 0; k < K; ++k) {
      int32_t i = __ldg(out_nbr + (size_t)k * n_out + o);
      if (i < 0) continue;
      acc += to_f32<T>(in[(size_t)i * C + c]);
      ++cnt;
    }
    if (MODE == MEB200_POOL_AVG) {
      if (cnt > 0) acc /= (float)cnt;
      if (c == 0) reinterpret_cast<T *>(aux)[o] = from_f32<T>((float)cnt);
    }
    out[t] = from_f32<T>(acc);
  }
}

template <typename T, int MODE>
__global__ void __launch_bounds__(256)
k_pool_bwd_gather(const T *__restrict__ grad_out, uint32_t C, const int32_t *__restrict__ in_nbr,
                  uint32_t K, uint32_t n_in, const T *__restrict__ num_nonzero,
                  T *__restrict__ grad_in) {
  uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (uint64_t)n_in * C) return;
  uint32_t i = (uint32_t)(t / C), c = (uint32_t)(t % C);
  float acc = 0.f;
  for (uint32_t k = 0; k < K; ++k) {
    int32_t o = __ldg(in_nbr + (size_t)k * n_in + i);
    if (o < 0) continue;
    float g = to_f32<T>(grad_out[(size_t)o * C + c]);
    if (MODE == MEB200_POOL_AVG) {
      float cnt = to_f32<T>(num_nonzero[o]);
      if (cnt > 0.f) acc += g / cnt;
    } else {
      acc += g;
    }
  }
  grad_in[t] = from_f32<T>(acc);
}

// Input-stationary: grad_in[i, c] = sum over k ascending of grad_out[o, c] where o = in_nbr[k][i]
// picked input element (i, c) as its arg-max.  Each element is written once, summed in fp32 and
// rounded once, whatever the number of windows it won.
template <typename T>
__global__ void __launch_bounds__(256)
k_pool_bwd_max(const T *__restrict__ grad_out, uint32_t C, const int32_t *__restrict__ in_nbr,
               uint32_t K, uint32_t n_in, const int32_t *__restrict__ max_index,
               T *__restrict__ grad_in) {
  uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (uint64_t)n_in * C) return;
  uint32_t i = (uint32_t)(t / C), c = (uint32_t)(t % C);
  const int32_t self = (int32_t)t;   // i * C + c: max_index is int32 (checked by the forward)
  float acc = 0.f;
  for (uint32_t k = 0; k < K; ++k) {
    int32_t o = __ldg(in_nbr + (size_t)k * n_in + i);
    if (o < 0) continue;
    const size_t oc = (size_t)o * C + c;
    if (__ldg(max_index + oc) == self) acc += to_f32<T>(grad_out[oc]);
  }
  grad_in[t] = from_f32<T>(acc);
}

template <typename T>
static int pool_fwd_t(const void *in, uint32_t C, const int32_t *nbr, uint32_t K, uint32_t n_out,
                      int mode, void *out, void *aux, cudaStream_t s) {
  unsigned blocks = cdiv((uint64_t)n_out * C, 256);
  switch (mode) {
    case MEB200_POOL_SUM:
      k_pool_fwd<T, MEB200_POOL_SUM><<<blocks, 256, 0, s>>>((const T *)in, C, nbr, K, n_out, (T *)out, aux);
      break;
    case MEB200_POOL_AVG:
      k_pool_fwd<T, MEB200_POOL_AVG><<<blocks, 256, 0, s>>>((const T *)in, C, nbr, K, n_out, (T *)out, aux);
      break;
    case MEB200_POOL_MAX:
      k_pool_fwd<T, MEB200_POOL_MAX><<<blocks, 256, 0, s>>>((const T *)in, C, nbr, K, n_out, (T *)out, aux);
      break;
    default:
      set_error("pooling mode %d is not a local pooling mode", mode);
      return MEB200_ERR_INVALID;
  }
  MEB_LAUNCH_OK();
  return MEB200_OK;
}

template <typename T>
static int pool_bwd_t(const void *grad_out, uint32_t n_in, uint32_t C, const int32_t *in_nbr,
                      uint32_t K, uint32_t n_out, int mode, const void *aux, void *grad_in,
                      cudaStream_t s) {
  (void)n_out;
  if (mode == MEB200_POOL_MAX) {
    if (n_in == 0) return MEB200_OK;
    k_pool_bwd_max<T><<<cdiv((uint64_t)n_in * C, 256), 256, 0, s>>>(
        (const T *)grad_out, C, in_nbr, K, n_in, (const int32_t *)aux, (T *)grad_in);
  } else if (mode == MEB200_POOL_AVG) {
    if (n_in == 0) return MEB200_OK;
    k_pool_bwd_gather<T, MEB200_POOL_AVG><<<cdiv((uint64_t)n_in * C, 256), 256, 0, s>>>(
        (const T *)grad_out, C, in_nbr, K, n_in, (const T *)aux, (T *)grad_in);
  } else if (mode == MEB200_POOL_SUM) {
    if (n_in == 0) return MEB200_OK;
    k_pool_bwd_gather<T, MEB200_POOL_SUM><<<cdiv((uint64_t)n_in * C, 256), 256, 0, s>>>(
        (const T *)grad_out, C, in_nbr, K, n_in, nullptr, (T *)grad_in);
  } else {
    set_error("pooling mode %d is not a local pooling mode", mode);
    return MEB200_ERR_INVALID;
  }
  MEB_LAUNCH_OK();
  return MEB200_OK;
}

}  // namespace meb200

using namespace meb200;

extern "C" {

int meb200_pool_forward(const void *in, int dtype, uint32_t n_in, uint32_t C,
                        const int32_t *out_nbr, uint32_t K, uint32_t n_out, int mode, void *out,
                        void *aux, void *stream) {
  (void)n_in;
  if (n_out == 0 || C == 0) return MEB200_OK;
  MEB_CHECK_ARG(in && out_nbr && out, "null buffer");
  MEB_CHECK_ARG(mode == MEB200_POOL_SUM || aux != nullptr, "aux buffer required");
  MEB_CHECK_ARG((uint64_t)n_in * C < 0x7FFFFFFFull || mode != MEB200_POOL_MAX,
                "max_index is int32: n_in*C too large");
  cudaStream_t s = (cudaStream_t)stream;
  MEB_DISPATCH_DTYPE(dtype, return pool_fwd_t<T>(in, C, out_nbr, K, n_out, mode, out, aux, s));
}

int meb200_pool_backward(const void *grad_out, int dtype, uint32_t n_in, uint32_t C,
                         const int32_t *in_nbr, uint32_t K, uint32_t n_out, int mode,
                         const void *aux, void *grad_in, void *stream) {
  if (C == 0) return MEB200_OK;
  MEB_CHECK_ARG(grad_in != nullptr || n_in == 0, "null grad_in");
  MEB_CHECK_ARG(mode == MEB200_POOL_SUM || aux != nullptr, "aux buffer required");
  MEB_CHECK_ARG(in_nbr != nullptr || n_in == 0, "in_nbr required");
  MEB_CHECK_ARG((uint64_t)n_in * C < 0x7FFFFFFFull || mode != MEB200_POOL_MAX,
                "max_index is int32: n_in*C too large");
  cudaStream_t s = (cudaStream_t)stream;
  MEB_DISPATCH_DTYPE(dtype, return pool_bwd_t<T>(grad_out, n_in, C, in_nbr, K, n_out, mode, aux,
                                                  grad_in, s));
}

}
