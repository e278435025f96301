// The fp8 formats and the per-tensor scale formula shared by the quantisation kernels (quant.cu)
// and the batch-norm passes that write fp8 copies of their output (batchnorm.cu).  The arithmetic
// is documented at the top of quant.cu and in include/meb200.h.
#pragma once
#include <float.h>
#include <stdint.h>

#include "ptx.cuh"

namespace meb200 {

// The two fp8 formats: the largest finite value, and the saturating conversion of a pair (lo = a)
struct E4M3 {
  static constexpr float kMax = 448.f;
  static __device__ __forceinline__ uint16_t cvt2(float a, float b) {
    return ptx::e4m3x2_satfinite(a, b);
  }
};
struct E5M2 {
  static constexpr float kMax = 57344.f;
  static __device__ __forceinline__ uint16_t cvt2(float a, float b) {
    return ptx::e5m2x2_satfinite(a, b);
  }
};

// scale and inv of a tensor (or column) whose finite values have the maximum magnitude amax
template <typename F>
__device__ __forceinline__ void fp8_scales(float amax, float &scale, float &inv) {
  if (amax == 0.f) {
    scale = inv = 1.f;
  } else if (isinf(inv = __fdiv_rn(F::kMax, amax))) {
    inv = FLT_MAX;
    scale = __fdiv_rn(1.f, FLT_MAX);
  } else {
    scale = __fdiv_rn(amax, F::kMax);
  }
}

__device__ __forceinline__ float finite_abs(float v) { return isfinite(v) ? fabsf(v) : 0.f; }

template <typename F>
__device__ __forceinline__ uint8_t fp8_byte(float x, float inv) {
  return (uint8_t)(F::cvt2(__fmul_rn(x, inv), 0.f) & 0xFFu);
}

// The max of m over the lanes of the warp that arrive together, atomically maxed into *slot by
// one of them (non-negative floats order as their bit patterns; a max is order-free).  For
// kernels whose idle threads have returned, so that no CTA barrier can be used.
__device__ __forceinline__ void warp_amax_to(float m, uint32_t *slot) {
  const uint32_t mask = __activemask();
  const uint32_t v = __reduce_max_sync(mask, __float_as_uint(m));
  if ((threadIdx.x & 31) == (uint32_t)(__ffs(mask) - 1)) atomicMax(slot, v);
}

}  // namespace meb200
