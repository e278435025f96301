// Library-level state: last error (per thread), launch counter, build facts; the split reduction
// shared by the weight gradients.
#include <stdarg.h>

#include <algorithm>
#include <atomic>

#include "common.cuh"

namespace meb200 {

static thread_local char g_err[1024] = "";
static std::atomic<uint64_t> g_launches{0};
static std::atomic<uint64_t> g_tc_launches{0};

void set_error(const char *fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

void set_arg_error(const char *file, int line, const char *cond, const char *fmt, ...) {
  char msg[384];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(msg, sizeof(msg), fmt, ap);
  va_end(ap);
  set_error("%s:%d invalid argument (%s): %s", file, line, cond, msg);
}

void count_launch(unsigned n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
void count_tc_launch() { g_tc_launches.fetch_add(1, std::memory_order_relaxed); }
uint64_t tc_launches() { return g_tc_launches.load(std::memory_order_relaxed); }

int num_sms() {
  static int cached = 0;
  if (cached == 0) {
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) == cudaSuccess &&
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0)
      cached = n;
    else
      cached = 132;   // H100 SXM
  }
  return cached;
}

uint32_t workspace_splits(uint32_t planned, const void *workspace, uint64_t workspace_bytes,
                          uint64_t slot_bytes) {
  if (workspace == nullptr || !aligned(16, workspace)) return 1;
  return (uint32_t)std::min<uint64_t>(planned, std::max<uint64_t>(1, workspace_bytes / slot_bytes));
}

__device__ __forceinline__ void add(float &a, float b) { a += b; }
__device__ __forceinline__ void add(float4 &a, float4 b) {
  a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
}

// F = float4: four consecutive elements per thread, each summed over the splits on its own
template <typename F>
__global__ void __launch_bounds__(256)
k_split_sum(const F *__restrict__ part, F *__restrict__ dW, size_t n, uint32_t splits) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n;
       i += (size_t)gridDim.x * blockDim.x) {
    F a = part[i];
    for (uint32_t s = 1; s < splits; ++s) add(a, part[s * n + i]);
    dW[i] = a;
  }
}

int launch_split_sum(const float *part, float *dW, size_t n, uint32_t splits,
                     cudaStream_t stream) {
  if (n % 4 == 0 && aligned(16, part, dW)) {
    const size_t n4 = n / 4;
    k_split_sum<float4><<<std::min(cdiv(n4, 256), 4096u), 256, 0, stream>>>(
        reinterpret_cast<const float4 *>(part), reinterpret_cast<float4 *>(dW), n4, splits);
  } else {
    k_split_sum<float><<<std::min(cdiv(n, 256), 4096u), 256, 0, stream>>>(part, dW, n, splits);
  }
  MEB_LAUNCH_OK();
  return MEB200_OK;
}

}  // namespace meb200

extern "C" {

const char *meb200_last_error(void) { return meb200::g_err; }

const char *meb200_build_arch(void) { return "sm_90a"; }

int meb200_cudart_version(void) { return CUDART_VERSION; }

uint64_t meb200_launch_count(void) { return meb200::g_launches.load(std::memory_order_relaxed); }

uint64_t meb200_tc_launch_count(void) { return meb200::tc_launches(); }

}
