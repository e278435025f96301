// Library-level state: last error (per thread), launch counter, build facts.
#include <stdarg.h>

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

}  // namespace meb200

extern "C" {

const char *meb200_last_error(void) { return meb200::g_err; }

const char *meb200_build_arch(void) { return "sm_90a"; }

int meb200_cudart_version(void) { return CUDART_VERSION; }

uint64_t meb200_launch_count(void) { return meb200::g_launches.load(std::memory_order_relaxed); }

uint64_t meb200_tc_launch_count(void) { return meb200::tc_launches(); }

}
