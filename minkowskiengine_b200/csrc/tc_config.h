// Host-side launch configuration of the wgmma kernels (plain C++, no CUDA): stage widths,
// shared-memory footprints and row splits.  Kept separate so it can be unit-tested on a machine
// without a GPU (tests/test_tc_config.py).
#pragma once
#include <stdint.h>

namespace meb200 {
namespace tc {

constexpr uint32_t kStages = 4;             // cp.async ring depth (loads run 2 stages ahead)
constexpr uint32_t kSmemLimit = 227 * 1024; // opt-in shared memory of one CTA on sm_90
constexpr uint32_t kMaxCols = 256;          // accumulator columns of one CTA (one launch slice)
constexpr uint32_t kFwdRows = 128;          // forward / dgrad: output rows per CTA (2 warpgroups)
constexpr uint32_t kWgRows = 64;            // wgrad: reduction rows per stage
constexpr uint32_t kWgChannels = 128;       // wgrad: input channels per CTA (2 warpgroups)

inline uint32_t cdiv_u(uint64_t a, uint64_t b) { return (uint32_t)((a + b - 1) / b); }

// forward / dgrad: reduction channels per stage (64, 32 or 16), 0 = unsupported
inline uint32_t fwd_bk(uint32_t c_red) {
  return c_red % 64 == 0 ? 64 : (c_red % 32 == 0 ? 32 : (c_red % 16 == 0 ? 16 : 0));
}
// one stage = A [128 rows x bk] + B [c_cols x bk], 16-bit elements; +1 KB for alignment
inline uint32_t fwd_smem_bytes(uint32_t bk, uint32_t c_cols) {
  return 1024 + kStages * (kFwdRows + c_cols) * bk * 2;
}
// one stage = A [64 rows x 128 channels] + B [64 rows x c_out]
inline uint32_t wgrad_smem_bytes(uint32_t c_out) {
  return 1024 + kStages * kWgRows * (kWgChannels + c_out) * 2;
}

// wgrad row splits: enough CTAs for two waves over (k, channel tile) pairs, but at least
// 4 stages of work per CTA so the store of its 128 x c_out partial sums (and their later
// ordered addition) stays amortised.
// `stages` is the (estimated) number of 64-row stages one (k, channel tile) has in total.
inline uint32_t wgrad_splits(uint32_t stages, uint32_t K, uint32_t m_tiles, uint32_t n_sms) {
  const uint64_t base = (uint64_t)K * m_tiles;
  uint64_t want = (2ull * n_sms + base - 1) / base;
  uint64_t by_work = stages / 4;
  if (by_work < 1) by_work = 1;
  if (want > by_work) want = by_work;
  if (want < 1) want = 1;
  if (want > 65535) want = 65535;
  return (uint32_t)want;
}

}  // namespace tc
}  // namespace meb200
