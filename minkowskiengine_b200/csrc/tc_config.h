// Host-side launch configuration of the wgmma kernels (plain C++, no CUDA): stage widths,
// shared-memory footprints and row splits.  Kept separate so it can be unit-tested on a machine
// without a GPU (tests/test_tc_config.py, tests/test_tc_col_slices.py).
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

// forward / dgrad: bytes of every operand row one stage holds (128, 64 or 32: one wgmma k-step
// reads 32 bytes of a row whatever the element size), for `c_red` reduction channels of `esz`
// bytes each; 0 = unsupported (the row is not a whole number of 32-byte k-steps)
inline uint32_t fwd_stage_bytes(uint32_t c_red, uint32_t esz) {
  const uint32_t b = c_red * esz;
  return b % 128 == 0 ? 128 : (b % 64 == 0 ? 64 : (b % 32 == 0 ? 32 : 0));
}
// one stage = A [128 rows x width] + B [c_cols x width], width in bytes; +1 KB for alignment
inline uint32_t fwd_ring_bytes(uint32_t width, uint32_t c_cols) {
  return 1024 + kStages * (kFwdRows + c_cols) * width;
}
// 16-bit elements: reduction channels per stage (64, 32 or 16), 0 = unsupported
inline uint32_t fwd_bk(uint32_t c_red) { return fwd_stage_bytes(c_red, 2) / 2; }
inline uint32_t fwd_smem_bytes(uint32_t bk, uint32_t c_cols) { return fwd_ring_bytes(bk * 2, c_cols); }

// N of the wgmma instructions that cover c_cols columns: the widest of 64, 32, 16 dividing it
// (MEB_COLS_DISPATCH in conv_tc.cu)
inline uint32_t wgmma_n(uint32_t c_cols) {
  return c_cols % 64 == 0 ? 64 : (c_cols % 32 == 0 ? 32 : 16);
}

// forward / dgrad: columns each CTA computes of a launch's c_cols (<= kMaxCols) output columns;
// the launch runs c_cols / slice CTAs per 128-row tile (blockIdx.y = slice).  A launch with few
// row tiles (the coarse levels of a U-Net) takes the narrowest slice that keeps its CTAs within
// one per SM: more CTAs, each with a fraction of the MMAs and of the weight bytes, for the same
// gathered rows (which such small levels keep in L2).  A CTA's time is mostly its stages'
// gathers and barriers, not its MMAs, so slices that spill into a second wave of CTAs cost more
// than they save (measured on an H100: BASELINE.md section 17).  The slice is a multiple of
// wgmma_n(c_cols) dividing c_cols, so an output element is the same sequence of m64nNk16
// instructions on the same operands either way: slicing does not change a bit.
inline uint32_t fwd_col_slice(uint32_t n_rows, uint32_t c_cols, uint32_t n_sms) {
  const uint64_t tiles = cdiv_u(n_rows, kFwdRows), n = wgmma_n(c_cols);
  for (uint32_t s = n; s < c_cols; s += n)
    if (c_cols % s == 0 && tiles * (c_cols / s) <= n_sms) return s;
  return c_cols;
}

// one stage = A [64 rows x 128 channels] + B [64 rows x c_out], 16-bit elements
inline uint32_t wgrad_smem_bytes(uint32_t c_out) {
  return 1024 + kStages * kWgRows * (kWgChannels + c_out) * 2;
}

// TF32 wgrad (warp-level mma.sync, fp32 operands read as stored): stages of kWgRowsTf32 pairs, each
// row padded by kWgPadTf32 floats, so that a row stride is 8 or 24 words modulo the 32 banks and the
// fragment loads of a warp (lanes = 4 rows x 8 columns) hit 32 different banks.
constexpr uint32_t kWgRowsTf32 = 32;
constexpr uint32_t kWgPadTf32 = 8;
inline uint32_t wgrad_tf32_smem_bytes(uint32_t c_out) {
  return 1024 + kStages * kWgRowsTf32 * (kWgChannels + kWgPadTf32 + c_out + kWgPadTf32) * 4;
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
