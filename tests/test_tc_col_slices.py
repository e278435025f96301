"""Column slices of the tensor-core forward and dgrad (csrc/tc_config.h fwd_col_slice), checked on
CPU: every slice is a whole number of the wgmma instructions the full width would use and divides
the launch's columns, its ring fits the 227 KB a CTA may use on sm_90, and the bench's layers get
the slices they were measured with (stride 16 sliced, stride 8 and finer at full width)."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SRC = r"""
#include <stdio.h>
#include <initializer_list>
#include "tc_config.h"
using namespace meb200::tc;
int main() {
  int bad = 0;
  const unsigned rows[] = {1, 127, 128, 129, 3513, 15063, 16895, 16896, 60000, 800000};
  for (unsigned cc = 16; cc <= kMaxCols; cc += 16)
    for (unsigned n : rows) {
      const unsigned s = fwd_col_slice(n, cc, 132);
      const unsigned tiles = (n + kFwdRows - 1) / kFwdRows;
      bool ok = s >= 16 && s % wgmma_n(cc) == 0 && cc % s == 0 && wgmma_n(s) == wgmma_n(cc) &&
                (s == cc || tiles * (cc / s) <= 132);
      for (unsigned w = wgmma_n(cc); w < s; w += wgmma_n(cc))   // no narrower slice fits one wave
        if (cc % w == 0 && tiles * (cc / w) <= 132) ok = false;
      for (unsigned width : {32u, 64u, 128u})
        if (fwd_ring_bytes(width, s) > kSmemLimit) { printf("RING BAD cc=%u s=%u\n", cc, s); ++bad; }
      if (!ok) { printf("SLICE BAD n=%u cc=%u s=%u\n", n, cc, s); ++bad; }
    }
  // bench (MinkUNet34C, 8 x 100k voxels; rows per level from profiles/tile_order_counts.py)
  struct { unsigned n, cc, want; } bench[] = {
      {3513, 256, 64},       // stride 16, 256 -> 256: 28 tiles
      {3513, 96, 32},        // 28 tiles, 96 columns: three 32-column slices
      {15063, 256, 256},     // stride 8, 256 -> 256 and 384 -> 256: 118 tiles, full width
      {15063, 128, 128},     // stride 8, 128 -> 128
      {800000, 96, 96},      // stride 1, 96 -> 96: full width
      {313707, 96, 96},      // stride 2
      {72332, 128, 128},     // stride 4, 192 -> 128
  };
  for (auto &b : bench) {
    const unsigned s = fwd_col_slice(b.n, b.cc, 132);
    if (s != b.want) { printf("BENCH BAD n=%u cc=%u s=%u want %u\n", b.n, b.cc, s, b.want); ++bad; }
  }
  printf("bad=%d\n", bad);
  return bad != 0;
}
"""


def test_fwd_col_slices(tmp_path):
    src = tmp_path / "slices.cpp"
    src.write_text(SRC)
    exe = tmp_path / "slices"
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-O1", "-I",
                    os.path.join(ROOT, "minkowskiengine_b200", "csrc"), str(src), "-o", str(exe)],
                   check=True)
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-3000:]
    assert "bad=0" in r.stdout
