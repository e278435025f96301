"""The bf16 / fp16 weight gradient (k_wgrad_wg) keeps two CTAs per SM for tiles of up to 96 output
columns: their rings (csrc/tc_config.h, wgrad_smem_bytes) plus the 1 KB the hardware reserves for
each CTA must fit the 228 KB of shared memory of an H100 SM twice.  At 96 columns that holds to
the byte, so the loader keeps its index words in registers, not in shared memory."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SRC = r"""
#include <stdio.h>
#include "tc_config.h"
using namespace meb200::tc;
int main() {
  const unsigned sm_bytes = 228 * 1024, reserved = 1024;
  int bad = 0;
  for (unsigned c = 16; c <= 96; c += 16) {
    const unsigned two = 2 * (wgrad_smem_bytes(c) + reserved);
    printf("c_cols %u: %u B per CTA, two CTAs %u of %u B\n", c, wgrad_smem_bytes(c), two, sm_bytes);
    if (two > sm_bytes) ++bad;
  }
  printf("bad=%d\n", bad);
  return bad != 0;
}
"""


def test_wgrad_two_ctas_per_sm(tmp_path):
    src = tmp_path / "smem.cpp"
    src.write_text(SRC)
    exe = tmp_path / "smem"
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-O1", "-I",
                    os.path.join(ROOT, "minkowskiengine_b200", "csrc"), str(src), "-o", str(exe)],
                   check=True)
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    assert r.returncode == 0 and "bad=0" in r.stdout, r.stdout
