"""Host-side launch configuration of the wgmma kernels (csrc/tc_config.h), checked on CPU:
every channel shape MinkUNet14/34C/... can produce must get a stage width and a shared-memory
ring that fit in the 227 KB a CTA may use on sm_90, and wgrad row splits that keep at most
about two waves of CTAs on the 132 SMs of an H100 while giving every CTA enough work."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SRC = r"""
#include <stdio.h>
#include <initializer_list>
#include "tc_config.h"
using namespace meb200::tc;
int main() {
  const unsigned chans[] = {16, 32, 48, 64, 96, 128, 160, 192, 256, 384, 512};
  const unsigned ncs[] = {16, 32, 48, 64, 96, 128, 192, 256};
  int bad = 0;
  for (unsigned cr : chans) for (unsigned cc : ncs) {
    const unsigned bk = fwd_bk(cr);
    const unsigned smem = fwd_smem_bytes(bk, cc);
    bool ok = (bk == 64 || bk == 32 || bk == 16) && cr % bk == 0 && smem <= kSmemLimit &&
              (cr % 64 != 0 || bk == 64);
    if (!ok) { printf("FWD BAD cr=%u cc=%u bk=%u smem=%u\n", cr, cc, bk, smem); ++bad; }
    printf("fwd %u %u : bk=%u smem=%u\n", cr, cc, bk, smem);
  }
  if (fwd_bk(24) != 0 || fwd_bk(8) != 0) { printf("FWD BAD: widths not a multiple of 16 accepted\n"); ++bad; }
  for (unsigned co : ncs) {
    const unsigned smem = wgrad_smem_bytes(co);
    if (smem > kSmemLimit) { printf("WG BAD co=%u smem=%u\n", co, smem); ++bad; }
    printf("wg %u : smem=%u\n", co, smem);
  }
  const unsigned sms = 132;
  for (unsigned K : {1u, 8u, 27u, 125u}) for (unsigned mt : {1u, 2u, 4u}) for (unsigned st : {0u, 1u, 5u, 100u, 20000u}) {
    const unsigned s = wgrad_splits(st, K, mt, sms);
    const unsigned by_work = st / 4 > 1 ? st / 4 : 1;
    bool ok = s >= 1 && s <= by_work && (s == 1 || (unsigned long long)(s - 1) * K * mt < 2ull * sms);
    if (!ok) { printf("SPLIT BAD K=%u mt=%u stages=%u splits=%u\n", K, mt, st, s); ++bad; }
  }
  printf("bad=%d\n", bad);
  return bad != 0;
}
"""


def test_tc_launch_configs(tmp_path):
    src = tmp_path / "cfg.cpp"
    src.write_text(SRC)
    exe = tmp_path / "cfg"
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-O1", "-I",
                    os.path.join(ROOT, "minkowskiengine_b200", "csrc"), str(src), "-o", str(exe)],
                   check=True)
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-3000:]
    assert "bad=0" in r.stdout


if __name__ == "__main__":
    import pathlib
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        test_tc_launch_configs(pathlib.Path(d))
        print("ok")
