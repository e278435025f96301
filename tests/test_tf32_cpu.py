"""TF32 convolutions, checked without a GPU: which operand code the host passes under torch's
float32 matmul switch, how it packs and re-packs TF32 weights (against a recording stub of the
native library), that the switch reads without raising after every setter style, and the stage
widths and shared-memory rings of the 4-byte forward / dgrad and of the TF32 wgrad."""
import os
import subprocess

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture
def restore_precision():
    """Leaves torch's fp32 precision strings as this test found them."""
    saved = (torch.backends.fp32_precision, torch.backends.cuda.matmul.fp32_precision)
    yield
    torch.backends.fp32_precision = saved[0]
    torch.backends.cuda.matmul.fp32_precision = saved[1]


class _Stub:
    def __init__(self, calls):
        self.calls = calls

    def __getattr__(self, name):
        def fn(*args):
            self.calls.append((name, args))
            return 1 if name == "meb200_conv_wgrad_uses_pairs" else 0
        return fn


class _Map:
    """The parts of a kernel map the convolution host code reads."""
    K, n_in, n_out, n_pairs = 27, 10, 12, 40
    out_nbr = in_nbr = out_order = in_order = None

    def pair_lists(self):
        self.pair_calls = getattr(self, "pair_calls", 0) + 1
        return None, None, None, 1


@pytest.fixture
def stub(monkeypatch):
    from minkowskiengine_b200 import _lib, backend as B
    calls = []
    monkeypatch.setattr(_lib, "load", lambda: _Stub(calls))
    monkeypatch.setattr(_lib, "current_stream", lambda: None)
    # the stub writes nothing: let the CPU tensors stand in for device buffers
    B._PACKED.clear()
    B._PACK_TABLES.clear()
    yield calls
    B._PACKED.clear()
    B._PACK_TABLES.clear()


def _conv(B, kernel, feats, km):
    B._conv_forward_impl(feats, kernel, km)
    return B._conv_backward_impl(feats, torch.zeros(km.n_out, kernel.shape[2]), kernel, km)


def _codes(calls, name, pos):
    return [c[1][pos] for c in calls if c[0] == name]


def test_default_flag_runs_exact_fp32_and_packs_nothing(stub, restore_precision):
    from minkowskiengine_b200 import _lib, backend as B
    torch.backends.cuda.matmul.fp32_precision = "ieee"
    k = torch.nn.Parameter(torch.randn(27, 32, 64))
    _conv(B, k, torch.randn(10, 32), _Map())
    assert _codes(stub, "meb200_conv_forward", 1) == [_lib.F32]
    assert _codes(stub, "meb200_conv_backward", 2) == [_lib.F32]
    assert _codes(stub, "meb200_conv_backward", 12) == [_lib.F32]          # grad_in dtype
    assert not any(c[0].startswith("meb200_conv_pack_weights") for c in stub)
    assert not B._PACK_TABLES


def test_tf32_flag_passes_tf32_and_packs_fp32_buffers(stub, restore_precision):
    from minkowskiengine_b200 import _lib, backend as B
    torch.backends.cuda.matmul.fp32_precision = "tf32"
    k = torch.nn.Parameter(torch.randn(27, 32, 64))
    km = _Map()
    _conv(B, k, torch.randn(10, 32), km)
    assert _codes(stub, "meb200_conv_forward", 1) == [_lib.TF32]
    assert _codes(stub, "meb200_conv_backward", 2) == [_lib.TF32]
    assert _codes(stub, "meb200_conv_backward", 12) == [_lib.F32]          # grad_in stays fp32
    assert _codes(stub, "meb200_conv_wgrad_uses_pairs", 0) == [_lib.TF32]
    assert _codes(stub, "meb200_conv_workspace_bytes", 4) == [_lib.TF32]
    assert km.pair_calls == 1                                               # pairs when the library asks
    packs = [c for c in stub if c[0] == "meb200_conv_pack_weights"]
    assert len(packs) == 1 and packs[0][1][4] == _lib.TF32                   # packed once for both calls
    w_cast, w_t = B._PACKED[id(k)][4]
    assert w_cast.dtype == w_t.dtype == torch.float32
    assert w_cast.shape == k.shape and w_t.shape == (27, 64, 32)
    # bf16 features still pass their own code, and the two tables live apart
    stub.clear()
    k16 = torch.nn.Parameter(torch.randn(27, 32, 64))
    B._conv_forward_impl(torch.randn(10, 32).bfloat16(), k16, _Map())
    assert _codes(stub, "meb200_conv_forward", 1) == [_lib.BF16]
    assert set(B._PACK_TABLES) == {(None, B.TF32), (None, torch.bfloat16)}


def test_tf32_repacks_in_one_batched_call_and_switches_without_stale_weights(stub, restore_precision):
    from minkowskiengine_b200 import _lib, backend as B
    torch.backends.cuda.matmul.fp32_precision = "tf32"
    ks = [torch.nn.Parameter(torch.randn(27, 32, 64)), torch.nn.Parameter(torch.randn(8, 16, 16))]
    for k in ks:
        B._packed_weights(k, B.TF32)
    # the same kernel packed for bf16 too: its table entry must not collide with the TF32 one
    B._packed_weights(ks[0], torch.bfloat16)
    assert len(B._PACK_TABLES[(None, B.TF32)].entries) == 2
    assert len(B._PACK_TABLES[(None, torch.bfloat16)].entries) == 1
    stub.clear()
    with torch.no_grad():
        for k in ks:
            k.add_(1.0)                                                     # the optimizer stepped
    B._feature_weights(ks[1], B._operand(torch.float32))
    assert [c[0] for c in stub] == ["meb200_conv_pack_weights_batched"]
    assert stub[0][1][1] == 2 and stub[0][1][3] == _lib.TF32
    stub.clear()
    B._feature_weights(ks[0], B._operand(torch.float32))                   # refreshed by that call
    assert stub == []
    # exact fp32 reads the kernel itself; a step taken meanwhile is seen when TF32 comes back
    torch.backends.cuda.matmul.fp32_precision = "ieee"
    w, w_t = B._feature_weights(ks[0], B._operand(torch.float32))
    assert w_t is None and w.data_ptr() == ks[0].data_ptr()
    with torch.no_grad():
        ks[0].mul_(2.0)
    torch.backends.cuda.matmul.fp32_precision = "tf32"
    B._feature_weights(ks[0], B._operand(torch.float32))
    assert [c[0] for c in stub] == ["meb200_conv_pack_weights_batched"]
    # a bf16 pack of the same kernel in between is not served to a TF32 call
    stub.clear()
    B._packed_weights(ks[0], torch.bfloat16)
    w_cast, _ = B._feature_weights(ks[0], B.TF32)
    assert w_cast.dtype == torch.float32 and B._PACKED[id(ks[0])][3] == B.TF32


def test_bf16_features_ignore_the_flag(stub, restore_precision):
    from minkowskiengine_b200 import backend as B
    torch.backends.cuda.matmul.fp32_precision = "tf32"
    assert B._operand(torch.bfloat16) == torch.bfloat16
    assert B._operand(torch.float16) == torch.float16
    assert B._operand(torch.float32) == B.TF32


SETTERS = {
    "allow_tf32 True": (lambda: setattr(torch.backends.cuda.matmul, "allow_tf32", True), True),
    "allow_tf32 False": (lambda: setattr(torch.backends.cuda.matmul, "allow_tf32", False), False),
    "precision high": (lambda: torch.set_float32_matmul_precision("high"), True),
    "precision medium": (lambda: torch.set_float32_matmul_precision("medium"), True),
    "precision highest": (lambda: torch.set_float32_matmul_precision("highest"), False),
    "global tf32": (lambda: setattr(torch.backends, "fp32_precision", "tf32"), True),
    "matmul tf32": (lambda: setattr(torch.backends.cuda.matmul, "fp32_precision", "tf32"), True),
    "matmul ieee": (lambda: setattr(torch.backends.cuda.matmul, "fp32_precision", "ieee"), False),
}


@pytest.mark.parametrize("name", list(SETTERS))
def test_flag_reads_after_every_setter_style(name, restore_precision):
    from minkowskiengine_b200 import backend as B
    torch.backends.fp32_precision = "ieee"
    torch.backends.cuda.matmul.fp32_precision = "none"
    setter, tf32 = SETTERS[name]
    setter()
    assert (B._operand(torch.float32) == B.TF32) == tf32


SRC = r"""
#include <stdio.h>
#include <initializer_list>
#include "tc_config.h"
using namespace meb200::tc;
int main() {
  const unsigned chans[] = {16, 24, 32, 48, 64, 96, 128, 160, 192, 256, 384, 512};
  const unsigned ncs[] = {16, 32, 48, 64, 96, 128, 160, 192, 256};
  int bad = 0;
  for (unsigned cr : chans) for (unsigned cc : ncs) {
    const unsigned w = fwd_stage_bytes(cr, 4), smem = fwd_ring_bytes(w, cc);
    const bool ok = (w == 128 || w == 64 || w == 32) && (cr * 4) % w == 0 && smem <= kSmemLimit &&
                    ((cr * 4) % 128 != 0 || w == 128);
    if (!ok) { printf("TF32 FWD BAD cr=%u cc=%u width=%u smem=%u\n", cr, cc, w, smem); ++bad; }
    printf("tf32 fwd %u %u : width=%u smem=%u\n", cr, cc, w, smem);
  }
  for (unsigned cr : {8u, 40u, 72u})
    if (fwd_stage_bytes(cr, 4) == 0) { printf("TF32 FWD BAD: %u channels rejected\n", cr); ++bad; }
  for (unsigned cr : {1u, 3u, 4u, 12u, 20u, 36u})
    if (fwd_stage_bytes(cr, 4) != 0) { printf("TF32 FWD BAD: %u channels accepted\n", cr); ++bad; }
  for (unsigned cr = 1; cr <= 1024; ++cr)    /* the 16-bit widths are the byte widths over 2 */
    if (fwd_bk(cr) * 2 != fwd_stage_bytes(cr, 2)) { printf("BK BAD %u\n", cr); ++bad; }
  for (unsigned co : ncs) {
    const unsigned smem = wgrad_tf32_smem_bytes(co);
    const unsigned sa = (kWgChannels + kWgPadTf32) % 32, sb = (co + kWgPadTf32) % 32;
    if (smem > kSmemLimit || (sa != 8 && sa != 24) || (sb != 8 && sb != 24)) {
      printf("TF32 WG BAD co=%u smem=%u\n", co, smem); ++bad;
    }
    printf("tf32 wg %u : smem=%u\n", co, smem);
  }
  if (kWgRows % kWgRowsTf32 != 0) { printf("TF32 WG BAD: stages do not tile the shares\n"); ++bad; }
  printf("bad=%d\n", bad);
  return bad != 0;
}
"""


def test_tf32_launch_configs(tmp_path):
    src = tmp_path / "cfg.cpp"
    src.write_text(SRC)
    exe = tmp_path / "cfg"
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-O1", "-I",
                    os.path.join(ROOT, "minkowskiengine_b200", "csrc"), str(src), "-o", str(exe)],
                   check=True)
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-3000:]
    assert "bad=0" in r.stdout
