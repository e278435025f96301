"""How the tensor-core weight gradient's fp32 accumulation errs with the length of a CTA's share.

k_wgrad_wg adds a CTA's share of an offset's pairs into wgmma accumulators, 16 pairs per wgmma
step.  The accumulation truncates: each step may lose part of an ulp of the running sum.  On
zero-mean operands those losses have both signs and mostly cancel, which is where TC_ACC
(tests/helpers.py) was measured.  On one-signed operands (ReLU outputs times gradients of one sign)
every loss has the same sign, the running sum grows towards A, and the error grows with the number
of steps: TC_ACC does not bound it.  This file runs one share (no workspace: one split) of an
identity map of L pairs, L from 4k to 256k, on both kinds of operands, against float64:

* zero-mean: within TC_ACC · 2^-20 · A at every length;
* one-signed: within WG_STEP · steps · 2^-24 · A (helpers.WG_STEP), beyond TC_ACC at the
  longest share, and growing with the share's length as that model says."""
import pytest
import torch

from helpers import TC_ACC, WG_STEP, lib_conv_backward

pytestmark = pytest.mark.gpu

LENGTHS = [4096, 32768, 262144]
C = 64


def _share(cuda, dtype, L, one_signed, seed):
    from minkowskiengine_b200 import backend
    g = torch.Generator().manual_seed(seed)
    x, gout = torch.rand(L, C, generator=g), torch.rand(L, C, generator=g)
    if not one_signed:
        x, gout = x - 0.5, gout - 0.5
    x, gout = x.to(dtype).to(cuda), gout.to(dtype).to(cuda)
    rows = torch.arange(L, dtype=torch.int32, device=cuda).view(1, L)
    km = backend._KernelMap(rows.clone(), rows.clone())
    w = torch.zeros(1, C, C, device=cuda)
    _, gw = lib_conv_backward(x, gout, w, km, need_w=True, pairs=True, workspace=None)
    x64, g64 = x.double(), gout.double()
    ref, A = x64.t() @ g64, x64.abs().t() @ g64.abs()
    err = (gw[0].double() - ref).abs()
    return float((err / (A * 2.0 ** -20)).max()), float((err / (A * 2.0 ** -24 * (L // 16))).max())


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def test_wgrad_error_follows_the_share_length(ME, cuda, dtype):
    zero_mean, one_signed = [], []
    for L in LENGTHS:
        zero_mean.append(_share(cuda, dtype, L, False, L))
        one_signed.append(_share(cuda, dtype, L, True, L + 1))
        print(f"[wgrad accumulation] {dtype} share {L} pairs ({L // 16} steps): zero-mean "
              f"{zero_mean[-1][0]:.3g} · 2^-20 A; one-signed {one_signed[-1][0]:.3g} · 2^-20 A = "
              f"{one_signed[-1][1]:.3g} · steps · 2^-24 A")
    assert all(u <= TC_ACC for u, _ in zero_mean), "zero-mean operands beyond TC_ACC"
    assert all(s <= WG_STEP for _, s in one_signed), "one-signed operands beyond the step model"
    assert one_signed[-1][0] > TC_ACC, "one-signed operands over a long share stay within TC_ACC"
    # linear in the steps: 64 times the steps give at least 16 times the error
    assert one_signed[-1][0] >= 16 * one_signed[0][0]
