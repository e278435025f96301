"""Pair-mode wgrad of offsets with far more pairs than the mean: k_wgrad_wg runs each of their units
as one CTA per column slice (one wgmma instruction's columns).  An output element is the same
sequence of instructions on the same operands either way, so the slicing must not change a bit.

Without a workspace every offset is one unit (one CTA, or one CTA per slice), summed in stage
order.  The heavy offset of a K = 27 map (sliced) must then equal, bit for bit, the K = 1 map of
its pairs alone (never sliced: one offset is never above the mean), and every offset must meet the
float64 bound TC_ACC * 2^-20 * A (tests/helpers.py)."""
import pytest
import torch

from helpers import TC_ACC, _pairs, _Route, assert_one_rounding, lib_conv_backward, ref_wgrad

pytestmark = pytest.mark.gpu

DTYPES = pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])


def _heavy_table(K, n, heavy, seed):
    """[K, n]: offset `heavy` pairs every row with a random row, the others at density 0.2."""
    g = torch.Generator().manual_seed(seed)
    nbr = torch.randint(0, n, (K, n), generator=g, dtype=torch.int32)
    nbr[torch.rand((K, n), generator=g) > 0.2] = -1
    nbr[heavy] = torch.randperm(n, generator=g).int()
    return nbr


# (c_in, c_out, rows, pair-list chunk rows or None): c_out 96 = 3 slices of 32, 128 = 2 of 64,
# 256 = 4 of 64, 48 = 3 of 16; two channel tiles at c_in = 192
CASES = [(96, 96, 20000, None), (128, 128, 12000, 4096), (64, 256, 6000, None),
         (192, 48, 9000, 2048)]


@DTYPES
@pytest.mark.parametrize("c_in,c_out,n,chunk_rows", CASES)
def test_sliced_offsets_keep_their_bits(ME, cuda, dtype, c_in, c_out, n, chunk_rows, monkeypatch):
    from minkowskiengine_b200 import backend
    if chunk_rows is not None:
        monkeypatch.setattr(backend._KernelMap, "PAIR_CHUNK_ROWS", chunk_rows)
    K, heavy = 27, 13
    g = torch.Generator().manual_seed(c_in * 7 + c_out)
    feats = (torch.rand(n, c_in, generator=g) - 0.5).to(dtype).to(cuda)
    gout = (torch.rand(n, c_out, generator=g) - 0.5).to(dtype).to(cuda)
    w = torch.zeros(K, c_in, c_out, device=cuda)
    nbr = _heavy_table(K, n, heavy, c_out).to(cuda)
    empty = torch.full((K, n), -1, dtype=torch.int32, device=cuda)
    km = backend._KernelMap(nbr, empty)
    if chunk_rows is not None:
        assert km.pair_lists()[3] > 1, "the case means to cover several row chunks"
    what = f"{c_in}->{c_out} {dtype}"
    with _Route(True, what):
        _, gw = lib_conv_backward(feats, gout, w, km, need_w=True, pairs=True)
        _, gw2 = lib_conv_backward(feats, gout, w, km, need_w=True, pairs=True)
        km1 = backend._KernelMap(nbr[heavy:heavy + 1].contiguous(), empty[:1].contiguous())
        _, gw1 = lib_conv_backward(feats, gout, w[:1].contiguous(), km1, need_w=True, pairs=True)
    ref, A = ref_wgrad(feats, gout, _pairs(nbr))
    assert_one_rounding(gw, ref, A, what, TC_ACC)
    assert torch.equal(gw, gw2), f"{what}: differs run to run"
    assert torch.equal(gw[heavy], gw1[0]), f"{what}: the sliced offset differs from the unsliced one"
