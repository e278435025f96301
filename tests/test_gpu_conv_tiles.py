"""CTA tiles of the tensor-core forward and dgrad (k_conv_wg, tc::fwd_col_slice): a launch with
fewer 128-row tiles than SMs runs its columns in slices one wgmma instruction wide, one CTA per
(tile, slice).  An output element is the same sequence of m64nNk16 instructions either way, so

  (a) the rows of a small table, which the kernel runs in column slices, carry exactly the bits of
      the same rows inside a table large enough to run at full width, in bf16, fp16 and TF32;
  (b) both tilings stay within the float64 bound of tests/test_gpu_tc.py, over ragged, odd, even
      and single tiles, every wgmma width and the > 256-column launches, on ordered tables
      (K = 8 and 27) and on a K > 32 table without an order."""
import contextlib

import pytest
import torch

from helpers import TC_ACC, _pairs, assert_one_rounding, ref_conv, unique_cloud

pytestmark = pytest.mark.gpu

BIG_TILES = 200          # more 128-row tiles than an H100 has SMs: full-width CTAs


def _table(K, n_rows, n_other, density, seed, device):
    g = torch.Generator().manual_seed(seed)
    idx = torch.randint(0, n_other, (K, n_rows), generator=g, dtype=torch.int32)
    idx[torch.rand((K, n_rows), generator=g) > density] = -1
    return idx.to(device)


class _tf32:
    """fp32 operands multiplied in TF32 inside the block (the switch torch users set)."""

    def __enter__(self):
        self.saved = torch.backends.cuda.matmul.fp32_precision
        torch.backends.cuda.matmul.fp32_precision = "tf32"

    def __exit__(self, *exc):
        torch.backends.cuda.matmul.fp32_precision = self.saved


def _inputs(n_in, n_out, cin, cout, K, dtype, device, seed):
    g = torch.Generator().manual_seed(seed)
    feats = (torch.rand(n_in, cin, generator=g) - 0.5).to(dtype).to(device)
    gout = (torch.rand(n_out, cout, generator=g) - 0.5).to(dtype).to(device)
    w = ((torch.rand(K, cin, cout, generator=g) - 0.5) / cin ** 0.5).to(device)
    return feats, gout, w


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32])
@pytest.mark.parametrize("cin,cout", [(96, 96), (128, 256), (256, 384)])
def test_sliced_rows_equal_full_width_rows(ME, cuda, dtype, cin, cout):
    from minkowskiengine_b200 import _lib, backend
    K, n_small, n_other = 8, 5 * 128 + 77, 3000
    n_big = BIG_TILES * 128 + 5
    # forward: the small table is the first rows of the big one, over the same n_other input rows
    # (the reverse table only gives the maps their input row count)
    big = _table(K, n_big, n_other, 0.4, seed=cin + cout, device=cuda)
    small = big[:, :n_small].contiguous()
    rev = _table(K, n_other, n_small, 0.4, seed=5, device=cuda)
    feats, _, w = _inputs(n_other, 1, cin, cout, K, dtype, cuda, seed=cout)
    # dgrad: tables of input rows (the small one the first rows of the big one) into the same
    # n_other gradient rows, c_cols = cin
    big_in = _table(K, n_big, n_other, 0.4, seed=cin + cout + 1, device=cuda)
    x_big = (torch.rand(n_big, cin, device=cuda) - 0.5).to(dtype)
    _, gout, _ = _inputs(1, n_other, cin, cout, K, dtype, cuda, seed=cin)
    with _tf32() if dtype == torch.float32 else contextlib.nullcontext():
        n0 = _lib.tc_launch_count()
        for out_dtype in (None, torch.float32):
            a = backend._conv_forward(feats, w, backend._KernelMap(small, rev), out_dtype)
            b = backend._conv_forward(feats, w, backend._KernelMap(big, rev), out_dtype)
            assert torch.equal(a, b[:n_small]), f"forward ({out_dtype}): sliced rows differ"
        a, _ = backend._conv_backward(x_big[:n_small], gout, w,
                                      backend._KernelMap(rev, big_in[:, :n_small].contiguous()),
                                      need_in=True, need_w=False)
        b, _ = backend._conv_backward(x_big, gout, w, backend._KernelMap(rev, big_in),
                                      need_in=True, need_w=False)
        assert torch.equal(a, b[:n_small]), "dgrad: sliced rows differ"
        assert _lib.tc_launch_count() > n0, "did not take the tensor-core path"


def _manager_map(ME, cuda, n, ks, seed):
    coords = unique_cloud(n, 12, seed=seed)
    x = ME.SparseTensor(torch.zeros(len(coords), 1), coords, device=cuda)
    key = x.coordinate_map_key
    km = x.coordinate_manager._manager._kernel_map(
        key, key, [ks] * 3, [1] * 3, [1] * 3, ME.RegionType.HYPER_CUBE, torch.IntTensor(), False,
        False)
    assert km.out_order is not None and km.in_order is not None
    return km


# (rows of the map, kernel size or K of an unordered table): 128-row tiles 3 (odd), 2 (even) and
# 1, each ragged; K = 36 has no tile order; BIG_TILES runs full width
MAPS = [(300, 3), (250, 2), (90, 3), (1000, 36), (BIG_TILES * 128 + 9, 36)]


@pytest.mark.parametrize("c", [16, 48, 96, 128, 160, 256, 384])
@pytest.mark.parametrize("n,ks", MAPS)
def test_tiles_match_fp64(ME, cuda, c, n, ks):
    from minkowskiengine_b200 import backend
    dtype = torch.bfloat16
    if ks > 3:
        K = ks
        km = backend._KernelMap(_table(K, n, n, 0.3, seed=n, device=cuda),
                                _table(K, n, n, 0.3, seed=n + 1, device=cuda))
    else:
        km = _manager_map(ME, cuda, n, ks, seed=n + ks)
        K = km.K
        assert km.n_out % 128 != 0
    feats, gout, w = _inputs(km.n_in, km.n_out, c, c, K, dtype, cuda, seed=c + n)
    wq = w.to(dtype)
    y = backend._conv_forward(feats, w, km, out_dtype=torch.float32)
    ref, A = ref_conv(feats, wq, _pairs(km.out_nbr), km.n_out)
    assert_one_rounding(y, ref, A, f"forward c={c} n={n}", TC_ACC)
    gi, _ = backend._conv_backward(feats, gout, w, km, need_in=True, need_w=False)
    ref, A = ref_conv(gout, wq.transpose(1, 2), _pairs(km.in_nbr), km.n_in)
    assert_one_rounding(gi, ref, A, f"dgrad c={c} n={n}", TC_ACC)
