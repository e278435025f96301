"""Every instantiation of the wgmma convolution kernels, and the edges of their pipeline and row
splits, in bf16 / fp16 against float64, element by element.

`MEB_COLS_DISPATCH` (csrc/conv_tc.cu) maps c_cols / 16 = 1..16 to one (NI, NT) instantiation per
kernel and dtype, and for `k_conv_wg` per stage width bk = fwd_bk(c_red) in {16, 32, 64}
(csrc/tc_config.h).  The forward's columns are c_out and its reduction c_in; the dgrad's are c_in
and c_out; the wgrad's columns are c_out, its rows c_in in 128-channel m-tiles.  Layers wider
than 256 columns run in 256-column slices (forward / dgrad) or off the tensor cores (wgrad).
`test_cases_cover_the_dispatch_table` derives from the case list what each case reaches, so
dropping a case fails without a GPU.

Bound (tests/helpers.py): |y - ref| <= acc * 2^-20 * A, plus one rounding for bf16 / fp16
outputs, with acc = TC_ACC on the tensor cores and 1 on CUDA cores.  Every result must repeat
bitwise: forward and dgrad write each element once, the wgrad adds its splits in order."""
import math

import pytest
import torch

from helpers import (TC_ACC, _inputs, _pairs, _Route, _table, assert_one_rounding,
                     lib_conv_backward, ref_conv, ref_wgrad)

DTYPES = pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])

# name -> (c_in, c_out, forward on tensor cores, dgrad on tensor cores, wgrad on tensor cores)
CASES = {f"diag_{16 * i}x{16 * (17 - i)}": (16 * i, 16 * (17 - i), True, True, True)
         for i in range(1, 17)}
CASES.update({
    # forward slices past 256 columns; their wgrad (c_out > 256) runs on CUDA cores
    "fwd_slices_64x272": (64, 272, True, True, False),
    "fwd_slices_48x400": (48, 400, True, True, False),
    "fwd_slices_32x528": (32, 528, True, True, False),
    "fwd_slices_128x1024": (128, 1024, True, True, False),
    # the mirrors: dgrad slices, wgrad with 3, 4 and 8 m-tiles
    "dgrad_slices_272x64": (272, 64, True, True, True),
    "dgrad_slices_400x48": (400, 48, True, True, True),
    "dgrad_slices_1024x128": (1024, 128, True, True, True),
    # c_in % 16 == 8: forward and dgrad on CUDA cores, a ragged last m-tile of 8 channels
    "ragged_wgrad_136x32": (136, 32, False, False, True),
    "ragged_wgrad_264x80": (264, 80, False, False, True),
})


# ---- the dispatch rule, restated (tc_config.h: fwd_bk, conv_tc.cu: *_supported, kMaxCols) ------
def _fwd_bk(c_red):
    return 64 if c_red % 64 == 0 else 32 if c_red % 32 == 0 else 16 if c_red % 16 == 0 else 0


def _fwd_tc(c_red, c_cols):
    return _fwd_bk(c_red) > 0 and c_cols % 16 == 0 and 16 <= c_cols <= 1024


def _wgrad_tc(c_in, c_out):
    return c_in % 8 == 0 and c_in >= 16 and c_out % 16 == 0 and 16 <= c_out <= 256


def _slices(c_cols):
    """c_cols / 16 of every launch slice of at most 256 columns."""
    return [min(256, c_cols - n0) // 16 for n0 in range(0, c_cols, 256)]


def test_cases_cover_the_dispatch_table():
    reach = {"fwd": set(), "dgrad": set(), "wgrad": set()}
    bks = {"fwd": set(), "dgrad": set()}
    wgrad_m_tiles = set()
    for name, (cin, cout, fwd, dgrad, wgrad) in CASES.items():
        assert (fwd, dgrad, wgrad) == (_fwd_tc(cin, cout), _fwd_tc(cout, cin),
                                       _wgrad_tc(cin, cout)), f"{name}: stated route"
        if fwd:
            reach["fwd"].update(_slices(cout))
            bks["fwd"].add(_fwd_bk(cin))
        if dgrad:
            reach["dgrad"].update(_slices(cin))
            bks["dgrad"].add(_fwd_bk(cout))
        if wgrad:
            reach["wgrad"].add(cout // 16)
            wgrad_m_tiles.add((-(-cin // 128), cin % 128))
    for d, hit in reach.items():
        assert hit == set(range(1, 17)), f"{d}: column cases {sorted(set(range(1, 17)) - hit)} missed"
    for d, hit in bks.items():
        assert hit == {16, 32, 64}, f"{d}: stage widths {sorted({16, 32, 64} - hit)} missed"
    n_tiles = {t for t, _ in wgrad_m_tiles}
    assert {1, 2, 8} <= n_tiles, f"wgrad m-tile counts {sorted(n_tiles)}"
    assert any(t > 1 and r % 16 == 8 for t, r in wgrad_m_tiles), "no ragged 8-channel last m-tile"


# ---- one layer, every direction ---------------------------------------------------------------
def _acc(tc):
    return TC_ACC if tc else 1.0


def _run_layer(what, feats, gout, w, km, routes):
    """Forward (feature dtype and fp32), dgrad (feature dtype and fp32) and wgrad of one layer,
    each on its stated route, against float64, and each repeated bitwise."""
    from minkowskiengine_b200 import backend
    fwd_tc, dgrad_tc, wgrad_tc = routes
    wl = w.to(feats.dtype)
    ref, A = ref_conv(feats, wl, _pairs(km.out_nbr), km.n_out)
    with _Route(fwd_tc, f"{what} forward"):
        y = backend._conv_forward(feats, w, km)
        y2 = backend._conv_forward(feats, w, km)
        y32 = backend._conv_forward(feats, w, km, out_dtype=torch.float32)
    assert_one_rounding(y, ref, A, f"{what} forward", _acc(fwd_tc))
    assert_one_rounding(y32, ref, A, f"{what} forward, fp32 output", _acc(fwd_tc))
    assert torch.equal(y, y2), f"{what}: forward differs run to run"

    ref, A = ref_conv(gout, wl.transpose(1, 2), _pairs(km.in_nbr), km.n_in)
    with _Route(dgrad_tc, f"{what} dgrad"):
        gi, _ = backend._conv_backward(feats, gout, w, km, need_in=True, need_w=False)
        gi2, _ = backend._conv_backward(feats, gout, w, km, need_in=True, need_w=False)
        gi32, _ = lib_conv_backward(feats, gout, w, km, grad_in_dtype=torch.float32)
    assert_one_rounding(gi, ref, A, f"{what} dgrad", _acc(dgrad_tc))
    assert_one_rounding(gi32, ref, A, f"{what} dgrad, fp32 output", _acc(dgrad_tc))
    assert torch.equal(gi, gi2), f"{what}: dgrad differs run to run"

    ref, A = ref_wgrad(feats, gout, _pairs(km.out_nbr))
    with _Route(wgrad_tc, f"{what} wgrad"):
        _, gw = backend._conv_backward(feats, gout, w, km, need_in=False, need_w=True)
        _, gw2 = backend._conv_backward(feats, gout, w, km, need_in=False, need_w=True)
    assert_one_rounding(gw, ref, A, f"{what} wgrad", _acc(wgrad_tc))
    assert torch.equal(gw, gw2), f"{what}: wgrad differs run to run"


def _layer(cin, cout, n_in, n_out, K, dtype, device, seed, density=0.35):
    from minkowskiengine_b200 import backend
    feats, gout, w = _inputs(cin, cout, n_in, n_out, K, dtype, device, seed)
    km = backend._KernelMap(_table(K, n_out, n_in, density, seed + 1, device),
                            _table(K, n_in, n_out, density, seed + 2, device))
    return feats, gout, w, km


@pytest.mark.gpu
@DTYPES
@pytest.mark.parametrize("case", list(CASES))
def test_dispatch_case(ME, cuda, case, dtype):
    cin, cout, *routes = CASES[case]
    n = 2000 if max(cin, cout) > 512 else 3000
    feats, gout, w, km = _layer(cin, cout, n, n + 77, 27, dtype, cuda, seed=cin * 7 + cout)
    _run_layer(case, feats, gout, w, km, routes)


# ---- edges of the 4-stage ring and of the row tiles ---------------------------------------------
@pytest.mark.gpu
@DTYPES
@pytest.mark.parametrize("K", [1, 2, 3])
@pytest.mark.parametrize("c", [16, 32, 64])
def test_few_stages(ME, cuda, dtype, c, K):
    """c_in = c_out = bk: forward and dgrad have n_st = K stages, fewer than the ring preloads."""
    feats, gout, w, km = _layer(c, c, 1500, 1400, K, dtype, cuda, seed=c + K, density=0.6)
    _run_layer(f"{c}x{c} K={K}", feats, gout, w, km, (True, True, True))


@pytest.mark.gpu
@DTYPES
@pytest.mark.parametrize("n_out", [1, 127, 128, 129, 257])
def test_row_counts_with_one_input_row(ME, cuda, dtype, n_out):
    """Output tiles of 128 rows around their ends, all gathering input row 0 (n_in = 1)."""
    from minkowskiengine_b200 import backend
    K, cin, cout = 27, 64, 96
    feats, gout, w = _inputs(cin, cout, 1, n_out, K, dtype, cuda, seed=n_out)
    g = torch.Generator().manual_seed(n_out + 1)
    out_nbr = torch.where(torch.rand(K, n_out, generator=g) < 0.7, 0, -1).int().to(cuda)
    in_nbr = torch.randint(0, n_out, (K, 1), generator=g, dtype=torch.int32).to(cuda)
    km = backend._KernelMap(out_nbr, in_nbr)
    _run_layer(f"n_out={n_out}, n_in=1", feats, gout, w, km, (True, True, True))


@pytest.mark.gpu
@DTYPES
def test_wgrad_stage_shares(ME, cuda, dtype):
    """Offsets with 1, 64, 65, 128 and 129 pairs (one stage holds 64), and one with none: the
    pair-list and the dense-table wgrad."""
    from minkowskiengine_b200 import backend
    counts = [1, 64, 65, 0, 128, 129]
    K, n, cin, cout = len(counts), 1000, 144, 48
    feats, gout, w = _inputs(cin, cout, n, n, K, dtype, cuda, seed=65)
    g = torch.Generator().manual_seed(66)
    out_nbr = torch.full((K, n), -1, dtype=torch.int32)
    for k, c in enumerate(counts):
        rows = torch.randperm(n, generator=g)[:c]
        out_nbr[k, rows] = torch.randint(0, n, (c,), generator=g, dtype=torch.int32)
    out_nbr = out_nbr.to(cuda)
    km = backend._KernelMap(out_nbr, torch.full((K, n), -1, dtype=torch.int32, device=cuda))
    assert [int(c) for c in (out_nbr >= 0).sum(1)] == counts
    ref, A = ref_wgrad(feats, gout, _pairs(out_nbr))
    for pairs in (True, False):
        what = "pair-list" if pairs else "dense-table"
        with _Route(True, f"{what} wgrad"):
            _, gw = lib_conv_backward(feats, gout, w, km, need_w=True, pairs=pairs)
            _, gw2 = lib_conv_backward(feats, gout, w, km, need_w=True, pairs=pairs)
        assert_one_rounding(gw, ref, A, f"{what} wgrad", TC_ACC)
        assert torch.equal(gw, gw2), f"{what} wgrad differs run to run"
        assert not bool(gw[counts.index(0)].any()), f"{what}: an offset without pairs is not zero"


# ---- row splits and their workspace --------------------------------------------------------------
@pytest.mark.gpu
@DTYPES
def test_wgrad_split_workspaces(ME, cuda, dtype):
    """K = 1 at 60k rows plans far more than two splits.  No workspace, one that fits two splits,
    one offset by 8 bytes (not 16-byte aligned: one split) and the planned size must each meet the
    bound and repeat bitwise; the one-split runs must agree bitwise."""
    from minkowskiengine_b200 import _lib, backend
    K, n, cin, cout = 1, 60_000, 64, 64
    feats, gout, w = _inputs(cin, cout, n, n, K, dtype, cuda, seed=300)
    out_nbr = _table(K, n, n, 0.9, seed=301, device=cuda)
    km = backend._KernelMap(out_nbr, torch.full((K, n), -1, dtype=torch.int32, device=cuda))
    full = int(_lib.load().meb200_conv_workspace_bytes(n, cin, cout, K, _lib.dtype_code(dtype)))
    one = K * cin * cout * 4
    assert full >= 3 * one, "the layer no longer plans more than two splits"
    ws_full = torch.empty(full, dtype=torch.uint8, device=cuda)
    workspaces = {"none": None, "two splits": ws_full[:2 * one], "offset by 8 bytes": ws_full[8:],
                  "planned": ws_full}
    ref, A = ref_wgrad(feats, gout, _pairs(out_nbr))
    got = {}
    for name, ws in workspaces.items():
        for pairs in (True, False):
            what = f"{'pair-list' if pairs else 'dense-table'} wgrad, workspace {name}"
            with _Route(True, what):
                _, gw = lib_conv_backward(feats, gout, w, km, need_w=True, pairs=pairs, workspace=ws)
                _, gw2 = lib_conv_backward(feats, gout, w, km, need_w=True, pairs=pairs,
                                           workspace=ws)
            assert_one_rounding(gw, ref, A, what, TC_ACC)
            assert torch.equal(gw, gw2), f"{what}: differs run to run"
            got[name, pairs] = gw
    for pairs in (True, False):
        assert torch.equal(got["none", pairs], got["offset by 8 bytes", pairs]), \
            "a workspace the wgrad cannot use must give the one-split result"


@pytest.mark.gpu
@DTYPES
def test_low_density_pair_lists(ME, cuda, dtype, monkeypatch):
    """Density 0.002 at 200k rows, in chunks of 2048 table rows: the planned splits far exceed the
    pairs, so most shares are empty and must still store zeros into their slot, and some
    (chunk, offset) segments are empty."""
    from minkowskiengine_b200 import _lib, backend
    monkeypatch.setattr(backend._KernelMap, "PAIR_CHUNK_ROWS", 2048)
    K, n, cin, cout = 8, 200_000, 64, 64
    feats, gout, w = _inputs(cin, cout, n, n, K, dtype, cuda, seed=2)
    out_nbr = _table(K, n, n, 0.002, seed=3, device=cuda)
    km = backend._KernelMap(out_nbr, torch.full((K, n), -1, dtype=torch.int32, device=cuda))
    pin, pout, seg, nch = km.pair_lists()
    assert nch == -(-n // 2048)
    assert bool(((seg[1:] - seg[:-1]) == 0).any()), "no empty (chunk, offset) segment"
    ref, A = ref_wgrad(feats, gout, _pairs(out_nbr))
    with _Route(True, "low-density pair-list wgrad"):
        _, gw = backend._conv_backward(feats, gout, w, km, need_in=False, need_w=True)
        _, gw2 = backend._conv_backward(feats, gout, w, km, need_in=False, need_w=True)
    assert_one_rounding(gw, ref, A, "low-density pair-list wgrad", TC_ACC)
    assert torch.equal(gw, gw2)
    ws, _ = backend._workspace(n, cin, cout, K, _lib.dtype_code(dtype), cuda)
    with _Route(True, "low-density dense-table wgrad"):
        _, gd = lib_conv_backward(feats, gout, w, km, need_w=True, workspace=ws)
        _, gd2 = lib_conv_backward(feats, gout, w, km, need_w=True, workspace=ws)
    assert_one_rounding(gd, ref, A, "low-density dense-table wgrad", TC_ACC)
    assert torch.equal(gd, gd2)


# ---- fp16 range -------------------------------------------------------------------------------
def _scaled_fp16_layer(cuda, top_log2):
    """A 64 -> 64, K = 27 fp16 layer whose features and output gradients are multiplied by a
    power of two, and for small outputs its weights too, so that the largest |output| of the
    forward and the dgrad is about 2^top_log2.  Returns the layer and [(direction, output,
    float64 value, A)] of both."""
    from minkowskiengine_b200 import backend
    K, c, n = 27, 64, 3000
    feats, gout, w = _inputs(c, c, n, n, K, torch.float16, cuda, seed=16)
    km = backend._KernelMap(_table(K, n, n, 0.6, seed=17, device=cuda),
                            _table(K, n, n, 0.6, seed=18, device=cuda))
    wl = w.half()
    top = max(float(ref_conv(feats, wl, _pairs(km.out_nbr), n)[0].abs().max()),
              float(ref_conv(gout, wl.transpose(1, 2), _pairs(km.in_nbr), n)[0].abs().max()))
    e = math.floor(top_log2 - math.log2(top))     # largest |output| in (2^(top_log2 - 1), 2^top_log2]
    ew = e // 2 if e < 0 else 0
    feats = (feats.float() * 2.0 ** (e - ew)).half()
    gout = (gout.float() * 2.0 ** (e - ew)).half()
    w = w * 2.0 ** ew
    wl = w.half()
    with _Route(True, "fp16 forward / dgrad"):
        y = backend._conv_forward(feats, w, km)
        gi, _ = backend._conv_backward(feats, gout, w, km, need_in=True, need_w=False)
        assert torch.equal(y, backend._conv_forward(feats, w, km))
        assert torch.equal(gi, backend._conv_backward(feats, gout, w, km, True, False)[0])
    return [("forward", y, *ref_conv(feats, wl, _pairs(km.out_nbr), n)),
            ("dgrad", gi, *ref_conv(gout, wl.transpose(1, 2), _pairs(km.in_nbr), n))]


@pytest.mark.gpu
def test_fp16_outputs_near_the_top_of_the_range(ME, cuda):
    for what, y, ref, A in _scaled_fp16_layer(cuda, 15):
        top = float(ref.abs().max())
        assert 2.0 ** 14 < top < 65504, f"{what}: largest |ref| {top} not near the top of fp16"
        assert bool(torch.isfinite(y).all())
        assert_one_rounding(y, ref, A, f"fp16 {what} near 2^15", TC_ACC)


@pytest.mark.gpu
def test_fp16_subnormal_outputs(ME, cuda):
    for what, y, ref, A in _scaled_fp16_layer(cuda, -15):
        top = float(ref.abs().max())
        assert 2.0 ** -20 < top < 2.0 ** -14, f"{what}: largest |ref| {top} not subnormal in fp16"
        assert_one_rounding(y, ref, A, f"fp16 {what} below 2^-14", TC_ACC)


@pytest.mark.gpu
def test_fp16_overflow_gives_signed_inf(ME, cuda):
    """Outputs whose float64 value is past the fp16 range are +-inf, as ref.to(float16) is."""
    for what, y, ref, A in _scaled_fp16_layer(cuda, 17):
        delta = A * (TC_ACC * 2.0 ** -20)
        over = ref.abs() - delta >= 65520            # rounds to inf whatever the accumulation
        under = ref.abs() + delta < 65520
        assert bool((over & (ref > 0)).any()) and bool((over & (ref < 0)).any()), what
        expect = ref.to(torch.float16)
        assert bool(torch.isinf(expect[over]).all())
        assert torch.equal(y[over], expect[over]), f"fp16 {what}: overflow is not a signed inf"
        assert bool(torch.isfinite(y[under]).all())
        assert_one_rounding(y[under], ref[under], A[under], f"fp16 {what} in range", TC_ACC)
