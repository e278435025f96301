"""The exact-fp32 convolution kernels (csrc/conv_simt.cu, csrc/chwise.cu) against float64, element
by element: the path of every fp32 layer under torch's default matmul switch, and of every fp32
layer off the tensor-core grid under TF32.

Two kinds of check:
  * the bound of tests/helpers.py, |y - ref| <= 2^-20 * A, A the same reduction over absolute
    values, on centred random operands, over the tile, row-split and workspace edges of
    `k_conv_gather_gemm` and `k_conv_wgrad`;
  * exact arithmetic: operands on a dyadic grid, sized so that every partial sum is an fp32 value
    (see `_grid`).  Then every fma is exact in any order and the result must equal float64 bit for
    bit: a dropped, duplicated or misrouted term shows however small it is, and one-signed
    operands, whose rounding errors do not cancel, can be tested too.
Every result must also repeat bit for bit."""
import pytest
import torch

import chwise_oracle as CO
from helpers import (_Route, _inputs, _pairs, _table, assert_one_rounding, lib_conv_backward,
                     one_rounding_ratio, ref_conv, ref_wgrad)

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def exact_fp32():
    """fp32 convolutions on the CUDA cores: torch's default matmul switch, restored afterwards."""
    saved = torch.backends.cuda.matmul.fp32_precision
    torch.backends.cuda.matmul.fp32_precision = "ieee"
    yield
    torch.backends.cuda.matmul.fp32_precision = saved


def _maps(K, n_rows, n_other, seed, device):
    """A forward map writing n_rows output rows from n_other input rows, and a dgrad map writing
    n_rows input-gradient rows from n_other output rows (random tables, tests/helpers.py)."""
    from minkowskiengine_b200 import backend
    empty = torch.full((K, n_other), -1, dtype=torch.int32, device=device)
    fwd = backend._KernelMap(_table(K, n_rows, n_other, 0.35, seed, device), empty)
    dgrad = backend._KernelMap(empty, _table(K, n_rows, n_other, 0.35, seed + 1, device))
    return fwd, dgrad


def _fwd(feats, w, km, what):
    from minkowskiengine_b200 import backend
    with _Route(False, what):
        y = backend._conv_forward(feats, w, km)
        y2 = backend._conv_forward(feats, w, km)
    assert torch.equal(y, y2), f"{what}: differs run to run"
    return y


def _dgrad(gout, w, km, what):
    from minkowskiengine_b200 import backend
    feats = torch.empty((km.n_in, w.shape[1]), device=gout.device)     # not read by the dgrad
    with _Route(False, what):
        gi, _ = backend._conv_backward(feats, gout, w, km, need_in=True, need_w=False)
        gi2, _ = backend._conv_backward(feats, gout, w, km, need_in=True, need_w=False)
    assert torch.equal(gi, gi2), f"{what}: differs run to run"
    return gi


# ---- k_conv_gather_gemm: TM = TN = 64 rows / columns, TK = 16 reduction channels per step --------
C_RED = [5, 15, 16, 17, 33, 100]
C_COLS = [1, 63, 64, 65, 130]
ROWS = [1, 63, 64, 65, 4097]
KS = [1, 27, 125, 343]
# Every pair of values of any two of the four lists occurs in some case (30 cases, not 600)
GG_CASES = [(C_RED[i], C_COLS[j], ROWS[(i + 2 * j) % 5], KS[(i + 3 * j) % 4])
            for i in range(len(C_RED)) for j in range(len(C_COLS))]


@pytest.mark.parametrize("c_red,c_cols,n_rows,K", GG_CASES)
def test_gather_gemm_forward_and_dgrad(ME, cuda, c_red, c_cols, n_rows, K):
    """The forward (c_red -> c_cols, TRANS_W = false) and the dgrad of the layer c_cols -> c_red
    (reduction over its c_red output channels, c_cols columns, TRANS_W = true), both writing
    n_rows rows."""
    km_f, km_d = _maps(K, n_rows, 3000, seed=c_red * 7 + c_cols + K, device=cuda)
    feats, _, w = _inputs(c_red, c_cols, 3000, n_rows, K, torch.float32, cuda, seed=c_red + K)
    what = f"gather-GEMM forward {c_red}->{c_cols} rows={n_rows} K={K}"
    y = _fwd(feats, w, km_f, what)
    ref, A = ref_conv(feats, w, _pairs(km_f.out_nbr), n_rows)
    assert_one_rounding(y, ref, A, what)
    r_f = one_rounding_ratio(y, ref, A)

    _, gout, wd = _inputs(c_cols, c_red, n_rows, 3000, K, torch.float32, cuda, seed=c_cols + K)
    what = f"gather-GEMM dgrad {c_red}->{c_cols} rows={n_rows} K={K}"
    gi = _dgrad(gout, wd, km_d, what)
    ref, A = ref_conv(gout, wd.transpose(1, 2), _pairs(km_d.in_nbr), n_rows)
    assert_one_rounding(gi, ref, A, what)
    print(f"fp32 ratio gather-GEMM c_red={c_red} c_cols={c_cols} rows={n_rows} K={K}: "
          f"fwd {r_f:.3f} dgrad {one_rounding_ratio(gi, ref, A):.3f}")


# ---- k_conv_wgrad: row splits and the workspace that holds them --------------------------------
def _wgrad_case(n_out, K, seed, device, c_in=65, c_out=130):
    """65 -> 130: two input-channel tiles and three output-channel tiles of 64."""
    from minkowskiengine_b200 import backend
    feats, gout, w = _inputs(c_in, c_out, 20_000, n_out, K, torch.float32, device, seed)
    km = backend._KernelMap(_table(K, n_out, 20_000, 0.5, seed, device),
                            torch.full((K, 20_000), -1, dtype=torch.int32, device=device))
    return feats, gout, w, km


def _lib_wgrad(feats, gout, w, km, workspace, what):
    with _Route(False, what):
        _, gw = lib_conv_backward(feats, gout, w, km, need_w=True, workspace=workspace)
        _, gw2 = lib_conv_backward(feats, gout, w, km, need_w=True, workspace=workspace)
    assert torch.equal(gw, gw2), f"{what}: differs run to run"
    return gw


def test_wgrad_one_split(ME, cuda):
    """Fewer than 128 rows: one split, written to dW directly (the library plans no workspace)."""
    from minkowskiengine_b200 import _lib
    feats, gout, w, km = _wgrad_case(100, 27, 3, cuda)
    assert int(_lib.load().meb200_conv_workspace_bytes(100, 65, 130, 27, _lib.F32)) == 0
    gw = _lib_wgrad(feats, gout, w, km, None, "wgrad one split")
    ref, A = ref_wgrad(feats, gout, _pairs(km.out_nbr))
    assert_one_rounding(gw, ref, A, "wgrad one split")
    print(f"fp32 ratio k_conv_wgrad one split, 100 rows: {one_rounding_ratio(gw, ref, A):.3f}")


def test_wgrad_workspace_full_small_none_and_unaligned(ME, cuda):
    """120k rows, K = 4: the planned splits with the planned workspace, two splits with room for
    two, and one split without a workspace or with one that is not 16-byte aligned."""
    from minkowskiengine_b200 import _lib
    n_out, K, c_in, c_out = 120_000, 4, 65, 130
    feats, gout, w, km = _wgrad_case(n_out, K, 4, cuda)
    nbytes = int(_lib.load().meb200_conv_workspace_bytes(n_out, c_in, c_out, K, _lib.F32))
    slot = K * c_in * c_out * 4
    assert nbytes >= 3 * slot, "the plan should split this layer's rows"
    ref, A = ref_wgrad(feats, gout, _pairs(km.out_nbr))
    runs = {
        "full": torch.empty(nbytes, dtype=torch.uint8, device=cuda),
        "two slots": torch.empty(2 * slot, dtype=torch.uint8, device=cuda),
        "none": None,
        "unaligned": torch.empty(nbytes + 16, dtype=torch.uint8, device=cuda)[8:8 + nbytes],
    }
    gws = {}
    for what, ws in runs.items():
        gws[what] = _lib_wgrad(feats, gout, w, km, ws, f"wgrad workspace {what}")
        assert_one_rounding(gws[what], ref, A, f"wgrad workspace {what}")
    assert torch.equal(gws["none"], gws["unaligned"])      # both mean one split
    print("fp32 ratio k_conv_wgrad over 120k rows: " + ", ".join(
        f"{k} {one_rounding_ratio(v, ref, A):.3f}" for k, v in gws.items()))


def test_empty_output_map(ME, cuda):
    """n_out = 0: the forward launches nothing, the weight gradient is zero and the input
    gradient (no input row has a neighbour) is zero."""
    from minkowskiengine_b200 import _lib, backend
    K, c_in, c_out, n_in = 27, 20, 40, 500
    feats, _, w = _inputs(c_in, c_out, n_in, 0, K, torch.float32, cuda, seed=9)
    gout = torch.empty((0, c_out), device=cuda)
    km = backend._KernelMap(torch.empty((K, 0), dtype=torch.int32, device=cuda),
                            torch.full((K, n_in), -1, dtype=torch.int32, device=cuda))
    n0 = _lib.launch_count()
    y = backend._conv_forward(feats, w, km)
    torch.cuda.synchronize()
    assert _lib.launch_count() == n0 and y.shape == (0, c_out)
    gw_out = torch.full((K, c_in, c_out), float("nan"), device=cuda)
    gi, gw = lib_conv_backward(feats, gout, w, km, grad_in_dtype=torch.float32, need_w=True,
                               grad_w=gw_out)
    assert gw is gw_out and torch.equal(gw, torch.zeros_like(gw))
    assert torch.equal(gi, torch.zeros_like(gi))


# ---- exact arithmetic ------------------------------------------------------------------------------
# Operands k / 8 (features, gradients) and k / 16 (weights), k an integer with |k| <= 8.  A product
# of two of them is an integer multiple of q (1/128 or 1/64) at most 64 q in magnitude, and a sum of
# n products is a multiple of q at most 64 n q in magnitude.  fp32 holds every multiple m q with
# |m| <= 2^24, so with n <= MAX_TERMS = 2^24 / 64 terms per output every partial sum is an fp32 value:
# each fma is exact, in any order and over any split, and so is the float64 reference.
MAX_TERMS = 2 ** 18


def _grid(shape, denom, seed, device, one_signed=False):
    """k / denom, k uniform over the integers of [-8, 8] ([0, 8] when one-signed)."""
    g = torch.Generator().manual_seed(seed)
    k = torch.randint(0 if one_signed else -8, 9, shape, generator=g)
    return (k.float() / denom).to(device)


def _exact_operands(c_in, c_out, n_in, n_out, K, seed, device, one_signed):
    return (_grid((n_in, c_in), 8, seed, device, one_signed),
            _grid((n_out, c_out), 8, seed + 1, device, one_signed),
            _grid((K, c_in, c_out), 16, seed + 2, device, one_signed))


def _assert_exact(y, ref, terms, what):
    assert terms <= MAX_TERMS, f"{what}: {terms} terms per output is too many to be exact"
    if not torch.equal(y.double(), ref):
        bad = y.double() != ref
        j = int(torch.nonzero(bad.flatten())[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements differ from "
                             f"float64; first at flat index {j}: got {y.flatten()[j].item()!r}, "
                             f"float64 {ref.flatten()[j].item()!r}")


# (c_in, c_out, n_out, K): gather-GEMM forward and dgrad; k_conv_small_cin_fwd for c_in <= 4,
# c_out <= 64 (one and two 32-channel slabs), except the shared-memory fallback 4 -> 56, K = 343
# (K c_in 64 fp32 weights are more than 200 KB), which runs the gather-GEMM
EXACT_CONV = [(5, 1, 4097, 343), (17, 65, 1000, 27), (100, 130, 700, 125), (64, 64, 3000, 27),
              (1, 32, 5000, 125), (2, 20, 5000, 27), (3, 33, 5000, 125), (4, 64, 5000, 27),
              (4, 56, 5000, 343), (3, 72, 5000, 27)]


@pytest.mark.parametrize("one_signed", [False, True], ids=["signed", "one_signed"])
@pytest.mark.parametrize("c_in,c_out,n_out,K", EXACT_CONV)
def test_exact_forward_and_dgrad(ME, cuda, c_in, c_out, n_out, K, one_signed):
    n_in = 3000
    feats, gout, w = _exact_operands(c_in, c_out, n_in, n_out, K, c_in + c_out + K, cuda,
                                     one_signed)
    from minkowskiengine_b200 import backend
    out_nbr = _table(K, n_out, n_in, 0.5, seed=K + c_out, device=cuda)
    in_nbr = _table(K, n_in, n_out, 0.5, seed=K + c_in, device=cuda)
    km = backend._KernelMap(out_nbr, in_nbr)
    what = f"exact forward {c_in}->{c_out} K={K}"
    ref, _ = ref_conv(feats, w, _pairs(out_nbr), n_out)
    _assert_exact(_fwd(feats, w, km, what), ref, K * c_in, what)
    what = f"exact dgrad {c_in}->{c_out} K={K}"
    ref, _ = ref_conv(gout, w.transpose(1, 2), _pairs(in_nbr), n_in)
    _assert_exact(_dgrad(gout, w, km, what), ref, K * c_out, what)


# (c_in, c_out, n_out, K): k_conv_wgrad with one split (n_out < 128) and with many;
# k_conv_small_cin_wgrad for c_in 1 to 4, one and two slabs, one row slice and several
EXACT_WGRAD = [(65, 130, 100, 27), (65, 130, 120_000, 4), (20, 40, 200_000, 1),
               (1, 32, 100, 125), (2, 20, 50_000, 27), (3, 33, 50_000, 125), (4, 64, 200_000, 8),
               (4, 56, 20_000, 343), (3, 72, 50_000, 27)]


@pytest.mark.parametrize("one_signed", [False, True], ids=["signed", "one_signed"])
@pytest.mark.parametrize("c_in,c_out,n_out,K", EXACT_WGRAD)
def test_exact_wgrad(ME, cuda, c_in, c_out, n_out, K, one_signed):
    """Through the backend, which passes the planned workspace: the row splits and their sum
    (launch_split_sum) are exact too."""
    from minkowskiengine_b200 import backend
    n_in = 20_000
    feats, gout, w = _exact_operands(c_in, c_out, n_in, n_out, K, c_in * c_out + K, cuda,
                                     one_signed)
    out_nbr = _table(K, n_out, n_in, 0.6, seed=n_out + K, device=cuda)
    km = backend._KernelMap(out_nbr, torch.full((K, n_in), -1, dtype=torch.int32, device=cuda))
    what = f"exact wgrad {c_in}->{c_out} rows={n_out} K={K}"
    with _Route(False, what):
        _, gw = backend._conv_backward(feats, gout, w, km, need_in=False, need_w=True)
        _, gw2 = backend._conv_backward(feats, gout, w, km, need_in=False, need_w=True)
    assert torch.equal(gw, gw2), f"{what}: differs run to run"
    ref, _ = ref_wgrad(feats, gout, _pairs(out_nbr))
    _assert_exact(gw, ref, n_out, what)


def _chwise_gather(x, W, nbr):
    from minkowskiengine_b200 import _lib
    K, n_rows = nbr.shape
    y = torch.empty((n_rows, x.shape[1]), dtype=x.dtype, device=x.device)
    _lib.check(_lib.load().meb200_chwise_gather(
        _lib.ptr(x), _lib.F32, x.shape[0], x.shape[1], _lib.ptr(W), _lib.ptr(nbr), K, n_rows,
        _lib.ptr(y), _lib.current_stream()))
    return y


def _chwise_wgrad(x, g, nbr):
    from minkowskiengine_b200 import _lib
    lib = _lib.load()
    K, n_out = nbr.shape
    C = x.shape[1]
    nbytes = int(lib.meb200_chwise_wgrad_workspace_bytes(n_out, C, K, _lib.F32))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=x.device) if nbytes else None
    dW = torch.empty((K, C), dtype=torch.float32, device=x.device)
    _lib.check(lib.meb200_chwise_wgrad(
        _lib.ptr(x), _lib.ptr(g), _lib.F32, x.shape[0], C, _lib.ptr(nbr), K, n_out, _lib.ptr(dW),
        _lib.ptr(ws), nbytes, _lib.current_stream()))
    return dW


@pytest.mark.parametrize("one_signed", [False, True], ids=["signed", "one_signed"])
@pytest.mark.parametrize("C,K,n_out", [(12, 27, 50_000), (4, 343, 3000), (5, 27, 50_000),
                                       (1, 125, 3000), (64, 8, 200_000)])
def test_exact_channelwise(cuda, C, K, n_out, one_signed):
    """k_chwise_gather and k_chwise_wgrad in fp32: 16-byte vectors of 4 channels (C % 4 == 0) and
    single channels (C = 5, 1), with the planned row splits."""
    n_in = 20_000
    x, g, _ = _exact_operands(C, C, n_in, n_out, 1, C + K, cuda, one_signed)
    W = _grid((K, C), 16, C + K + 3, cuda, one_signed)
    out_nbr = _table(K, n_out, n_in, 0.5, seed=C * K, device=cuda)
    y = _chwise_gather(x, W, out_nbr)
    assert torch.equal(y, _chwise_gather(x, W, out_nbr))
    _assert_exact(y, CO.gather(x, W, out_nbr)[0], K, f"exact chwise gather C={C} K={K}")
    dW = _chwise_wgrad(x, g, out_nbr)
    assert torch.equal(dW, _chwise_wgrad(x, g, out_nbr))
    _assert_exact(dW, CO.wgrad(x, g, out_nbr)[0], n_out, f"exact chwise wgrad C={C} K={K}")
