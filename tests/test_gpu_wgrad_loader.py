"""The tensor-core weight gradients (k_wgrad_wg, k_wgrad_tf32) load each stage's index words one
stage before the copies that use them.  A pair that is dropped, taken twice, or taken from the
neighbouring stage changes dW, and these tests see every such change exactly: the operands lie on
a dyadic grid (features k / 8, gradients k / 4, |k| <= 8) where every product is a multiple of
2^-5 and every partial sum stays below 2^19, so each fp32 sum is exact whatever its order and dW
must equal its float64 restatement bit for bit.

Covered: pair mode over several row chunks, an offset without pairs, an offset with fewer stages
than row splits, and a heavy offset that runs in column slices; no workspace, the planned one and
one too small for the plan; every loader shape of the columns (c_out 16, 48, 96, 128, 256, of
which 16 and 48 do not fill the four threads of a row) and a ragged second channel tile
(c_in = 200); dense mode, stem mode; bf16, fp16 and TF32."""
import pytest
import torch

from helpers import _pairs, _Route, lib_conv_backward, ref_wgrad

pytestmark = pytest.mark.gpu

N = 6000            # table rows (input rows = output rows)
K = 27
HEAVY, EMPTY, SPARSE = 13, 5, 3
CHUNK_ROWS = 2048   # three row chunks in pair mode


def _grid(rows, cols, scale, g):
    return torch.randint(-8, 9, (rows, cols), generator=g).float() / scale


def _table(seed):
    """[K, N]: offset HEAVY pairs every row (more than twice the mean: column slices), EMPTY none,
    SPARSE a few dozen rows (one stage per chunk, fewer than the row splits), the rest 20 %."""
    g = torch.Generator().manual_seed(seed)
    nbr = torch.randint(0, N, (K, N), generator=g, dtype=torch.int32)
    nbr[torch.rand((K, N), generator=g) > 0.2] = -1
    nbr[SPARSE][torch.rand(N, generator=g) > 0.01] = -1
    nbr[EMPTY] = -1
    nbr[HEAVY] = torch.randperm(N, generator=g).int()
    return nbr


def _operands(c_in, c_out, dtype, seed, cuda):
    g = torch.Generator().manual_seed(seed)
    feats = _grid(N, c_in, 8, g).to(dtype).to(cuda)
    gout = _grid(N, c_out, 4, g).to(dtype).to(cuda)
    nbr = _table(seed).to(cuda)
    return feats, gout, nbr


def _workspace(kind, c_in, c_out, code, cuda):
    from minkowskiengine_b200 import _lib
    planned = int(_lib.load().meb200_conv_workspace_bytes(N, c_in, c_out, K, code))
    assert planned >= 3 * K * c_in * c_out * 4, "the case means to plan several row splits"
    if kind == "none":
        return None
    # "small": room for two of the planned splits
    n = planned if kind == "planned" else 2 * K * c_in * c_out * 4
    return torch.empty(n, dtype=torch.uint8, device=cuda)


def _backward(feats, gout, nbr, c_in, c_out, tf32, pairs, ws):
    """dW of the layer through meb200_conv_backward (wgrad only)."""
    from minkowskiengine_b200 import _lib, backend
    cuda = feats.device
    empty = torch.full((K, N), -1, dtype=torch.int32, device=cuda)
    km = backend._KernelMap(nbr, empty)
    w = torch.zeros(K, c_in, c_out, device=cuda)
    if not tf32:
        return lib_conv_backward(feats, gout, w, km, need_w=True, pairs=pairs, workspace=ws)[1]
    lib = _lib.load()
    w_cast, _ = backend._packed_weights(w, backend.TF32)
    gw = torch.empty((K, c_in, c_out), dtype=torch.float32, device=cuda)
    pin = pout = seg = None
    nch = 0
    if pairs:
        pin, pout, seg, nch = km.pair_lists()
    _lib.check(lib.meb200_conv_backward(
        _lib.ptr(feats), _lib.ptr(gout), _lib.TF32, N, c_in, _lib.ptr(w_cast), K, c_out,
        _lib.ptr(nbr), None, N, None, _lib.F32, _lib.ptr(gw), _lib.ptr(pin), _lib.ptr(pout),
        _lib.ptr(seg), nch, _lib.ptr(ws), 0 if ws is None else ws.numel(), None,
        _lib.current_stream()))
    return gw


def _check(dtype, c_in, c_out, ws_kind, pairs, cuda, monkeypatch):
    from minkowskiengine_b200 import _lib, backend
    monkeypatch.setattr(backend._KernelMap, "PAIR_CHUNK_ROWS", CHUNK_ROWS)
    tf32 = dtype == "tf32"
    feats, gout, nbr = _operands(c_in, c_out, torch.float32 if tf32 else dtype,
                                 c_in * 1000 + c_out, cuda)
    code = _lib.TF32 if tf32 else _lib.dtype_code(dtype)
    ws = _workspace(ws_kind, c_in, c_out, code, cuda)
    what = f"{dtype} {c_in}->{c_out} {'pairs' if pairs else 'dense'} ws={ws_kind}"
    if pairs:
        assert backend._KernelMap(nbr, nbr).pair_lists()[3] == 3, "three row chunks"
    with _Route(True, what):
        gw = _backward(feats, gout, nbr, c_in, c_out, tf32, pairs, ws)
    ref, _ = ref_wgrad(feats, gout, _pairs(nbr))
    bad = gw.double() != ref
    assert not bool(bad.any()), \
        f"{what}: {int(bad.sum())} elements differ, offsets {sorted(set(bad.nonzero()[:, 0].tolist()))}"
    return gw


WIDTHS = pytest.mark.parametrize("c_out", [16, 48, 96, 128, 256])
CHANNELS = pytest.mark.parametrize("c_in", [16, 96, 200])
WORKSPACES = pytest.mark.parametrize("ws_kind", ["none", "planned", "small"])


@WIDTHS
@CHANNELS
@WORKSPACES
def test_pairs_bf16(ME, cuda, c_in, c_out, ws_kind, monkeypatch):
    _check(torch.bfloat16, c_in, c_out, ws_kind, True, cuda, monkeypatch)


@WIDTHS
@pytest.mark.parametrize("dtype", [torch.float16, "tf32"], ids=["fp16", "tf32"])
def test_pairs_fp16_tf32(ME, cuda, dtype, c_out, monkeypatch):
    _check(dtype, 200, c_out, "planned", True, cuda, monkeypatch)


@pytest.mark.parametrize("c_in,c_out", [(16, 16), (96, 96), (200, 48), (96, 256)])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, "tf32"], ids=["bf16", "fp16", "tf32"])
@pytest.mark.parametrize("ws_kind", ["none", "planned"])
def test_dense(ME, cuda, dtype, c_in, c_out, ws_kind, monkeypatch):
    _check(dtype, c_in, c_out, ws_kind, False, cuda, monkeypatch)


def test_pairs_repeat_bitwise(ME, cuda, monkeypatch):
    a = _check(torch.bfloat16, 96, 96, "planned", True, cuda, monkeypatch)
    b = _check(torch.bfloat16, 96, 96, "planned", True, cuda, monkeypatch)
    assert torch.equal(a, b)


@pytest.mark.parametrize("c_out", [32, 48])
@pytest.mark.parametrize("K_stem", [27, 125])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def test_stem(ME, cuda, dtype, K_stem, c_out):
    """Stem mode (c_in = 3, fp32 master kernel): virtual channels 4 k + c over all rows."""
    from minkowskiengine_b200 import backend
    g = torch.Generator().manual_seed(K_stem + c_out)
    feats = _grid(N, 3, 8, g).to(dtype).to(cuda)
    gout = _grid(N, c_out, 4, g).to(dtype).to(cuda)
    nbr = torch.randint(0, N, (K_stem, N), generator=g, dtype=torch.int32)
    nbr[torch.rand((K_stem, N), generator=g) > 0.3] = -1
    nbr = nbr.to(cuda)
    w = torch.zeros(K_stem, 3, c_out, device=cuda)
    km = backend._KernelMap(nbr, torch.full((K_stem, N), -1, dtype=torch.int32, device=cuda))
    assert backend._is_stem(w, dtype)
    what = f"stem {dtype} K={K_stem} c_out={c_out}"
    with _Route(True, what):
        _, gw = backend._conv_backward(feats, gout, w, km, need_in=False, need_w=True)
    ref, _ = ref_wgrad(feats, gout, _pairs(nbr))
    bad = gw.double() != ref
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} elements differ"
