"""fp32 convolutions on the tensor cores in TF32, chosen by torch's float32 matmul switch
(`torch.backends.cuda.matmul.fp32_precision == "tf32"`).

Element-wise bounds against a float64 restatement (tests/helpers.py), A the same reduction over
absolute values:
  * operands already tf32-representable (low 13 mantissa bits zero): products are exact, so only
    the accumulation errs, as on the bf16 / fp16 path: |y - ref| <= TC_ACC * 2^-20 * A;
  * arbitrary fp32 operands: each product also carries the reduction of its two factors to tf32
    (weights rounded to nearest when packed, features and gradients reduced by the tensor cores),
    at most 2^-9 relative: |y - ref| <= (2^-9 + TC_ACC * 2^-20) * A.
Every test that sets the switch restores the previous value."""
import numpy as np
import pytest
import torch

from examples.minkunet import minkunet
from helpers import (TC_ACC, _Route, _pairs, _table, assert_one_rounding, golden, ref_conv,
                     ref_wgrad, state_digest, unique_cloud)
from oracle import oracle_np as O

pytestmark = pytest.mark.gpu

ACC_ANY = TC_ACC + 2.0 ** 11           # 2^-9 = 2^11 * 2^-20


@pytest.fixture
def tf32():
    saved = torch.backends.cuda.matmul.fp32_precision
    torch.backends.cuda.matmul.fp32_precision = "tf32"
    yield
    torch.backends.cuda.matmul.fp32_precision = saved


def _tf32_exact(t):
    """t with the low 13 mantissa bits cleared: a tf32-representable fp32 tensor."""
    return (t.contiguous().view(torch.int32) & ~0x1FFF).view(torch.float32)


def _ratio(y, ref, A):
    """max |y - ref| / (2^-20 A) (the bound's unit), over elements with A > 0."""
    err = (y.double() - ref.double()).abs()
    unit = A.double() * 2.0 ** -20
    m = unit > 0
    return float((err[m] / unit[m]).max()) if bool(m.any()) else 0.0


def _lib_forward(feats, w, nbr, n_out, order=None):
    from minkowskiengine_b200 import _lib, backend
    lib = _lib.load()
    K, c_in, c_out = w.shape
    w_cast, w_t = backend._packed_weights(w, backend.TF32)
    out = torch.empty((n_out, c_out), dtype=torch.float32, device=feats.device)
    _lib.check(lib.meb200_conv_forward(
        _lib.ptr(feats), _lib.TF32, feats.shape[0], c_in, _lib.ptr(w_cast), _lib.ptr(w_t), K, c_out,
        _lib.ptr(nbr), n_out, _lib.ptr(out), _lib.F32, _lib.ptr(order), _lib.current_stream()))
    return out


def _lib_backward(feats, gout, w, out_nbr, in_nbr, need_in, need_w, pairs=False, workspace=None):
    """meb200_conv_backward with the TF32 code; workspace: None, or a uint8 tensor."""
    from minkowskiengine_b200 import _lib, backend
    lib = _lib.load()
    K, c_in, c_out = w.shape
    n_in, n_out = feats.shape[0], gout.shape[0]
    w_cast, _ = backend._packed_weights(w, backend.TF32)
    gi = torch.empty((n_in, c_in), dtype=torch.float32, device=feats.device) if need_in else None
    gw = torch.empty((K, c_in, c_out), dtype=torch.float32, device=feats.device) if need_w else None
    pin = pout = seg = None
    nch = 0
    if pairs:
        assert lib.meb200_conv_wgrad_uses_pairs(_lib.TF32, c_in, c_out, K) == 1
        pin, pout, seg, nch = backend._KernelMap(out_nbr, in_nbr).pair_lists()
    _lib.check(lib.meb200_conv_backward(
        _lib.ptr(feats), _lib.ptr(gout), _lib.TF32, n_in, c_in, _lib.ptr(w_cast), K, c_out,
        _lib.ptr(out_nbr), _lib.ptr(in_nbr) if need_in else None, n_out, _lib.ptr(gi), _lib.F32,
        _lib.ptr(gw), _lib.ptr(pin), _lib.ptr(pout), _lib.ptr(seg), nch, _lib.ptr(workspace),
        0 if workspace is None else workspace.numel(), None, _lib.current_stream()))
    return gi, gw


def _operands(c_in, c_out, n_in, n_out, K, seed, cuda, exact):
    g = torch.Generator().manual_seed(seed)
    feats = (torch.rand(n_in, c_in, generator=g) - 0.5) * 4
    gout = torch.rand(n_out, c_out, generator=g) - 0.5
    w = (torch.rand(K, c_in, c_out, generator=g) - 0.5) / c_in ** 0.5
    if exact:
        feats, gout, w = _tf32_exact(feats), _tf32_exact(gout), _tf32_exact(w)
    return feats.to(cuda), gout.to(cuda), w.to(cuda)


def _inverse(nbr, n_in):
    """in_nbr[k][i] = some o with out_nbr[k][o] = i, or -1."""
    K, n_out = nbr.shape
    inv = torch.full((K, n_in), -1, dtype=torch.int32, device=nbr.device)
    for k in range(K):
        o = torch.nonzero(nbr[k] >= 0).flatten()
        inv[k, nbr[k][o].long()] = o.int()
    return inv


def _injective(nbr, n_in):
    """nbr with every input row used at most once per offset (a real kernel map's property)."""
    inv = _inverse(nbr, n_in)
    out = torch.full_like(nbr, -1)
    for k in range(nbr.shape[0]):
        i = torch.nonzero(inv[k] >= 0).flatten()
        out[k, inv[k][i].long()] = i.int()
    return out, inv


# (c_red, c_cols, K): every forward instantiation (columns 16..256 in steps of 16, 384 for the
# column slices), every stage width (8, 16, 32 fp32 channels and wider multiples), K 1 / 8 / 27 / 125
FWD_CASES = [(8, 16, 27), (16, 32, 8), (24, 48, 1), (32, 64, 27), (40, 80, 8), (64, 96, 125),
             (96, 112, 27), (128, 128, 8), (8, 144, 27), (16, 160, 1), (48, 176, 27),
             (256, 192, 8), (32, 208, 27), (72, 224, 8), (128, 240, 27), (384, 256, 8),
             (64, 384, 27)]


@pytest.mark.parametrize("exact", [True, False], ids=["representable", "arbitrary"])
@pytest.mark.parametrize("c_red,c_cols,K", FWD_CASES)
def test_forward_and_dgrad_bounds(ME, cuda, tf32, c_red, c_cols, K, exact):
    """Forward (reduction c_red, c_cols output columns) and the dgrad of the transposed layer
    (reduction c_red = its c_out, c_cols = its c_in columns) on random tables with empty rows,
    an empty offset and a ragged last tile; both run twice and must repeat bit for bit."""
    n_in, n_out = 1500, 1000 + c_red % 7
    feats, _, w = _operands(c_red, c_cols, n_in, n_out, K, c_red * 31 + c_cols, cuda, exact)
    nbr, inv = _injective(_table(K, n_out, n_in, 0.4, c_cols + K, cuda), n_in)
    acc = TC_ACC if exact else ACC_ANY
    with _Route(True, "tf32 forward"):
        y = _lib_forward(feats, w, nbr, n_out)
    ref, A = ref_conv(feats, w, _pairs(nbr), n_out)
    assert_one_rounding(y, ref, A, f"tf32 forward {c_red}->{c_cols} K={K}", acc)
    assert torch.equal(y, _lib_forward(feats, w, nbr, n_out)), "forward differs run to run"
    # dgrad: the layer W'[k] = w[k]^T ([K, c_cols, c_red]) maps c_cols -> c_red channels; its
    # input gradient reduces over c_red and writes c_cols columns
    wt = w.transpose(1, 2).contiguous()
    x2 = torch.zeros(n_out, c_cols, device=cuda)       # the layer's input (unused by dgrad)
    gi, _ = _lib_backward(x2, feats, wt, inv, nbr, need_in=True, need_w=False)
    ref_g, A_g = ref, A                                 # the same sums
    assert_one_rounding(gi, ref_g, A_g, f"tf32 dgrad {c_red}->{c_cols} K={K}", acc)
    gi2, _ = _lib_backward(x2, feats, wt, inv, nbr, need_in=True, need_w=False)
    assert torch.equal(gi, gi2), "dgrad differs run to run"
    print(f"\n[tf32 {'exact' if exact else 'any'} fwd {c_red}->{c_cols} K={K}] "
          f"err/2^-20A fwd {_ratio(y, ref, A):.3f} dgrad {_ratio(gi, ref_g, A_g):.3f}")


# (c_in, c_out, K): every wgrad instantiation (c_out 16..256), one and two 128-channel tiles
WG_CASES = [(16, 16, 27), (24, 32, 8), (32, 48, 27), (40, 64, 1), (64, 80, 8), (96, 96, 27),
            (128, 112, 125), (136, 128, 8), (256, 144, 27), (32, 160, 8), (64, 176, 1),
            (128, 192, 27), (16, 208, 8), (96, 224, 27), (200, 240, 8), (256, 256, 27)]


@pytest.mark.parametrize("exact", [True, False], ids=["representable", "arbitrary"])
@pytest.mark.parametrize("c_in,c_out,K", WG_CASES)
def test_wgrad_bounds(ME, cuda, tf32, c_in, c_out, K, exact):
    """wgrad over the pair lists and over the dense table, with no, a small and a full
    workspace (one split, fewer, all planned): every variant inside the bound, and each one
    bit-identical when repeated."""
    from minkowskiengine_b200 import _lib
    n_in, n_out = 3000, 5000 + c_in
    feats, gout, w = _operands(c_in, c_out, n_in, n_out, K, c_in * 17 + c_out, cuda, exact)
    nbr, inv = _injective(_table(K, n_out, n_in, 0.5, c_out + K, cuda), n_in)
    ref, A = ref_wgrad(feats, gout, _pairs(nbr))
    acc = TC_ACC if exact else ACC_ANY
    full = int(_lib.load().meb200_conv_workspace_bytes(n_out, c_in, c_out, K, _lib.TF32))
    per_split = K * c_in * c_out * 4
    worst = 0.0
    for pairs in (True, False):
        for ws_bytes in (None, 2 * per_split, full):
            ws = None if ws_bytes is None else torch.empty(max(ws_bytes, 16), dtype=torch.uint8,
                                                          device=cuda)
            with _Route(True, "tf32 wgrad"):
                _, gw = _lib_backward(feats, gout, w, nbr, inv, False, True, pairs, ws)
            what = f"tf32 wgrad {c_in}->{c_out} K={K} pairs={pairs} ws={ws_bytes}"
            assert_one_rounding(gw, ref, A, what, acc)
            _, gw2 = _lib_backward(feats, gout, w, nbr, inv, False, True, pairs, ws)
            assert torch.equal(gw, gw2), what + ": differs run to run"
            worst = max(worst, _ratio(gw, ref, A))
    print(f"\n[tf32 {'exact' if exact else 'any'} wgrad {c_in}->{c_out} K={K}] "
          f"err/2^-20A {worst:.3f}")


def test_hardware_reduction_of_fp32_operands_to_tf32(ME, cuda, tf32):
    """Records how the tensor cores reduce fp32 features to tf32 (the packed weights are rounded
    by cvt.rna when packed): x = +-(1 + 0.75 ulp_tf32) times the weight 1.  Truncation reads it as
    +-1, rounding to nearest as +-(1 + 2^-10).  The forward reads features through wgmma, the wgrad
    through mma.sync; both are reported."""
    v = 1.0 + 3 * 2.0 ** -12
    nbr = torch.arange(128, dtype=torch.int32, device=cuda).view(1, 128)
    x = torch.zeros(128, 16, device=cuda)
    x[:, 0] = v
    x[1::2, 0] = -v
    w = torch.zeros(1, 16, 16, device=cuda)
    w[0, 0, :] = 1.0
    fwd = {float(t) for t in _lib_forward(x, w, nbr, 128)[:, 0].abs().cpu()}
    g = torch.zeros(128, 16, device=cuda)
    g[0::2, 0] = 1.0                                   # the positive rows only
    _, gw = _lib_backward(x, g, w, nbr, nbr, False, True)
    wg = float(gw[0, 0, 0]) / 64
    print(f"\n[tf32 feature reduction] 1 + 3*2^-12 read as: forward {sorted(fwd)}, wgrad {wg!r}")
    assert len(fwd) == 1 and fwd <= {1.0, 1.0 + 2.0 ** -10}
    assert wg in (1.0, 1.0 + 2.0 ** -10)


def _layer_case(ME, cuda, cin, cout, n=3000, seed=4, ks=3):
    coords = unique_cloud(n, 20, seed=seed)
    g = torch.Generator().manual_seed(seed)
    feats = torch.rand(len(coords), cin, generator=g)
    conv = ME.MinkowskiConvolution(cin, cout, kernel_size=ks, dimension=3).to(cuda)
    x = ME.SparseTensor(feats, coords, device=cuda, requires_grad=True)
    return conv, x


def _fwd_bwd(conv, x):
    y = conv(x)
    y.F.backward(torch.ones_like(y.F))
    return y


def _tf32_rna(t):
    """t rounded to the nearest tf32 value, ties away from zero, as cvt.rna rounds the packed
    weights: add half of the lowest kept mantissa bit to the magnitude, then clear the 13 dropped
    bits."""
    return ((t.contiguous().view(torch.int32) + 0x1000) & ~0x1FFF).view(torch.float32)


# Which directions of a layer run on the tensor cores under "tf32": (forward, dgrad, wgrad).
# 24 -> 48 is split: its dgrad writes 24 columns, off the 16-column grid.
_TF32_DIRECTIONS = {(32, 64): (True, True, True), (64, 32): (True, True, True),
                    (3, 32): (False, False, False), (32, 20): (False, False, False),
                    (24, 48): (True, False, True)}


@pytest.mark.parametrize("cin,cout,tc", [(32, 64, True), (64, 32, True), (3, 32, False),
                                         (32, 20, False), (24, 48, True)])
def test_route_follows_the_switch(ME, cuda, cin, cout, tc):
    """Default switch: an fp32 convolution launches no tensor-core kernel, forward or backward.
    "tf32": on-grid shapes launch some; the stem (c_in = 3) and c_out = 20 launch none.

    Per direction on the layer's kernel map, under "tf32": a forward or dgrad off the grid runs
    the exact CUDA-core kernels on the packed weights, which are rounded to tf32, so it equals bit
    for bit the default switch on the rounded weights; an off-grid wgrad reads no weights and
    equals the default switch's."""
    from minkowskiengine_b200 import backend
    saved = torch.backends.cuda.matmul.fp32_precision
    try:
        torch.backends.cuda.matmul.fp32_precision = "none"
        conv, x = _layer_case(ME, cuda, cin, cout)
        with _Route(False, f"fp32 {cin}->{cout} default"):
            _fwd_bwd(conv, x)
        torch.backends.cuda.matmul.fp32_precision = "tf32"
        x.F.grad = None
        with _Route(tc, f"fp32 {cin}->{cout} tf32"):
            _fwd_bwd(conv, x)

        key = x.coordinate_map_key
        km = x.coordinate_manager._manager._kernel_map(
            key, key, [3] * 3, [1] * 3, [1] * 3, ME.RegionType.HYPER_CUBE, torch.IntTensor(),
            False, False)
        feats = x.F.detach()
        g = torch.Generator().manual_seed(cin + cout)
        gout = (torch.rand(km.n_out, cout, generator=g) - 0.5).to(cuda)
        fwd_tc, dgrad_tc, wgrad_tc = _TF32_DIRECTIONS[(cin, cout)]
        with _Route(fwd_tc, f"tf32 {cin}->{cout} forward"):
            y = backend._conv_forward(feats, conv.kernel, km)
        with _Route(dgrad_tc, f"tf32 {cin}->{cout} dgrad"):
            gi, _ = backend._conv_backward(feats, gout, conv.kernel, km, need_in=True, need_w=False)
        with _Route(wgrad_tc, f"tf32 {cin}->{cout} wgrad"):
            _, gw = backend._conv_backward(feats, gout, conv.kernel, km, need_in=False, need_w=True)

        torch.backends.cuda.matmul.fp32_precision = "none"
        w_rna = _tf32_rna(conv.kernel.detach())
        assert not torch.equal(w_rna, conv.kernel.detach())     # the rounding changes something
        with _Route(False, f"fp32 {cin}->{cout} default, per direction"):
            y_rna = backend._conv_forward(feats, w_rna, km)
            gi_rna, _ = backend._conv_backward(feats, gout, w_rna, km, need_in=True, need_w=False)
            _, gw_exact = backend._conv_backward(feats, gout, conv.kernel, km, need_in=False,
                                                 need_w=True)
        if not fwd_tc:
            assert torch.equal(y, y_rna), "off-grid tf32 forward differs from fp32 on tf32 weights"
        if not dgrad_tc:
            assert torch.equal(gi, gi_rna), "off-grid tf32 dgrad differs from fp32 on tf32 weights"
        if not wgrad_tc:
            assert torch.equal(gw, gw_exact), "off-grid tf32 wgrad differs from the fp32 wgrad"
    finally:
        torch.backends.cuda.matmul.fp32_precision = saved


@pytest.mark.parametrize("stride,transpose", [(1, False), (2, False), (2, True)])
def test_tile_order_gives_the_same_bits_and_the_bound(ME, cuda, tf32, stride, transpose):
    """Manager kernel maps (tile-ordered tables, K <= 32) against the same tables without their
    orders: forward and dgrad bitwise equal; forward within the bound of arbitrary operands."""
    from minkowskiengine_b200 import backend
    coords = unique_cloud(9000, 30, seed=7)
    x = ME.SparseTensor(torch.zeros(len(coords), 1), coords, device=cuda)
    mgr, key = x.coordinate_manager, x.coordinate_map_key
    other = key if stride == 1 else mgr.stride(key, stride)
    ik, ok = (other, key) if transpose else (key, other)
    km = mgr._manager._kernel_map(ik, ok, [3 if stride == 1 else 2] * 3, [stride] * 3, [1] * 3,
                                  ME.RegionType.HYPER_CUBE, torch.IntTensor(), transpose, False)
    assert km.out_order is not None and km.in_order is not None
    plain = backend._KernelMap(km.out_nbr, km.in_nbr)
    feats, gout, w = _operands(64, 96, km.n_in, km.n_out, km.K, 11, cuda, exact=False)
    a = backend._conv_forward(feats, w, km)
    b = backend._conv_forward(feats, w, plain)
    assert torch.equal(a, b), "forward differs with the tile order"
    ref, A = ref_conv(feats, w, _pairs(km.out_nbr), km.n_out)
    assert_one_rounding(a, ref, A, "tf32 forward on a manager map", ACC_ANY)
    ga, gwa = backend._conv_backward(feats, gout, w, km)
    gb, gwb = backend._conv_backward(feats, gout, w, plain)
    assert torch.equal(ga, gb), "dgrad differs with the tile order"
    gw_ref, gw_A = ref_wgrad(feats, gout, _pairs(km.out_nbr))
    assert_one_rounding(gwa, gw_ref, gw_A, "tf32 wgrad on a manager map", ACC_ANY)


def test_optimizer_step_repacks(ME, cuda, tf32):
    """After an optimizer step under "tf32", the next forward uses the new weights: it equals
    a freshly constructed layer holding them, bit for bit."""
    conv, x = _layer_case(ME, cuda, 32, 64)
    opt = torch.optim.SGD(conv.parameters(), lr=0.5)
    _fwd_bwd(conv, x)
    opt.step()
    y = conv(x).F
    fresh = ME.MinkowskiConvolution(32, 64, kernel_size=3, dimension=3).to(cuda)
    fresh.load_state_dict(conv.state_dict())
    assert torch.equal(y, fresh(x).F)
    # and back to exact fp32 and to TF32 again: no stale operand copy on either side
    torch.backends.cuda.matmul.fp32_precision = "ieee"
    exact = conv(x).F
    with torch.no_grad():
        conv.kernel.mul_(-1.0)
    torch.backends.cuda.matmul.fp32_precision = "tf32"
    assert torch.equal(conv(x).F, -y)
    assert not torch.equal(exact, y)


# The fp32 reference runs of test_gpu_network.py (same keys, same seeds, loss = mean(out^2)).
# Tolerances are those of the bf16 network test, not looser: the TF32 path differs from the
# reference by at most 2^-9 per product and keeps fp32 activations, where bf16 rounds every stored
# value.  Measured on an H100 80GB HBM3 (700 W), MinkUNet14 / MinkUNet34C: logits rms 2.9e-3 /
# 4.1e-3, max 3.3e-3 / 3.8e-3, loss 6.6e-6 / 4.9e-5, gradient cosines final 1.000000, deep layer
# 0.992 / 0.981, first layer 0.993 / 0.981 (the badly conditioned backward through ~30 train-mode
# batch norms that test_gpu_network.py describes: already 4.5e-3 off in exact fp32).
_TOL = {"logits_rms": 6e-2, "logits_max": 1e-1, "loss": 2e-3}
_GRAD_COS = {"final.kernel": 0.9999, "block4.0.conv1.kernel": 0.6, "conv0p1s1.kernel": 0.6}


@pytest.mark.parametrize("name,n", [("MinkUNet14", 6000), ("MinkUNet34C", 4000)])
def test_minkunet_tf32_matches_reference(ME, cuda, tf32, name, n):
    G, key = golden("ref_network.npz"), f"fp32_{name}_{n}"
    torch.manual_seed(0)
    net = minkunet(name, ME, 3, 20, 3)
    assert (state_digest(net) == G[key + "/init_digest"]).all()
    net = net.to(cuda)
    coords = O.surface_cloud(n, seed=3)
    feats = torch.rand(n, 3, generator=torch.Generator().manual_seed(1))
    from minkowskiengine_b200 import _lib
    t0 = _lib.tc_launch_count()
    x = ME.SparseTensor(feats.to(cuda), coords.to(cuda))
    out = net(x)
    loss = out.F.float().pow(2).mean()
    loss.backward()
    assert _lib.tc_launch_count() > t0, "the fp32 network did not reach the tensor cores"
    loss_g, loss_r = loss.item(), float(G[key + "/loss"])
    a, b = out.F.detach().cpu().numpy()[G[key + "/rows"]], G[key + "/logits"]
    e_rms = np.sqrt(((a - b) ** 2).mean()) / float(G[key + "/logits_rms"])
    e_max = np.abs(a - b).max() / float(G[key + "/logits_absmax"])
    e_loss = abs(loss_g - loss_r) / abs(loss_r)
    print(f"\n[{name} tf32 vs reference fp32, {n} voxels] logits rms {e_rms:.2e} max {e_max:.2e} "
          f"loss {loss_g:.6f} vs {loss_r:.6f} ({e_loss:.2e})")
    fails = []
    if not (e_rms < _TOL["logits_rms"] and e_max < _TOL["logits_max"]):
        fails.append("logits")
    if not e_loss < _TOL["loss"]:
        fails.append("loss")
    pg = dict(net.named_parameters())
    for pname, cmin in _GRAD_COS.items():
        gg = pg[pname].grad.cpu().numpy().ravel()[G[f"{key}/{pname}/idx"]].astype(np.float64)
        gr = G[f"{key}/{pname}/grad"].astype(np.float64)
        cos = float(gg @ gr / (np.linalg.norm(gg) * np.linalg.norm(gr) + 1e-300))
        print(f"    grad {pname:24s} cos {cos:.6f}")
        if not cos > cmin:
            fails.append(pname)
    assert not fails, fails
