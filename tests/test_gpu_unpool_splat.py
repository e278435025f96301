"""MinkowskiPoolingTranspose and TensorField.splat on the GPU: against the compiled reference's
fixtures (fp32, 1e-5) and the float64 restatement (tests/unpool_splat_oracle.py) in bf16 / fp16
within one output rounding; adjointness between independent kernels; map reuse; bitwise repeats;
edge cases; the StackUNet and splat-FCNN training steps."""
import os

import numpy as np
import pytest
import torch

import minkowskiengine_b200 as ME
import unpool_splat_oracle as O
from helpers import assert_one_rounding

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
LOWP = [torch.bfloat16, torch.float16]

STACK_PARAMS = ("0.0.kernel", "0.1.0.kernel", "0.1.1.1.0.kernel", "0.1.1.1.1.kernel", "2.weight",
                "2.bias")
FCNN_PARAMS = ("mlp1.0.linear.weight", "conv2.0.kernel", "conv5.0.0.kernel", "conv5.2.0.kernel",
               "final.3.linear.weight", "final.3.linear.bias")


def stack_unet_net(MEh):
    """examples/stack_unet.py, 3 -> 5 channels, D = 2, seeded (shared with the fixture script)."""
    from examples.stack_unet import stack_unet
    torch.manual_seed(0)
    return stack_unet(MEh, 3, 5, D=2)


def stack_unet_step(MEh, net, dev):
    """One fp32 training step on 2 clouds of unique 2-D voxels -> (logits [N, 5] in input row
    order, loss)."""
    g = torch.Generator().manual_seed(13)
    c = torch.cat([torch.randint(0, 2, (3000, 1), generator=g),
                   torch.randint(0, 48, (3000, 2), generator=g)], 1).int()
    c = torch.unique(c, dim=0)
    c = c[torch.randperm(len(c), generator=g)]
    feats = torch.rand(len(c), 3, generator=g)
    labels = torch.randint(0, 5, (len(c),), generator=g)
    net = net.to(dev).train()
    logits = net(MEh.SparseTensor(feats, c, device=dev))
    loss = torch.nn.functional.cross_entropy(logits, labels.to(dev))
    loss.backward()
    return logits, float(loss)


def splat_fcnn_net(MEh):
    """MinkowskiSplatFCNN with small channels and no dropout, seeded (shared with the fixture
    script)."""
    from examples.fcnn import fcnn
    torch.manual_seed(0)
    return fcnn(MEh, 3, 10, embedding_channel=64, channels=(16, 16, 16, 32, 32), hidden=32,
                dropout=0.0, splat=True)


def splat_fcnn_step(MEh, net, dev):
    """One fp32 training step on 4 clouds of float points -> (logits SparseTensor, loss)."""
    g = torch.Generator().manual_seed(11)
    B, n = 4, 3000
    pts = torch.cat([torch.arange(B).repeat_interleave(n)[:, None].float(),
                     torch.rand(B * n, 3, generator=g) * 48], 1)
    feats = torch.rand(B * n, 3, generator=g)
    labels = torch.randint(0, 10, (B,), generator=g)
    net = net.to(dev).train()
    out = net(MEh.TensorField(feats.to(dev), pts.to(dev)))
    loss = torch.nn.functional.cross_entropy(out.F, labels.to(dev)[out.C[:, 0].long()])
    loss.backward()
    return out, float(loss)


def _load(name):
    return np.load(os.path.join(GOLDEN, name))


def _t(a, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a)).to(DEV, dtype)


def _np(t):
    return t.detach().double().cpu().numpy()


UNPOOL = {"k2s2_d3": (3, "max", 2, 2, False), "k3s2_d2": (2, "sum", 3, 2, False),
          "k2s2_expand": (3, "max", 2, 2, True), "k2s2_d4": (4, "max", 2, 2, False)}


def _coarse(name, z):
    """The stride-1 SparseTensor of the case and its pooled (stride-2) tensor."""
    D, pool, k, s, _ = UNPOOL[name]
    x = ME.SparseTensor(torch.ones(len(z["coords"]), 1, device=DEV), _t(z["coords"], torch.int32))
    P = ME.MinkowskiMaxPooling if pool == "max" else ME.MinkowskiSumPooling
    return x, P(kernel_size=k, stride=s, dimension=D)(x)


def _unpool(name, z, f_canon, dtype=torch.float32, coordinates=None):
    """(leaf on the coarse map, output, canonical perms of both) of one unpooling."""
    D, _, k, s, expand = UNPOOL[name]
    x, y = _coarse(name, z)
    pin = O.canon(y.C.cpu().numpy())
    f = np.empty_like(f_canon)
    f[pin] = f_canon
    leaf = _t(f, dtype).requires_grad_()
    ys = ME.SparseTensor(leaf, coordinate_map_key=y.coordinate_map_key,
                         coordinate_manager=y.coordinate_manager)
    out = ME.MinkowskiPoolingTranspose(kernel_size=k, stride=s, expand_coordinates=expand,
                                       dimension=D)(ys, coordinates)
    return x, ys, leaf, out, pin, O.canon(out.C.cpu().numpy())


@pytest.mark.parametrize("name", list(UNPOOL))
def test_unpool_matches_reference(name):
    z = _load(f"ref_unpool_{name}.npz")
    x, ys, leaf, out, pin, po = _unpool(name, z, z["in_feats"])
    assert (ys.C.cpu().numpy()[pin] == z["in_coords"]).all()
    assert (out.C.cpu().numpy()[po] == z["out_coords"]).all()
    assert out.tensor_stride == [1] * (z["coords"].shape[1] - 1)
    if not UNPOOL[name][4]:
        assert out.coordinate_map_key == x.coordinate_map_key   # the existing finer map
    np.testing.assert_allclose(_np(out.F)[po], z["out"], rtol=1e-5, atol=1e-5)
    g = np.empty_like(z["grad_out"])
    g[po] = z["grad_out"]
    out.F.backward(_t(g))
    np.testing.assert_allclose(_np(leaf.grad)[pin], z["grad_in"], rtol=1e-5, atol=1e-5)
    # repeats are bitwise identical
    g1 = leaf.grad.clone()
    leaf.grad = None
    out2 = ME.MinkowskiPoolingTranspose(*UNPOOL[name][2:4], expand_coordinates=UNPOOL[name][4],
                                        dimension=UNPOOL[name][0])(ys)
    # (an expanding unpooling makes a new map each time: the same coordinates, maybe new rows)
    out2.F.backward(_t(_reorder(g, out, out2)))
    assert torch.equal(g1, leaf.grad)


def _reorder(g, a, b):
    """Gradient rows of map a put in the row order of map b (same coordinate set)."""
    pa, pb = O.canon(a.C.cpu().numpy()), O.canon(b.C.cpu().numpy())
    out = np.empty_like(g)
    out[pb] = g[pa]
    return out


@pytest.mark.parametrize("dtype", LOWP)
@pytest.mark.parametrize("name", ["k2s2_d3", "k3s2_d2"])
def test_unpool_low_precision_one_rounding(name, dtype):
    z = _load(f"ref_unpool_{name}.npz")
    x, ys, leaf, out, pin, po = _unpool(name, z, z["in_feats"], dtype)
    D, _, k, s, _ = UNPOOL[name]
    cin, cout = ys.C.cpu().numpy(), out.C.cpu().numpy()
    pairs = O.unpool_pairs(cin, 2, cout, k, s)
    fx = _np(leaf)                                  # the same rounded inputs
    ref = O.unpool_forward(fx, pairs, len(cout))
    A = O.unpool_forward(np.abs(fx), pairs, len(cout))
    assert_one_rounding(out.F, _t(ref, torch.float64), _t(A, torch.float64), f"unpool {dtype}")
    g = _t(np.random.default_rng(1).standard_normal(out.F.shape), dtype)
    out.F.backward(g)
    gref = O.unpool_backward(_np(g), pairs, len(cin))
    Ag = O.unpool_backward(np.abs(_np(g)), pairs, len(cin))
    assert_one_rounding(leaf.grad, _t(gref, torch.float64), _t(Ag, torch.float64),
                        f"unpool backward {dtype}")


@pytest.mark.parametrize("name", ["k2s2_d3", "k3s2_d2"])
def test_unpool_is_the_adjoint_of_sum_pooling(name):
    """<sum_pool(a), b> = <a, unpool(b)> on the same pair of maps: ties k_pool_fwd over the pooling
    map to k_pool_fwd over the transposed map, and both backwards (k_pool_bwd_gather)."""
    D, _, k, s, _ = UNPOOL[name]
    z = _load(f"ref_unpool_{name}.npz")
    x, y = _coarse(name, z)
    g = torch.Generator().manual_seed(3)
    a = torch.randn(len(x), 6, generator=g).to(DEV).requires_grad_()
    b = torch.randn(len(y), 6, generator=g).to(DEV).requires_grad_()
    xa = ME.SparseTensor(a, coordinate_map_key=x.coordinate_map_key,
                         coordinate_manager=x.coordinate_manager)
    yb = ME.SparseTensor(b, coordinate_map_key=y.coordinate_map_key,
                         coordinate_manager=y.coordinate_manager)
    pa = ME.MinkowskiSumPooling(kernel_size=k, stride=s, dimension=D)(xa)
    ub = ME.MinkowskiPoolingTranspose(kernel_size=k, stride=s, dimension=D)(yb, x.coordinate_map_key)
    assert pa.coordinate_map_key == y.coordinate_map_key and ub.coordinate_map_key == \
        x.coordinate_map_key
    lhs = float((pa.F.double() * b.double()).sum())
    rhs = float((a.double() * ub.F.double()).sum())
    assert abs(lhs - rhs) <= 1e-5 * (abs(lhs) + 1), (lhs, rhs)
    # the backwards: d<pool(a), b>/da = unpool(b) and d<a, unpool(b)>/db = pool(a)
    (pa.F * b.detach()).sum().backward()
    (a.detach() * ub.F).sum().backward()
    torch.testing.assert_close(a.grad, ub.F.detach(), rtol=1e-6, atol=1e-6)
    torch.testing.assert_close(b.grad, pa.F.detach(), rtol=1e-6, atol=1e-6)


def test_unpool_after_pool_reuses_the_stride_map():
    """A k2s2 unpooling after a k2s2 pooling of the same maps builds no kernel map: no forward map
    is added to the manager's cache, and the unpooling's tables are the pooling's, swapped.  (The
    transposed entry itself may already be there: the map prefetch of a new manager replays the
    requests of the previous one.)"""
    z = _load("ref_unpool_k2s2_d3.npz")
    x, y = _coarse("k2s2_d3", z)
    mgr = x.coordinate_manager._manager
    before = dict(mgr._kernel_maps)
    fwd = {k for k in before if not k[6]}
    out = ME.MinkowskiPoolingTranspose(kernel_size=2, stride=2, dimension=3)(y)
    assert out.coordinate_map_key == x.coordinate_map_key
    assert {k for k in mgr._kernel_maps if not k[6]} == fwd
    ik, ok = mgr._k(y.coordinate_map_key), mgr._k(x.coordinate_map_key)
    t_keys = [k for k in mgr._kernel_maps if k[:2] == (ik, ok) and k[6] and k[7]]
    assert len(t_keys) == 1 and t_keys[0][2:5] == ((2, 2, 2), (2, 2, 2), (1, 1, 1))
    t_key = t_keys[0]
    assert set(mgr._kernel_maps) - set(before) <= {t_key}
    pool_km = mgr._kernel_maps[(ok, ik) + t_key[2:6] + (False, True)]
    km = mgr._kernel_maps[t_key]
    assert km.out_nbr.data_ptr() == pool_km.in_nbr.data_ptr()
    assert km.in_nbr.data_ptr() == pool_km.out_nbr.data_ptr()


def test_unpool_coordinates_argument():
    z = _load("ref_unpool_k3s2_d2.npz")
    x, y = _coarse("k3s2_d2", z)
    layer = ME.MinkowskiPoolingTranspose(kernel_size=3, stride=2, dimension=2)
    ref = layer(y)
    by_key = layer(y, x.coordinate_map_key)
    by_tensor = layer(y, x)
    assert ref.coordinate_map_key == by_key.coordinate_map_key == by_tensor.coordinate_map_key
    assert torch.equal(ref.F, by_key.F) and torch.equal(ref.F, by_tensor.F)
    # a coordinate tensor: a new map of exactly those coordinates
    c = x.C[torch.randperm(len(x), generator=torch.Generator().manual_seed(0)).to(DEV)]
    by_coords = layer(y, c)
    assert (by_coords.C.cpu().numpy()[O.canon(by_coords.C.cpu().numpy())] ==
            x.C.cpu().numpy()[O.canon(x.C.cpu().numpy())]).all()
    assert torch.equal(by_coords.F[O.canon(by_coords.C.cpu().numpy())],
                       ref.F[O.canon(ref.C.cpu().numpy())])


# ---- splatting ------------------------------------------------------------------------------------
def _splat(pts, feats, dtype=torch.float32):
    x = _t(feats, dtype).requires_grad_()
    tf = ME.TensorField(x, _t(pts))
    st = tf.splat()
    return x, tf, st, O.canon(st.C.cpu().numpy())


@pytest.mark.parametrize("case", ["small_", "small2_", "cloud"])
def test_splat_matches_reference(case):
    z = _load("ref_splat_cloud.npz" if case == "cloud" else "ref_splat_small.npz")
    tag = "" if case == "cloud" else case
    x, tf, st, perm = _splat(z[f"{tag}coords"], z[f"{tag}feats"])
    c = st.C.cpu().numpy()
    assert (c[perm] == z[f"{tag}out_coords"]).all()
    assert st.tensor_stride == [1] * (c.shape[1] - 1)
    # rows by first occurrence of the point-major corners, as the reference's CPU insert numbers
    assert (c == O.splat_map(z[f"{tag}coords"])[0]).all()
    np.testing.assert_allclose(_np(st.F)[perm], z[f"{tag}out"], rtol=1e-5, atol=1e-5)
    g = np.empty_like(z[f"{tag}grad_out"])
    g[perm] = z[f"{tag}grad_out"]
    st.F.backward(_t(g))
    np.testing.assert_allclose(_np(x.grad), z[f"{tag}grad_in"], rtol=1e-5, atol=1e-5)
    assert st.coordinate_map_key in tf._splat


def test_interpolate_on_the_splat_map_matches_reference():
    """interpolate on X's splat map is the reference's transposed SPMM: features_at_coordinates
    computes the same corners and weights as the splat record."""
    z = _load("ref_splat_cloud.npz")
    x, tf, st, perm = _splat(z["coords"], z["feats"])
    rows, w, _ = tf._splat[st.coordinate_map_key]
    r2, w2 = st.coordinate_manager._manager._interp_map(st.coordinate_map_key, tf.C)
    assert torch.equal(rows, r2) and torch.equal(w, w2)
    f = np.empty_like(z["interp_feats"])
    f[perm] = z["interp_feats"]
    leaf = _t(f).requires_grad_()
    ys = ME.SparseTensor(leaf, coordinate_map_key=st.coordinate_map_key,
                         coordinate_manager=st.coordinate_manager)
    y = ys.interpolate(tf)
    assert y.coordinate_field_map_key == tf.coordinate_field_map_key
    np.testing.assert_allclose(_np(y.F), z["interp_out"], rtol=1e-5, atol=1e-5)
    y.F.backward(_t(z["interp_grad_out"]))
    np.testing.assert_allclose(_np(leaf.grad)[perm], z["interp_grad_feats"], rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("dtype", LOWP)
def test_splat_low_precision_one_rounding(dtype):
    z = _load("ref_splat_cloud.npz")
    feats = np.random.default_rng(4).standard_normal((len(z["coords"]), 40)).astype(np.float32)
    x, tf, st, perm = _splat(z["coords"], feats, dtype)
    coords, rows, w64 = O.splat_map(z["coords"])
    assert (st.C.cpu().numpy() == coords).all()
    r32, w32, _ = tf._splat[st.coordinate_map_key]
    assert (r32.cpu().numpy() == rows).all()
    np.testing.assert_allclose(_np(w32), w64, rtol=0, atol=1e-6)
    # the same rounded inputs: the features in `dtype` and the kernel's fp32 weights
    w = _np(w32)
    fx = _np(x)
    ref = O.splat_forward(fx, rows, w, len(coords))
    A = O.splat_forward(np.abs(fx), rows, w, len(coords))
    assert_one_rounding(st.F, _t(ref, torch.float64), _t(A, torch.float64), f"splat {dtype}")
    g = _t(np.random.default_rng(5).standard_normal(st.F.shape), dtype)
    st.F.backward(g)
    gref = O.splat_backward(_np(g), rows, w)
    Ag = O.splat_backward(np.abs(_np(g)), rows, w)
    assert_one_rounding(x.grad, _t(gref, torch.float64), _t(Ag, torch.float64),
                        f"splat backward {dtype}")


def test_splat_is_the_adjoint_of_interpolation():
    """<splat(F), G> = <F, G.interpolate(X)> on the splat map, accumulated in float64: ties the
    weighted k_field_reduce to k_interp_fwd."""
    z = _load("ref_splat_cloud.npz")
    g = torch.Generator().manual_seed(8)
    Fp = torch.randn(len(z["coords"]), 16, generator=g).to(DEV)
    tf = ME.TensorField(Fp, _t(z["coords"]))
    st = tf.splat()
    G = torch.randn(len(st), 16, generator=g).to(DEV)
    Gs = ME.SparseTensor(G, coordinate_map_key=st.coordinate_map_key,
                         coordinate_manager=st.coordinate_manager)
    lhs = float((st.F.double() * G.double()).sum())
    rhs = float((Fp.double() * Gs.interpolate(tf).F.double()).sum())
    assert abs(lhs - rhs) <= 1e-5 * (abs(lhs) + 1), (lhs, rhs)


def test_splat_determinism_and_cache():
    """200k points, C = 32 bf16: two runs of splat forward and backward and of unpooling backward
    are bitwise identical; the splat record is reused by the backward."""
    g = torch.Generator().manual_seed(1)
    n = 200_000
    pts = torch.cat([torch.randint(0, 4, (n, 1), generator=g).float(),
                     torch.rand(n, 3, generator=g) * 40 - 20], 1).to(DEV)
    x = torch.randn(n, 32, generator=g).to(DEV, torch.bfloat16).requires_grad_()

    def run():
        x.grad = None
        tf = ME.TensorField(x, pts)
        st = tf.splat()
        y = ME.MinkowskiPoolingTranspose(2, 2, dimension=3)(
            ME.MinkowskiSumPooling(2, 2, dimension=3)(st))
        gy = torch.randn(y.F.shape, generator=torch.Generator().manual_seed(2)).to(DEV, y.F.dtype)
        y.F.backward(gy)
        return st.F.detach().clone(), x.grad.clone()

    (f1, g1), (f2, g2) = run(), run()
    assert torch.equal(f1, f2) and torch.equal(g1, g2)


def test_splat_edge_cases():
    # a point on integer coordinates: its upper corners weigh 0 and are zero rows
    pts = torch.tensor([[0, 1.0, 2.0, -3.0]], device=DEV)
    tf = ME.TensorField(torch.tensor([[2.5]], device=DEV), pts)
    st = tf.splat()
    assert len(st) == 8
    assert st.F[0].item() == 2.5 and (st.F[1:] == 0).all()
    assert (st.C[0] == torch.tensor([0, 1, 2, -3], device=DEV, dtype=torch.int32)).all()
    assert (st.C[1] == torch.tensor([0, 1, 2, -2], device=DEV, dtype=torch.int32)).all()
    # non-finite coordinates, a corner outside int32, a non-integer batch index
    for bad in ([0, float("nan"), 0, 0], [0, 0, float("inf"), 0], [0, 0, 0, 2.0 ** 31],
                [0, -2.0 ** 31 - 256, 0, 0], [0.5, 0, 0, 0]):
        tf = ME.TensorField(torch.ones(2, 3, device=DEV),
                            torch.tensor([[0, 0.5, 0.5, 0.5], bad], device=DEV))
        with pytest.raises(ValueError):
            tf.splat()
    # the lowest float coordinate inside int32 is fine
    ME.TensorField(torch.ones(1, 1, device=DEV),
                   torch.tensor([[1, -2.0 ** 31, 0, 0]], device=DEV)).splat()
    # SPLAT_LINEAR_INTERPOLATION stays rejected as a quantisation mode, and points to splat()
    with pytest.raises(NotImplementedError, match="splat"):
        ME.TensorField(torch.ones(1, 1, device=DEV), pts,
                       quantization_mode=ME.SparseTensorQuantizationMode.SPLAT_LINEAR_INTERPOLATION)
    with pytest.raises(NotImplementedError, match="SPLAT"):
        ME.TensorField(torch.ones(1, 1, device=DEV), pts).sparse(
            quantization_mode=ME.SparseTensorQuantizationMode.SPLAT_LINEAR_INTERPOLATION)


def test_stack_containers_and_reductions():
    c = torch.tensor([[0, 0, 0], [0, 1, 0], [0, 2, 1]], dtype=torch.int32)
    a = ME.SparseTensor(torch.randn(3, 4), c, device=DEV)
    b = ME.SparseTensor(torch.randn(3, 4, device=DEV), coordinate_map_key=a.coordinate_map_key,
                        coordinate_manager=a.coordinate_manager)
    xs = torch.stack([a.F, b.F])
    assert torch.equal(ME.sum(a, b).F, a.F + b.F)
    assert torch.equal(ME.sum([a, b, a]).F, a.F + b.F + a.F)
    torch.testing.assert_close(ME.mean(a, b).F, xs.mean(0))
    torch.testing.assert_close(ME.var(a, b).F, xs.var(0, unbiased=False))
    ident = torch.nn.Identity()
    neg = ME.MinkowskiLinear(4, 4, bias=False).to(DEV)
    assert torch.equal(ME.MinkowskiStackCat(ident, ident)(a).F, torch.cat([a.F, a.F], 1))
    assert torch.equal(ME.MinkowskiStackSum(ident, ident)(a).F, a.F + a.F)
    torch.testing.assert_close(ME.MinkowskiStackMean(ident, neg)(a).F, (a.F + neg(a).F) / 2)
    torch.testing.assert_close(ME.MinkowskiStackVar(ident, neg)(a).F,
                               torch.stack([a.F, neg(a).F]).var(0, unbiased=False))
    assert ME.MinkowskiToFeature()(a) is a.F
    tf = ME.TensorField(torch.randn(3, 2, device=DEV), c.float().to(DEV))
    s = ME.sum(tf, tf)
    assert isinstance(s, ME.TensorField) and torch.equal(s.F, tf.F * 2)
    other = ME.SparseTensor(torch.randn(3, 4), c, device=DEV)
    with pytest.raises(AssertionError):
        ME.sum(a, other)


def test_stack_unet_matches_reference():
    from helpers import state_digest
    G = _load("ref_unpool_stack_unet.npz")
    net = stack_unet_net(ME)
    assert (state_digest(net) == G["init_digest"]).all(), \
        "seeded initial weights differ from the reference's"
    logits, loss = stack_unet_step(ME, net, DEV)
    F, R = logits.detach().cpu().numpy(), G["logits"]
    assert F.shape == R.shape
    assert np.abs(F - R).max() / np.abs(R).max() < 1e-3
    assert abs(loss - float(G["loss"])) / abs(float(G["loss"])) < 1e-3
    params = dict(net.named_parameters())
    for p in STACK_PARAMS:
        gg = params[p].grad.cpu().numpy().ravel()[G[f"{p}/idx"]].astype(np.float64)
        gr = G[f"{p}/grad"].astype(np.float64)
        err = np.abs(gg - gr).max() / float(G[f"{p}/absmax"])
        assert err < 2e-3, (p, err)


def test_splat_fcnn_matches_reference():
    """examples/fcnn.py with splat=True, one fp32 training step, against the compiled reference's
    run, with the tolerances of the FCNN step in tests/test_gpu_field.py."""
    from helpers import state_digest
    G = _load("ref_splat_fcnn.npz")
    net = splat_fcnn_net(ME)
    assert (state_digest(net) == G["init_digest"]).all(), \
        "seeded initial weights differ from the reference's"
    out, loss = splat_fcnn_step(ME, net, DEV)
    assert (out.C.cpu().numpy() == G["out_coords"]).all()
    F, R = out.F.detach().cpu().numpy(), G["logits"]
    assert np.abs(F - R).max() / np.abs(R).max() < 1e-3
    assert abs(loss - float(G["loss"])) / abs(float(G["loss"])) < 1e-3
    params = dict(net.named_parameters())
    for p in FCNN_PARAMS:
        gg = params[p].grad.cpu().numpy().ravel()[G[f"{p}/idx"]].astype(np.float64)
        gr = G[f"{p}/grad"].astype(np.float64)
        err = np.abs(gg - gr).max() / float(G[f"{p}/absmax"])
        if p.startswith("final.3"):
            assert err < 2e-3, (p, err)
        else:
            cos = float(gg @ gr / (np.linalg.norm(gg) * np.linalg.norm(gr)))
            assert cos > 0.999 and err < 5e-2, (p, cos, err)
