"""TensorField on the GPU: quantisation in the four modes, slice / cat_slice, interpolation, their
backwards, against the compiled reference's fixtures (fp32, 1e-5) and the float64 restatement
(tests/field_oracle.py) in bf16 / fp16 within one output rounding; bitwise repeats; edge cases."""
import os

import numpy as np
import pytest
import torch

import field_oracle as O
import minkowskiengine_b200 as ME
from helpers import assert_one_rounding

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
Q = ME.SparseTensorQuantizationMode
MODES = {O.SUM: Q.UNWEIGHTED_SUM, O.AVG: Q.UNWEIGHTED_AVERAGE, O.SUBSAMPLE: Q.RANDOM_SUBSAMPLE,
         O.MAX: Q.MAX_POOL}
LOWP = [torch.bfloat16, torch.float16]


def _load(name):
    return np.load(os.path.join(GOLDEN, name))


def _t(a, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a)).to(DEV, dtype)


def _np(t):
    return t.detach().double().cpu().numpy()


FCNN_PARAMS = ("mlp1.0.linear.weight", "conv2.0.kernel", "conv5.0.0.kernel", "conv5.2.0.kernel",
               "final.3.linear.weight", "final.3.linear.bias")


def fcnn_net(MEh):
    """MinkowskiFCNN with small channels and no dropout, seeded (shared with the fixture script)."""
    from examples.fcnn import fcnn
    torch.manual_seed(0)
    return fcnn(MEh, 3, 10, embedding_channel=64, channels=(16, 16, 16, 32, 32), hidden=32,
                dropout=0.0)


def fcnn_step(MEh, net, dev):
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


def _quantise(pts, feats, mode, stride, dtype=torch.float32, grad_seed=3):
    """(coords, out, grad_in) of one .sparse() + backward with a seeded gradient."""
    x = _t(feats, dtype).requires_grad_()
    tf = ME.TensorField(x, _t(pts), quantization_mode=MODES[mode])
    st = tf.sparse(tensor_stride=stride)
    g = torch.randn(st.F.shape, generator=torch.Generator().manual_seed(grad_seed)).to(DEV, dtype)
    st.F.backward(g)
    return st, x.grad, g


@pytest.mark.parametrize("stride", [1, 2])
@pytest.mark.parametrize("mode", list(MODES))
def test_quantisation_matches_reference(mode, stride):
    z = _load("ref_field_quantize.npz")
    tag = f"{mode}_s{stride}"
    x = _t(z["feats"]).requires_grad_()
    st = ME.TensorField(x, _t(z["coords"]), quantization_mode=MODES[mode]).sparse(
        tensor_stride=stride)
    c = st.C.cpu().numpy()
    perm = O.canon(c)
    assert (c[perm] == z[f"{tag}_out_coords"]).all()
    np.testing.assert_allclose(_np(st.F)[perm], z[f"{tag}_out"], rtol=1e-5, atol=1e-5)
    g = np.empty_like(z[f"{tag}_grad_out"])
    g[perm] = z[f"{tag}_grad_out"]
    st.F.backward(_t(g))
    np.testing.assert_allclose(_np(x.grad), z[f"{tag}_grad_in"], rtol=1e-5, atol=1e-5)
    x2 = _t(z["feats"]).requires_grad_()
    st2 = ME.TensorField(x2, _t(z["coords"]), quantization_mode=MODES[mode]).sparse(
        tensor_stride=stride)
    st2.F.backward(_t(g))
    assert torch.equal(st.F, st2.F) and torch.equal(x.grad, x2.grad)


@pytest.mark.parametrize("dtype", LOWP)
@pytest.mark.parametrize("mode", list(MODES))
def test_quantisation_low_precision_one_rounding(mode, dtype):
    z = _load("ref_field_quantize.npz")
    feats = z["feats"] * np.where(np.arange(z["feats"].size).reshape(z["feats"].shape) % 3, 1, -1)
    st, grad, g = _quantise(z["coords"], feats, mode, 2, dtype)
    fx = _np(_t(feats, dtype))
    _, _, inv = O.insert(O.quantize(z["coords"], 2))
    uniq = O.insert(O.quantize(z["coords"], 2))[0]
    assert (st.C.cpu().numpy() == uniq).all()     # rows in first-point order
    M = len(uniq)
    ref, _ = O.reduce(fx, inv, M, mode)
    A, _ = O.reduce(np.abs(fx), inv, M, mode)     # the same reduction over |x|
    assert_one_rounding(st.F, torch.from_numpy(ref).to(DEV), torch.from_numpy(A).to(DEV),
                        f"{mode} {dtype}")
    gref = O.reduce_backward(_np(g), fx, inv, M, mode)
    assert_one_rounding(grad, torch.from_numpy(gref).to(DEV), torch.from_numpy(np.abs(gref)).to(DEV),
                        f"{mode} {dtype} backward")
    st2, grad2, _ = _quantise(z["coords"], feats, mode, 2, dtype)
    assert torch.equal(st.F, st2.F) and torch.equal(grad, grad2)


@pytest.mark.parametrize("dtype", [torch.float32] + LOWP)
@pytest.mark.parametrize("stride", [1, 2, 4])
def test_slice_and_cat_slice(stride, dtype):
    z = _load("ref_field_slice.npz")
    tf = ME.TensorField(_t(z["feats"], dtype), _t(z["coords"]))
    st = tf.sparse()
    pool = ME.MinkowskiMaxPooling(kernel_size=2, stride=2, dimension=3)
    y = st
    while y.tensor_stride[0] < stride:
        y = pool(y)
    c = y.C.cpu().numpy()
    perm = O.canon(c)
    assert (c[perm] == z[f"s{stride}_coords"]).all()
    f = np.empty_like(z[f"s{stride}_feats"])
    f[perm] = z[f"s{stride}_feats"]
    leaf = _t(f, dtype).requires_grad_()
    ys = ME.SparseTensor(leaf, coordinate_map_key=y.coordinate_map_key,
                         coordinate_manager=y.coordinate_manager)
    out = ys.slice(tf)
    assert isinstance(out, ME.TensorField) and out.coordinate_field_map_key == \
        tf.coordinate_field_map_key
    inv = O.find(c, O.quantize(z["coords"], stride))
    assert (tf.inverse_mapping(y.coordinate_map_key).cpu().numpy() == inv).all()
    ref = O.slice_forward(_np(leaf), inv)
    assert (_np(out.F) == ref).all()
    if stride == 1 and dtype == torch.float32:
        np.testing.assert_allclose(_np(out.F), z["s1_out"], rtol=0, atol=0)
    g = _t(z[f"s{stride}_grad_out"], dtype)
    out.F.backward(g)
    gref = O.slice_backward(_np(g), inv, len(c))
    if dtype == torch.float32:
        np.testing.assert_allclose(_np(leaf.grad), gref, rtol=1e-5, atol=1e-5)
        if stride == 1:
            np.testing.assert_allclose(_np(leaf.grad)[perm], z["s1_grad_feats"], rtol=1e-5,
                                       atol=1e-5)
    else:
        A = O.slice_backward(np.abs(_np(g)), inv, len(c))
        assert_one_rounding(leaf.grad, torch.from_numpy(gref).to(DEV), torch.from_numpy(A).to(DEV),
                            f"slice backward {dtype}")
    g1 = leaf.grad.clone()
    leaf.grad = None
    ys.slice(tf).F.backward(g)
    assert torch.equal(g1, leaf.grad)
    cs = ys.cat_slice(tf)
    assert torch.equal(cs.F, torch.cat([out.F, tf.F], 1))


@pytest.mark.parametrize("D", [3, 4])
def test_interpolation_matches_reference(D):
    z = _load("ref_field_interp.npz")
    x = _t(z[f"d{D}_feats"]).requires_grad_()
    st = ME.SparseTensor(x, _t(z[f"d{D}_coords"], torch.int32), tensor_stride=2)
    ys = []
    for qdt in (torch.float32, torch.float64, torch.float32):
        y = st.features_at_coordinates(_t(z[f"d{D}_query"], qdt))
        np.testing.assert_allclose(_np(y), z[f"d{D}_out"], rtol=1e-5, atol=1e-5)
        ys.append(y.detach())
    assert torch.equal(ys[0], ys[2])
    x.grad = None
    y.backward(_t(z[f"d{D}_grad_out"]))
    np.testing.assert_allclose(_np(x.grad), z[f"d{D}_grad_feats"], rtol=1e-5, atol=1e-5)
    g1 = x.grad.clone()
    x.grad = None
    st.features_at_coordinates(_t(z[f"d{D}_query"])).backward(_t(z[f"d{D}_grad_out"]))
    assert torch.equal(g1, x.grad)
    out, (in_rows, out_rows), w = ME.MinkowskiInterpolation(True, True)(st, _t(z[f"d{D}_query"]))
    rows, wr = O.interp_map(z[f"d{D}_query"], z[f"d{D}_coords"], 2)
    hit = rows >= 0
    assert (in_rows.cpu().numpy() == rows[hit]).all()
    assert (out_rows.cpu().numpy() == np.nonzero(hit)[0]).all()
    assert (w.cpu().numpy() == wr[hit]).all()


@pytest.mark.parametrize("dtype", LOWP)
def test_interpolation_low_precision_one_rounding(dtype):
    z = _load("ref_field_interp.npz")
    x = _t(z["d3_feats"], dtype).requires_grad_()
    st = ME.SparseTensor(x, _t(z["d3_coords"], torch.int32), tensor_stride=2)
    tf = ME.TensorField(torch.zeros(len(z["d3_query"]), 1, device=DEV), _t(z["d3_query"]),
                        coordinate_manager=st.coordinate_manager)
    y = st.interpolate(tf).F
    rows, w = O.interp_map(z["d3_query"], z["d3_coords"], 2)
    fx = _np(x)
    ref = O.interp_forward(fx, rows, w)
    A = O.interp_forward(np.abs(fx), rows, w)
    assert_one_rounding(y, torch.from_numpy(ref).to(DEV), torch.from_numpy(A).to(DEV), "interp")
    g = _t(z["d3_grad_out"], dtype)
    y.backward(g)
    gref = O.interp_backward(_np(g), rows, w, len(fx))
    A = O.interp_backward(np.abs(_np(g)), rows, w, len(fx))
    assert_one_rounding(x.grad, torch.from_numpy(gref).to(DEV), torch.from_numpy(A).to(DEV),
                        "interp backward")


@pytest.mark.parametrize("C", [3, 7, 8, 32])
def test_edge_cases(C):
    g = torch.Generator().manual_seed(C)
    # batch indices 0 and 2 only, one voxel holding 5000 points, odd and vector widths
    big = torch.cat([torch.zeros(5000, 1), torch.rand(5000, 3, generator=g) * 0.99 + 3], 1)
    rest = torch.cat([torch.randint(0, 2, (3000, 1), generator=g).float() * 2,
                      torch.rand(3000, 3, generator=g) * 20 - 10], 1)
    pts = torch.cat([big, rest])[torch.randperm(8000, generator=g)]
    feats = torch.randn(8000, C, generator=g)
    for mode in MODES:
        st, grad, gout = _quantise(pts.numpy(), feats.numpy(), mode, 1)
        _, _, inv = O.insert(O.quantize(pts.numpy(), 1))
        M = len(st)
        ref, _ = O.reduce(feats.numpy(), inv, M, mode)
        # fp32 sums of up to 5000 points: 2^-20 of the same reduction over |x|, per element
        A, _ = O.reduce(np.abs(feats.numpy()), inv, M, mode)
        assert_one_rounding(st.F, torch.from_numpy(ref).to(DEV), torch.from_numpy(A).to(DEV),
                            f"{mode} C={C}")
        np.testing.assert_allclose(_np(grad), O.reduce_backward(_np(gout), feats.numpy(), inv, M,
                                                                mode), rtol=1e-5, atol=1e-5)
    # no duplicates: the field's own features; one point
    tf = ME.TensorField(feats[:1].to(DEV), pts[:1].to(DEV))
    assert tf.sparse().F is tf.F
    u = torch.cat([torch.zeros(50, 1), torch.arange(50).float()[:, None] * 3 + 0.5,
                   torch.zeros(50, 2)], 1)
    tf = ME.TensorField(torch.randn(50, C).to(DEV), u.to(DEV))
    assert tf.sparse().F is tf.F
    # NaN coordinates raise
    bad = pts.clone()
    bad[17, 2] = float("nan")
    with pytest.raises(ValueError):
        ME.TensorField(feats.to(DEV), bad.to(DEV)).sparse()


def test_cached_quantisation_and_manager_integration():
    z = _load("ref_field_quantize.npz")
    tf = ME.TensorField(_t(z["feats"]), _t(z["coords"]))
    a = tf.sparse()
    b = tf.sparse()
    assert a.coordinate_map_key == b.coordinate_map_key
    mgr = tf.coordinate_manager
    assert mgr.exists_field_to_sparse(tf.coordinate_field_map_key, a.coordinate_map_key)
    assert a.coordinate_map_key in mgr.field_to_sparse_keys(tf.coordinate_field_map_key)
    uidx, inv = mgr.get_field_to_sparse_map(tf.coordinate_field_map_key, a.coordinate_map_key)
    assert len(uidx) == len(a) and len(inv) == len(tf)
    # global pooling needs the map among the origin map's inserted maps
    pooled = ME.MinkowskiGlobalAvgPooling()(a)
    assert len(pooled) == 3
    # the point network layers keep the field
    lin = ME.MinkowskiLinear(5, 16).to(DEV)
    h = ME.MinkowskiReLU()(ME.MinkowskiBatchNorm(16).to(DEV)(lin(tf)))
    assert isinstance(h, ME.TensorField)
    h2 = ME.cat(h, h)
    assert isinstance(h2, ME.TensorField) and h2.F.shape[1] == 32
    s = ME.MinkowskiToSparseTensor()(h2)
    assert isinstance(s, ME.SparseTensor) and s.coordinate_map_key == a.coordinate_map_key
    # onto an existing map
    s2 = tf.sparse(coordinate_map_key=a.coordinate_map_key)
    np.testing.assert_allclose(_np(s2.F), _np(a.F), rtol=1e-6, atol=1e-6)


def test_profile_size_values_and_repeats():
    """8 clouds x 250k points (the size profiles/field_bench.py times), C = 32 bf16: sparse() AVG
    and slice, forward and backward, against the float64 restatement and bitwise repeated."""
    g = torch.Generator().manual_seed(0)
    B, per = 8, 250_000
    n = B * per
    pts = torch.cat([torch.arange(B).repeat_interleave(per)[:, None].float(),
                     torch.rand(n, 3, generator=g) * 60], 1)
    x = torch.randn(n, 32, generator=g).to(DEV, torch.bfloat16).requires_grad_()
    gp = torch.randn(n, 32, generator=g).to(DEV, torch.bfloat16)
    ptsd = pts.to(DEV)

    def run():
        x.grad = None
        tf = ME.TensorField(x, ptsd)
        st = tf.sparse()
        st.F.retain_grad()
        st.slice(tf).F.backward(gp)
        return st, x.grad.clone()

    (st, g1), (st2, g2) = run(), run()
    assert torch.equal(st.F, st2.F) and torch.equal(st.F.grad, st2.F.grad)
    assert torch.equal(g1, g2)
    uniq, _, inv = O.insert(O.quantize(pts.numpy(), 1))
    assert (st.C.cpu().numpy() == uniq).all()
    M = len(uniq)
    fx = _np(x)
    ref, _ = O.reduce(fx, inv, M, O.AVG)
    A, _ = O.reduce(np.abs(fx), inv, M, O.AVG)
    assert_one_rounding(st.F, torch.from_numpy(ref).to(DEV), torch.from_numpy(A).to(DEV), "avg")
    # slice backward: the gradients of each voxel's points summed
    gv, _ = O.reduce(_np(gp), inv, M, O.SUM)
    Av, _ = O.reduce(np.abs(_np(gp)), inv, M, O.SUM)
    assert_one_rounding(st.F.grad, torch.from_numpy(gv).to(DEV), torch.from_numpy(Av).to(DEV),
                        "slice backward")
    # the average's backward, fed the voxel gradient the slice backward produced
    gx = O.reduce_backward(_np(st.F.grad), fx, inv, M, O.AVG)
    assert_one_rounding(g1, torch.from_numpy(gx).to(DEV), torch.from_numpy(np.abs(gx)).to(DEV),
                        "avg backward")


def test_tensor_field_arithmetic_repr_and_batches():
    pts = torch.tensor([[0, 0.5, 0, 0], [2.5, 1.5, 0, 0], [-0.5, 3, 1, 2], [1.49, 0, 0, 0],
                        [0.5, 4, 4, 4]], device=DEV)
    f = torch.arange(10.0, device=DEV).reshape(5, 2)
    a = ME.TensorField(f, pts)
    b = ME.TensorField(f * 2, coordinate_field_map_key=a.coordinate_field_map_key,
                       coordinate_manager=a.coordinate_manager)
    for y, ref in ((a + b, f * 3), (a - b, -f), (a * b, f * f * 2), (a / (b + 1), f / (f * 2 + 1)),
                   (a + 1.5, f + 1.5), (a * torch.full_like(f, 3), f * 3), (-a, -f)):
        assert isinstance(y, ME.TensorField)
        assert y.coordinate_field_map_key == a.coordinate_field_map_key
        assert torch.equal(y.F, ref)
    c = ME.TensorField(f, pts, coordinate_manager=a.coordinate_manager)
    with pytest.raises(AssertionError):
        a + c                                     # another field key
    assert "TensorField(" in repr(a) and "coordinate_field_map_key" in repr(a)
    # batch indices round half away from zero, as the quantisation does: 2.5 -> 3, -0.5 -> -1
    assert [int(v) for v in a.sparse().C[:, 0].cpu()] == [0, 3, -1, 1, 1]
    rows = a.decomposition_permutations
    assert [r.tolist() for r in rows] == [[0], [3, 4], [], [1]]
    assert torch.equal(a.features_at(1), f[[3, 4]])
    assert torch.equal(a.coordinates_at(3), pts[[1], 1:])


def test_cat_slice_of_a_sparse_tensor_with_duplicates_and_missing_voxels():
    g = torch.Generator().manual_seed(2)
    coords = torch.randint(0, 4, (300, 4), generator=g, dtype=torch.int32)
    coords[:, 0] = 0
    feats = torch.randn(300, 3, generator=g)
    x = ME.SparseTensor(feats, coords, device=DEV,
                        quantization_mode=Q.UNWEIGHTED_AVERAGE)
    assert len(x) < 300
    y = ME.SparseTensor((x.F * 2).requires_grad_(), coordinate_map_key=x.coordinate_map_key,
                        coordinate_manager=x.coordinate_manager)
    out = y.cat_slice(x)
    inv = x.inverse_mapping
    assert out.F.shape == (300, 6)
    assert torch.equal(out.F, torch.cat([y.F[inv], x.F[inv]], 1))
    assert torch.equal(out.C, coords.to(DEV).float())
    # a field whose stride-1 relation lacks voxels: the composed map keeps -1 for those points
    pts = torch.cat([torch.zeros(6, 1), torch.tensor([[0.5, 0, 0], [1.5, 0, 0], [2.5, 0, 0],
                                                      [3.5, 0, 0], [8.5, 0, 0], [9.5, 0, 0]])], 1)
    big = ME.SparseTensor(torch.ones(4, 1), torch.tensor([[0, 0, 0, 0], [0, 1, 0, 0], [0, 2, 0, 0],
                                                          [0, 3, 0, 0]], dtype=torch.int32),
                          device=DEV)
    tf = ME.TensorField(torch.ones(6, 1, device=DEV), pts.to(DEV),
                        coordinate_manager=big.coordinate_manager)
    inv1, _ = big.coordinate_manager.field_to_sparse_map(tf.coordinate_field_map_key,
                                                         big.coordinate_map_key)
    assert inv1.tolist() == [0, 1, 2, 3, -1, -1]
    s2 = ME.MinkowskiMaxPooling(kernel_size=2, stride=2, dimension=3)(big)
    inv2 = tf.inverse_mapping(s2.coordinate_map_key)
    assert inv2.tolist()[4:] == [-1, -1] and (inv2[:4] >= 0).all()
    assert (s2.slice(tf).F[4:] == 0).all()


def test_fcnn_matches_reference():
    """examples/fcnn.py, one fp32 training step, against the compiled reference's run
    (ref_field_fcnn.npz; its strided slices are put in input-row order, see the fixture script)."""
    from helpers import state_digest
    G = _load("ref_field_fcnn.npz")
    net = fcnn_net(ME)
    assert (state_digest(net) == G["init_digest"]).all(), \
        "seeded initial weights differ from the reference's"
    out, loss = fcnn_step(ME, net, DEV)
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
            # below the head, fp32 round-off is amplified by the train-mode batch norms (as in the
            # ResNet14 and MinkUNet runs): the gradients must point the same way
            cos = float(gg @ gr / (np.linalg.norm(gg) * np.linalg.norm(gr)))
            assert cos > 0.999 and err < 5e-2, (p, cos, err)
