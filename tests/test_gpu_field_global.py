"""Global pooling and broadcast over the points of a TensorField (csrc/global.cu:
meb200_field_origin_group, meb200_field_origin_insert), against the compiled reference's fixtures
(tests/golden/ref_field_global_*, ref_field_pointnet, written by
tests/golden/make_field_global_fixtures.py) and the float64 restatement of tests/global_oracle.py:
all nine modes, fp32 / bf16 / fp16, lroundf batch values, the shared origin key, the field / map
key collision, errors, caching and determinism."""
import os

import numpy as np
import pytest
import torch

import global_oracle as GO
import minkowskiengine_b200 as ME
from helpers import assert_one_rounding, rel_err
from minkowskiengine_b200 import _lib

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
PM = ME.PoolingMode
KERNEL = {"sum": PM.GLOBAL_SUM_POOLING_KERNEL, "avg": PM.GLOBAL_AVG_POOLING_KERNEL,
          "max": PM.GLOBAL_MAX_POOLING_KERNEL}
ORACLE = {"SUM": GO.POOL_SUM, "AVG": GO.POOL_AVG, "MAX": GO.POOL_MAX}
GLOBAL_MODES = [m for m in PM if m.name.startswith("GLOBAL_")]
DTYPES = [torch.float32, torch.bfloat16, torch.float16]
# a segment tile's fp32 sum is at most ~140 sequential additions (the rows of a lane, then the
# lanes, then the tiles): 8 * 2^-20 * A bounds their worst case at 2^-24 each
ACC = 8.0


def _oracle_mode(mode):
    return ORACLE[mode.name.split("_")[1]]


# ---- helpers shared with tests/golden/make_field_global_fixtures.py ------------------------------
POINTNET_PARAMS = ("conv1.0.linear.weight", "conv3.0.linear.weight", "conv5.0.linear.weight",
                   "linear1.0.linear.weight", "linear2.linear.weight", "linear2.linear.bias")


def pointnet_net(MEh):
    """MinkowskiPointNet with small widths and no dropout, seeded (shared with the fixture script)."""
    from examples.pointnet import pointnet
    torch.manual_seed(0)
    return pointnet(MEh, 3, 10, embedding_channel=64, channels=(16, 16, 16, 32), hidden=32,
                    dropout=0.0)


def pointnet_step(MEh, net, dev):
    """One fp32 training step on 4 clouds of float points -> (logits SparseTensor, loss)."""
    g = torch.Generator().manual_seed(12)
    B, n = 4, 700
    pts = torch.cat([torch.arange(B).repeat_interleave(n)[:, None].float(),
                     torch.rand(B * n, 3, generator=g) * 20], 1)
    perm = torch.randperm(B * n, generator=g)
    pts = pts[perm]
    feats = torch.rand(B * n, 3, generator=g) * 2 - 1
    labels = torch.randint(0, 10, (B,), generator=g)
    net = net.to(dev).train()
    out = net(MEh.TensorField(feats.to(dev), pts.to(dev)))
    loss = torch.nn.functional.cross_entropy(out.F, labels.to(dev)[out.C[:, 0].long()])
    loss.backward()
    return out, float(loss)


# ---- inputs --------------------------------------------------------------------------------------
def _points(batches, n, seed, C=8, unique=False):
    """Shuffled float points of the clouds `batches` (each present), batch values b + u that
    lroundf rounds to b (b - 0.5 among them for b > 0), and standard normal features.
    `unique`: no two points share a stride-1 voxel.  -> (pts fp32 [n, 4], feats fp64, b int)."""
    g = np.random.default_rng(seed)
    b = np.concatenate([np.asarray(batches), g.choice(batches, n - len(batches))])
    g.shuffle(b)
    u = np.where(b > 0, g.choice([-0.5, -0.49, 0.0, 0.3, 0.49], n),
                 g.choice([-0.49, 0.0, 0.49], n))
    if unique:
        cell = g.choice(64 ** 3, n, replace=False)
        xyz = np.stack(np.unravel_index(cell, (64, 64, 64)), 1) + 0.5
    else:
        xyz = g.uniform(-6, 6, (n, 3))
    pts = np.concatenate([(b + u)[:, None], xyz], 1).astype(np.float32)
    return pts, g.standard_normal((n, C)), b


def _segments(b):
    """GO.origin_segments of points with batch indices b: (origin rows [B, 4], cloud of each)."""
    coords = np.zeros((len(b), 4), np.int32)
    coords[:, 0] = b
    return GO.origin_segments(coords)


def _t(a, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a)).to(DEV, dtype)


def _np(t):
    return t.detach().double().cpu().numpy()


def _field(pts, feats, dtype=torch.float32, **kw):
    return ME.TensorField(_t(feats, dtype).requires_grad_(True), _t(pts), **kw)


def _check_pool(x, mode, seg, B, g_seed=1):
    """Pools field x in `mode` and checks output, cloud coordinates and gradient against float64."""
    y = ME.MinkowskiGlobalPooling(mode)(x)
    om = _oracle_mode(mode)
    fin = _np(x.F)
    ref, aux = GO.global_pool_forward(fin, seg, B, om)
    A, _ = GO.global_pool_forward(np.abs(fin), seg, B, om)
    assert y.F.dtype == x.F.dtype
    assert_one_rounding(y.F, _t(ref, torch.float64), _t(np.abs(ref) if om == GO.POOL_MAX else A,
                                                         torch.float64), mode.name, ACC)
    gout = torch.randn(y.F.shape, generator=torch.Generator().manual_seed(g_seed)).to(DEV,
                                                                                      x.F.dtype)
    x.F.grad = None
    y.F.backward(gout)
    gref = GO.global_pool_backward(_np(gout), seg, len(fin), om, aux)
    assert_one_rounding(x.F.grad, _t(gref, torch.float64), _t(np.abs(gref), torch.float64),
                        mode.name + " backward")
    return y


# ---- fixtures of the compiled reference ----------------------------------------------------------
@pytest.mark.parametrize("mode", ["sum", "avg", "max"])
def test_field_pooling_matches_reference(mode):
    G = np.load(os.path.join(GOLDEN, f"ref_field_global_{mode}.npz"))
    x = _field(G["pts"], G["feats"])
    y = ME.MinkowskiGlobalPooling(KERNEL[mode])(x)
    assert (y.C.cpu().numpy() == G["out_coords"]).all()
    assert rel_err(_np(y.F), G["out_feats"]) < 1e-5
    y.F.backward(_t(G["grad_out"]))
    assert rel_err(_np(x.F.grad), G["grad_in"]) < 1e-5


def test_pointnet_matches_reference():
    """examples/pointnet.py, one fp32 training step, against the compiled reference's run."""
    from helpers import state_digest
    G = np.load(os.path.join(GOLDEN, "ref_field_pointnet.npz"))
    net = pointnet_net(ME)
    assert (state_digest(net) == G["init_digest"]).all(), \
        "seeded initial weights differ from the reference's"
    out, loss = pointnet_step(ME, net, DEV)
    assert (out.C.cpu().numpy() == G["out_coords"]).all()
    F, R = out.F.detach().cpu().numpy(), G["logits"]
    assert np.abs(F - R).max() / np.abs(R).max() < 1e-3
    assert abs(loss - float(G["loss"])) / abs(float(G["loss"])) < 1e-3
    params = dict(net.named_parameters())
    for p in POINTNET_PARAMS:
        gg = params[p].grad.cpu().numpy().ravel()[G[f"{p}/idx"]].astype(np.float64)
        gr = G[f"{p}/grad"].astype(np.float64)
        err = np.abs(gg - gr).max() / float(G[f"{p}/absmax"])
        if p.startswith("linear2"):
            assert err < 2e-3, (p, err)
        else:
            # the train-mode batch norms amplify fp32 round-off: the gradients must point the same
            # way (the bound test_fcnn_matches_reference uses)
            cos = float(gg @ gr / (np.linalg.norm(gg) * np.linalg.norm(gr)))
            assert cos > 0.999 and err < 5e-2, (p, cos, err)


# ---- the float64 oracle ------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("batches", [[0, 1, 2, 3], [0, 3, 7]])
def test_all_modes_match_float64(dtype, batches):
    pts, feats, b = _points(batches, 3000, len(batches), C=12)
    origin, seg = _segments(b)
    for i, mode in enumerate(GLOBAL_MODES):
        x = _field(pts, feats, dtype)
        y = _check_pool(x, mode, seg, len(batches), g_seed=i)
        assert (y.C.cpu().numpy() == origin).all()
        assert y.coordinate_map_key == x.coordinate_manager.origin_field()


def test_batch_values_round_as_lroundf_and_one_cloud():
    pts = torch.tensor([[2.5, 0, 0, 0], [1.49, 1, 0, 0], [0.5, 2, 0, 0], [2.49, 3, 0, 0],
                        [1.5, 4, 0, 0]], device=DEV)
    f = torch.tensor([[1.0], [2.0], [4.0], [8.0], [16.0]], device=DEV)
    y = ME.MinkowskiGlobalSumPooling()(ME.TensorField(f, pts))
    # 2.5 -> 3, 1.49 -> 1, 0.5 -> 1, 2.49 -> 2, 1.5 -> 2 (half away from zero)
    assert y.C[:, 0].tolist() == [1, 2, 3] and y.F.flatten().tolist() == [6, 24, 1]
    pts1, feats1, b1 = _points([5], 900, 3)
    _, seg = _segments(b1)
    for mode in KERNEL.values():
        _check_pool(_field(pts1, feats1), mode, seg, 1)


def test_empty_cloud_and_max_ties():
    """A field holding clouds 0 and 2 of an origin built from a map of clouds 0, 1, 2; ties of the
    maximum go to the lowest point, as does their gradient."""
    m = ME.SparseTensor(torch.ones(3, 2, device=DEV),
                        torch.tensor([[0, 0, 0, 0], [1, 0, 0, 0], [2, 0, 0, 0]], dtype=torch.int32,
                                     device=DEV))
    pts = torch.tensor([[0, 1, 1, 1], [2, 0, 0, 0], [0, 2, 2, 2], [2, 5, 5, 5], [0, 3, 3, 3]],
                       dtype=torch.float32, device=DEV)
    f = torch.tensor([[1., -2.], [3., 4.], [1., -2.], [3., 9.], [1., -2.]], device=DEV,
                     requires_grad=True)
    x = ME.TensorField(f, pts, coordinate_manager=m.coordinate_manager)
    ys = ME.MinkowskiGlobalPooling(KERNEL["sum"])(x)
    assert ys.F.tolist() == [[3, -6], [0, 0], [6, 13]]
    ya = ME.MinkowskiGlobalPooling(KERNEL["avg"])(x)
    assert ya.F.tolist() == [[1, -2], [0, 0], [3, 6.5]]
    out, idx = ME.backend.GlobalPoolingForwardGPU(f.detach(), KERNEL["max"], x.coordinate_map_key,
                                                  ME.CoordinateMapKey(4), x._manager._manager,
                                                  is_field=True)
    assert out.tolist() == [[1, -2], [0, 0], [3, 9]]
    assert idx.tolist() == [[0, 1], [-1, -1], [2, 7]]
    y = ME.MinkowskiGlobalPooling(KERNEL["max"])(x)
    y.F.backward(torch.tensor([[10., 20.], [30., 40.], [50., 60.]], device=DEV))
    assert f.grad.tolist() == [[10, 20], [50, 0], [0, 0], [0, 60], [0, 0]]
    bidx, rows = m.coordinate_manager.origin_field_map(x.coordinate_field_map_key)
    assert bidx.tolist() == [0, 1, 2]
    assert [r.tolist() for r in rows] == [[0, 2, 4], [], [1, 3]]


# ---- one origin key for fields and maps ----------------------------------------------------------
def test_field_and_its_sparse_share_the_origin_key():
    pts, feats, b = _points([0, 3, 7], 2000, 5)
    x = _field(pts, feats)
    mgr = x.coordinate_manager
    yf = ME.MinkowskiGlobalMaxPooling()(x)                       # origin built from the field
    assert mgr.origin_field() == mgr.origin()
    assert mgr.origin().get_key() == ([0, 0, 0], "")
    s = x.sparse()
    ys = ME.MinkowskiGlobalMaxPooling()(s)
    assert ys.coordinate_map_key == yf.coordinate_map_key
    assert ME.cat(yf, ys).F.shape == (3, 16)
    origin, seg = _segments(b)
    bidx, rows = mgr.origin_field_map(x.coordinate_field_map_key)
    assert bidx.tolist() == [0, 3, 7] and len(rows) == 8
    for s_, bb in enumerate([0, 3, 7]):
        assert rows[bb].tolist() == np.nonzero(seg == s_)[0].tolist()
    # the map made later pools on the same origin rows
    sc = s.C.cpu().numpy()
    ref, _ = GO.global_pool_forward(_np(s.F), GO.origin_segments(sc)[1], 3, GO.POOL_MAX)
    assert rel_err(_np(ys.F), ref) < 1e-6


@pytest.mark.parametrize("unique", [False, True])
def test_field_key_equal_to_a_map_key(unique):
    """The stride-1 map of a field gets the field key's tuple; pooling either gives its own rows."""
    pts, feats, b = _points([0, 1, 2], 1500, 9, unique=unique)
    if not unique:
        pts[:, 1:] = np.floor(pts[:, 1:] / 3) * 3 + 0.25            # many points per voxel
    x = _field(pts, feats)
    _, seg = _segments(b)
    _check_pool(x, KERNEL["sum"], seg, 3)
    s = x.sparse()
    assert s.coordinate_map_key.get_key() == x.coordinate_field_map_key.get_key()
    assert (len(s) == len(pts)) == unique
    sc = s.C.cpu().numpy()
    ref, _ = GO.global_pool_forward(_np(s.F), GO.origin_segments(sc)[1], 3, GO.POOL_SUM)
    ys = ME.MinkowskiGlobalSumPooling(KERNEL["sum"])(s)
    assert rel_err(_np(ys.F), ref) < 1e-5
    for mode in KERNEL.values():
        _check_pool(x, mode, seg, 3)


# ---- errors --------------------------------------------------------------------------------------
def test_errors():
    m = ME.SparseTensor(torch.ones(2, 1, device=DEV),
                        torch.tensor([[0, 0, 0, 0], [1, 0, 0, 0]], dtype=torch.int32, device=DEV))
    mgr = m.coordinate_manager
    ME.MinkowskiGlobalSumPooling()(m)
    far = ME.TensorField(torch.ones(2, 1, device=DEV),
                         torch.tensor([[0.0, 0, 0, 0], [2.0, 0, 0, 0]], device=DEV),
                         coordinate_manager=mgr)
    with pytest.raises(RuntimeError):
        ME.MinkowskiGlobalSumPooling()(far)
    for v in (float("nan"), float("inf"), 3e9):
        bad = ME.TensorField(torch.ones(2, 1, device=DEV),
                             torch.tensor([[0.0, 0, 0, 0], [v, 0, 0, 0]], device=DEV),
                             coordinate_manager=mgr)
        with pytest.raises(ValueError):                          # grouping onto an existing origin
            ME.MinkowskiGlobalMaxPooling()(bad)
        alone = ME.TensorField(torch.ones(2, 1, device=DEV),
                               torch.tensor([[0.0, 0, 0, 0], [v, 0, 0, 0]], device=DEV))
        with pytest.raises(ValueError):                          # the origin built from the field
            ME.MinkowskiGlobalMaxPooling()(alone)
    ok = ME.TensorField(torch.ones(2, 1, device=DEV), torch.zeros(2, 4, device=DEV))
    with pytest.raises(ValueError):
        ME.MinkowskiGlobalMaxPooling()(ok, coordinates=m)
    with pytest.raises(AssertionError):
        ME.MinkowskiInstanceNorm(1).to(DEV)(ok)


# ---- caching and determinism ---------------------------------------------------------------------
def test_second_pooling_launches_only_the_reduction():
    pts, feats, _ = _points([0, 1, 2, 3], 5000, 7, C=16, unique=True)
    x = _field(pts, feats)
    s = x.sparse()                                  # rows = points: the same reduction sizes
    pool = ME.MinkowskiGlobalPooling(KERNEL["avg"])
    with torch.no_grad():
        pool(x), pool(s)
        torch.cuda.synchronize()
        n0 = _lib.launch_count()
        pool(x)
        n1 = _lib.launch_count()
        pool(s)
        n2 = _lib.launch_count()
    assert n1 - n0 == n2 - n1 == 2, (n1 - n0, n2 - n1)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_bitwise_repeats(dtype):
    pts, feats, _ = _points([0, 2, 5], 60_000, 11, C=64)
    outs = []
    for _ in range(2):
        x = _field(pts, feats, dtype)
        ys = [ME.MinkowskiGlobalPooling(m)(x).F for m in KERNEL.values()]
        sum(y.float().sum() for y in ys).backward()
        outs.append([y.detach().clone() for y in ys] + [x.F.grad.clone()])
    for a, c in zip(*outs):
        assert torch.equal(a, c)


# ---- broadcast onto fields -----------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("op", ["add", "mul", "copy", "concat"])
def test_broadcast_onto_a_field(op, dtype):
    pts, feats, b = _points([0, 3, 7], 2500, 13, C=8, unique=True)
    _, seg = _segments(b)
    gl = np.random.default_rng(2).standard_normal((3, 8))
    layer = {"add": ME.MinkowskiBroadcastAddition, "mul": ME.MinkowskiBroadcastMultiplication,
             "copy": ME.MinkowskiBroadcast, "concat": ME.MinkowskiBroadcastConcatenation}[op]()
    gout = np.random.default_rng(3).standard_normal((len(pts), 16 if op == "concat" else 8))
    results = []
    for as_field in (True, False):
        x = _field(pts, feats, dtype)
        inp = x if as_field else x.sparse()
        assert as_field or len(inp) == len(pts)
        mgr = x.coordinate_manager
        g = _t(gl, dtype).requires_grad_(True)
        glob = ME.SparseTensor(g, coordinate_map_key=mgr.origin(), coordinate_manager=mgr)
        y = layer(inp, glob)
        assert isinstance(y, ME.TensorField) == as_field
        if as_field:
            assert y.coordinate_field_map_key == x.coordinate_field_map_key
        y.F.backward(_t(gout, dtype))
        results.append((y.F.detach(), x.F.grad, g.grad))
    (yf, gxf, ggf), (ys, gxs, ggs) = results
    assert torch.equal(yf, ys) and torch.equal(ggf, ggs)
    assert (gxf is None and gxs is None) or torch.equal(gxf, gxs)
    fin, gq, dy = _np(_t(feats, dtype)), _np(_t(gl, dtype)), _np(_t(gout, dtype))
    if op in ("add", "mul"):
        code = GO.BCAST_ADD if op == "add" else GO.BCAST_MUL
        ref = GO.broadcast_forward(fin, gq, seg, code)
        aref = GO.broadcast_forward(np.abs(fin), np.abs(gq), seg, code)
        dx, dg = GO.broadcast_backward(fin, gq, dy, seg, code)
        adg = GO.broadcast_backward(np.abs(fin), np.abs(gq), np.abs(dy), seg, code)[1]
    else:
        ref = gq[seg] if op == "copy" else np.concatenate([fin, gq[seg]], 1)
        aref = np.abs(ref)
        dgo = dy if op == "copy" else dy[:, 8:]
        dg = np.zeros_like(gq)
        np.add.at(dg, seg, dgo)
        adg = np.zeros_like(gq)
        np.add.at(adg, seg, np.abs(dgo))
        dx = None if op == "copy" else dy[:, :8]
    assert_one_rounding(yf, _t(ref, torch.float64), _t(aref, torch.float64), op)
    assert_one_rounding(ggf, _t(dg, torch.float64), _t(adg, torch.float64), op + " dg", ACC)
    if dx is None:
        assert gxf is None
    else:
        assert_one_rounding(gxf, _t(dx, torch.float64), _t(np.abs(dx), torch.float64), op + " dx")
