"""CPU tests of global pooling, broadcast and instance normalisation: the numpy restatements
(tests/global_oracle.py) match the compiled reference's fixtures (tests/golden/ref_global_*, ref_broadcast_*,
ref_instnorm), the ResNet / SE-block definitions match the reference's parameter counts, and the
new ops refuse CPU tensors and local pooling modes."""
import numpy as np
import pytest
import torch

from helpers import golden, rel_err
import global_oracle as O

MODES = {"sum": O.POOL_SUM, "avg": O.POOL_AVG, "max": O.POOL_MAX}


@pytest.mark.parametrize("mode", ["sum", "avg", "max"])
def test_oracle_global_pooling_matches_reference(mode):
    G = golden(f"ref_global_{mode}.npz")
    origin, seg = O.origin_segments(G["in_coords"])
    assert (origin == G["out_coords"]).all()
    out, aux = O.global_pool_forward(G["in_feats"], seg, len(origin), MODES[mode])
    assert rel_err(out, G["out_feats"]) < 1e-6
    gin = O.global_pool_backward(G["grad_out"], seg, len(seg), MODES[mode], aux)
    assert rel_err(gin, G["grad_in"]) < 1e-6


@pytest.mark.parametrize("mode", ["add", "mul"])
def test_oracle_broadcast_matches_reference(mode):
    G = golden(f"ref_broadcast_{mode}.npz")
    op = O.BCAST_ADD if mode == "add" else O.BCAST_MUL
    _, seg = O.origin_segments(G["in_coords"])
    y = O.broadcast_forward(G["in_feats"], G["glob_feats"], seg, op)
    assert rel_err(y, G["out_feats"]) < 1e-6
    dx, dg = O.broadcast_backward(G["in_feats"], G["glob_feats"], G["grad_out"], seg, op)
    assert rel_err(dx, G["grad_in"]) < 1e-6 and rel_err(dg, G["grad_glob"]) < 1e-5


def test_oracle_instance_norm_matches_reference():
    G = golden("ref_instnorm.npz")
    origin, seg = O.origin_segments(G["in_coords"])
    y, inv_std = O.instance_norm_forward(G["in_feats"], seg, len(origin))
    w, b = G["weight"].astype(np.float64), G["bias"].astype(np.float64)
    assert rel_err(y * w + b, G["out_feats"]) < 1e-5
    gy = G["grad_out"] * w
    assert rel_err(O.instance_norm_backward(gy, y, inv_std, seg, len(origin)), G["grad_in"]) < 1e-4
    assert rel_err((G["grad_out"] * y).sum(0, keepdims=True), G["grad_weight"]) < 1e-4
    assert rel_err(G["grad_out"].sum(0, keepdims=True), G["grad_bias"]) < 1e-5


def test_oracle_origin_order_and_empty_segments():
    coords = np.array([[7, 1, 1, 1], [0, 2, 2, 2], [3, 0, 0, 0], [7, 5, 5, 5]], np.int32)
    origin, seg = O.origin_segments(coords)
    assert origin[:, 0].tolist() == [0, 3, 7] and (origin[:, 1:] == 0).all()
    assert seg.tolist() == [2, 0, 1, 2]
    x = np.arange(8, dtype=np.float64).reshape(4, 2)
    out, aux = O.global_pool_forward(x, seg, 4, O.POOL_MAX)     # segment 3 is empty
    assert out[3].tolist() == [0, 0] and aux[3].tolist() == [-1, -1]
    assert aux[2].tolist() == [6, 7]                             # row 3 holds the maximum


def test_resnet_and_se_block_parameter_counts_match_reference():
    import minkowskiengine_b200 as ME
    from examples.resnet import resnet, se_basic_block
    counts = {"ResNet14": 21_442_408}
    net = resnet("ResNet14", ME, 3, 40, 3)
    assert sum(p.numel() for p in net.parameters()) == counts["ResNet14"]
    assert sum(1 for m in net.modules() if isinstance(m, ME.MinkowskiInstanceNorm)) == 2
    blk = se_basic_block(ME, 64, 64, dimension=3)
    assert sum(p.numel() for p in blk.parameters()) == 2 * 27 * 64 * 64 + 4 * 64 + 64 * 4 + 4 + 4 * 64 + 64
    mod = ME.modules.SEBasicBlock(64, 64, D=3)
    assert sum(p.numel() for p in mod.parameters()) == sum(p.numel() for p in blk.parameters())
    assert resnet("ResNet14", ME, dropout=0.0).conv5[0].module.p == 0.0


def test_global_ops_reject_cpu_tensors_and_local_modes():
    import minkowskiengine_b200 as ME
    from minkowskiengine_b200 import backend as _C
    mgr = _C.CoordinateMapManagerGPU_c10()
    key = ME.CoordinateMapKey([1, 1, 1], "")
    feats = torch.rand(4, 3)
    with pytest.raises(RuntimeError):
        _C.GlobalPoolingForwardGPU(feats, ME.PoolingMode.GLOBAL_SUM_POOLING_KERNEL, key,
                                   ME.CoordinateMapKey(4), mgr)
    with pytest.raises(RuntimeError):
        _C.BroadcastForwardGPU(feats, torch.rand(1, 3), ME.BroadcastMode.ELEMENTWISE_ADDITON, key,
                               key, mgr)
    with pytest.raises(RuntimeError):
        _C.BroadcastBackwardGPU(feats, torch.rand(1, 3), feats, ME.BroadcastMode.ELEMENTWISE_ADDITON,
                                key, key, mgr)
    with pytest.raises(RuntimeError):
        _C.GlobalPoolingBackwardGPU(feats, torch.rand(1, 3), torch.rand(1),
                                    ME.PoolingMode.GLOBAL_AVG_POOLING_KERNEL, key, key, mgr)
    if torch.cuda.is_available():
        coords = torch.zeros((4, 4), dtype=torch.int32, device="cuda")
        coords[:, 1] = torch.arange(4)
        k, _ = mgr.insert_and_map(coords, [1, 1, 1], "")
        f = torch.rand(4, 3, device="cuda")
        for mode in (ME.PoolingMode.LOCAL_SUM_POOLING, ME.PoolingMode.LOCAL_MAX_POOLING):
            with pytest.raises(RuntimeError, match="pooling mode"):
                _C.GlobalPoolingForwardGPU(f, mode, k, ME.CoordinateMapKey(4), mgr)
    else:
        with pytest.raises(RuntimeError):
            _C.GlobalPoolingForwardGPU(feats, ME.PoolingMode.LOCAL_SUM_POOLING, key,
                                       ME.CoordinateMapKey(4), mgr)
