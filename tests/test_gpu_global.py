"""Global pooling, broadcast and instance normalisation on the GPU, through the public API and
the native per-cloud kernels (csrc/global.cu), against the compiled reference's fixtures
(tests/golden/ref_global_*, ref_broadcast_*, ref_instnorm, ref_resnet, written by
tests/golden/make_global_fixtures.py), the numpy restatement (tests/global_oracle.py) and torch
autograd."""
import numpy as np
import pytest
import torch

import global_oracle as GO
from helpers import golden, rel_err, state_digest
from oracle import oracle_np as O

pytestmark = pytest.mark.gpu

def _modes(ME):
    return {"sum": ME.PoolingMode.GLOBAL_SUM_POOLING_KERNEL,
            "avg": ME.PoolingMode.GLOBAL_AVG_POOLING_KERNEL,
            "max": ME.PoolingMode.GLOBAL_MAX_POOLING_KERNEL}


def _tensor(ME, coords, feats, dev, **kw):
    return ME.SparseTensor(torch.as_tensor(feats).to(dev), torch.as_tensor(coords).to(dev), **kw)


# ---- helpers shared with tests/golden/make_global_fixtures.py (run there on the reference) ----
def _clouds(n=8000, batches=4, extent=None):
    if extent is None:
        return torch.cat([O.surface_cloud(n, seed=10 + b, batch=b) for b in range(batches)])
    # points spread over a cube `extent` wide: the stride-192 head of a ResNet keeps ~(extent/192)^3
    # voxels per cloud, so its instance norm is well conditioned (over one or two voxels the
    # normalised output is +-1 or 0 and the backward scales by 1 / |x1 - x2|, which amplifies
    # every rounding difference)
    out = []
    for b in range(batches):
        c = torch.randint(0, extent, (n, 3), generator=torch.Generator().manual_seed(10 + b),
                          dtype=torch.int32)
        c = torch.unique(c, dim=0)
        out.append(torch.cat([torch.full((len(c), 1), b, dtype=torch.int32), c], 1))
    return torch.cat(out)


def _resnet_step(MEh, net, dev):
    coords = _clouds(20_000, 4, extent=768)
    g = torch.Generator().manual_seed(4)
    feats = torch.rand(len(coords), 3, generator=g)
    labels = torch.randint(0, 40, (4,), generator=g)
    net = net.to(dev).train()
    out = net(MEh.SparseTensor(feats.to(dev), coords.to(dev)))
    # logits row s is the cloud of out.C[s, 0] (ascending here; implementation-defined there)
    loss = torch.nn.functional.cross_entropy(out.F.float(), labels.to(dev)[out.C[:, 0].long()])
    loss.backward()
    return out, float(loss)


def _se_step(MEh, blk, dev):
    coords = torch.cat([O.surface_cloud(600, seed=30 + b, batch=b) for b in range(3)])
    feats = torch.randn(len(coords), 32, generator=torch.Generator().manual_seed(5))
    blk = blk.to(dev).train()
    x = MEh.SparseTensor(feats.to(dev), coords.to(dev), requires_grad=True)
    y = blk(x)
    y.F.pow(2).mean().backward()
    return y, x


# ---- fixtures of the compiled reference ----------------------------------------------------------
@pytest.mark.parametrize("mode", ["sum", "avg", "max"])
def test_global_pooling_matches_reference(ME, cuda, mode):
    G = golden(f"ref_global_{mode}.npz")
    x = _tensor(ME, G["in_coords"], G["in_feats"], cuda, requires_grad=True)
    y = ME.MinkowskiGlobalPooling(_modes(ME)[mode])(x)
    assert (y.C.cpu().numpy() == G["out_coords"]).all()
    assert rel_err(y.F.detach().cpu(), G["out_feats"]) < 1e-5
    y.F.backward(torch.as_tensor(G["grad_out"]).to(cuda))
    assert rel_err(x.F.grad.cpu(), G["grad_in"]) < 1e-5


@pytest.mark.parametrize("mode", ["add", "mul"])
def test_broadcast_matches_reference(ME, cuda, mode):
    G = golden(f"ref_broadcast_{mode}.npz")
    x = _tensor(ME, G["in_coords"], G["in_feats"], cuda, requires_grad=True)
    pooled = ME.MinkowskiGlobalAvgPooling()(x)
    g = torch.as_tensor(G["glob_feats"]).to(cuda).requires_grad_(True)
    glob = ME.SparseTensor(g, coordinate_map_key=pooled.coordinate_map_key,
                           coordinate_manager=x.coordinate_manager)
    layer = {"add": ME.MinkowskiBroadcastAddition, "mul": ME.MinkowskiBroadcastMultiplication}[mode]()
    y = layer(x, glob)
    assert rel_err(y.F.detach().cpu(), G["out_feats"]) < 1e-5
    y.F.backward(torch.as_tensor(G["grad_out"]).to(cuda))
    assert rel_err(x.F.grad.cpu(), G["grad_in"]) < 1e-5
    assert rel_err(g.grad.cpu(), G["grad_glob"]) < 1e-5


def test_instance_norm_matches_reference(ME, cuda):
    G = golden("ref_instnorm.npz")
    x = _tensor(ME, G["in_coords"], G["in_feats"], cuda, requires_grad=True)
    layer = ME.MinkowskiInstanceNorm(x.F.shape[1]).to(cuda)
    with torch.no_grad():
        layer.weight.copy_(torch.as_tensor(G["weight"]))
        layer.bias.copy_(torch.as_tensor(G["bias"]))
    y = layer(x)
    assert rel_err(y.F.detach().cpu(), G["out_feats"]) < 1e-5
    y.F.backward(torch.as_tensor(G["grad_out"]).to(cuda))
    assert rel_err(x.F.grad.cpu(), G["grad_in"]) < 1e-4
    assert rel_err(layer.weight.grad.cpu(), G["grad_weight"]) < 1e-4
    assert rel_err(layer.bias.grad.cpu(), G["grad_bias"]) < 1e-5


# ---- our definition: origin order, edge cases ------------------------------------------------
@pytest.mark.parametrize("batches", [[0, 1, 2, 3], [0, 3, 7]])
def test_origin_is_ascending_and_pooling_matches_oracle(ME, cuda, batches):
    g = torch.Generator().manual_seed(len(batches))
    coords = torch.cat([O.surface_cloud(500 + 100 * i, seed=40 + i, batch=b)
                        for i, b in enumerate(batches)])
    coords = coords[torch.randperm(len(coords), generator=g)]          # batch rows shuffled
    feats = torch.randn(len(coords), 12, generator=g)
    x = _tensor(ME, coords, feats, cuda, requires_grad=True)
    mgr = x.coordinate_manager
    origin, seg = GO.origin_segments(x.C.cpu().numpy())
    okey = mgr.origin()
    assert okey.get_key() == ([0, 0, 0], "") and mgr.origin_map_size() == len(batches)
    assert (mgr.get_coordinates(okey).cpu().numpy() == origin).all()
    bidx, rows = mgr.origin_map(x.coordinate_map_key)
    assert bidx.tolist() == batches and len(rows) == max(batches) + 1
    for s, b in enumerate(batches):
        assert rows[b].cpu().tolist() == np.nonzero(seg == s)[0].tolist()
    fin = x.F.detach().cpu().numpy()
    for name, mode in (("sum", GO.POOL_SUM), ("avg", GO.POOL_AVG), ("max", GO.POOL_MAX)):
        y = ME.MinkowskiGlobalPooling(_modes(ME)[name])(x)
        ref, aux = GO.global_pool_forward(fin, seg, len(batches), mode)
        assert (y.C.cpu().numpy() == origin).all()
        assert rel_err(y.F.detach().cpu(), ref) < 1e-5, name
        gout = torch.rand(y.F.shape, generator=g)
        x.F.grad = None
        y.F.backward(gout.to(cuda))
        gref = GO.global_pool_backward(gout.numpy(), seg, len(fin), mode, aux)
        assert rel_err(x.F.grad.cpu(), gref) < 1e-5, name
    # broadcast follows the same origin order
    gl = torch.randn(len(batches), 12, generator=g)
    glob = ME.SparseTensor(gl.to(cuda), coordinate_map_key=okey, coordinate_manager=mgr)
    yb = ME.MinkowskiBroadcastAddition()(x, glob)
    assert rel_err(yb.F.detach().cpu(), GO.broadcast_forward(fin, gl.numpy(), seg, GO.BCAST_ADD)) < 1e-6
    yc = ME.MinkowskiBroadcastConcatenation()(x, glob)
    assert (yc.F[:, 12:].cpu() == gl[torch.as_tensor(seg)]).all()


def test_single_cloud_max_gradient_matches_autograd(ME, cuda):
    coords = O.surface_cloud(3000, seed=7)
    feats = torch.randn(3000, 16, generator=torch.Generator().manual_seed(7))
    x = _tensor(ME, coords, feats, cuda, requires_grad=True)
    y = ME.MinkowskiGlobalMaxPooling()(x)
    gout = torch.rand(1, 16, generator=torch.Generator().manual_seed(8))
    y.F.backward(gout.to(cuda))
    ft = x.F.detach().cpu().clone().requires_grad_(True)
    ref = ft.max(0, keepdim=True).values
    ref.backward(gout)
    assert torch.equal(y.F.detach().cpu(), ref.detach())
    assert torch.equal(x.F.grad.cpu(), ft.grad)


def test_single_voxel_clouds_and_empty_segments(ME, cuda):
    coords = torch.tensor([[0, 1, 2, 3], [1, 4, 4, 4], [1, 5, 5, 5], [2, 9, 9, 9]], dtype=torch.int32)
    feats = torch.tensor([[1., -2.], [3., 4.], [5., -6.], [-7., 8.]])
    x = _tensor(ME, coords, feats, cuda, requires_grad=True)
    for mode, want in (("sum", [[1, -2], [8, -2], [-7, 8]]), ("avg", [[1, -2], [4, -1], [-7, 8]]),
                       ("max", [[1, -2], [5, 4], [-7, 8]])):
        y = ME.MinkowskiGlobalPooling(_modes(ME)[mode])(x)
        assert y.F.detach().cpu().tolist() == want, mode
    # a map holding clouds 0 and 2 only: cloud 1 is an empty segment of the manager's origin map
    mgr = x.coordinate_manager
    sub = torch.tensor([[0, 7, 7, 7], [2, 1, 1, 1], [2, 2, 2, 2]], dtype=torch.int32, device=cuda)
    key, _ = mgr.insert_and_map(sub, 1, "sub")
    f = torch.tensor([[2., 3.], [4., -1.], [1., 5.]], device=cuda, requires_grad=True)
    xs = ME.SparseTensor(f, coordinate_map_key=key, coordinate_manager=mgr)
    fn = ME.MinkowskiGlobalPoolingFunction
    out_s = fn.apply(f, _modes(ME)["sum"], key, None, mgr)
    assert out_s.detach().cpu().tolist() == [[2, 3], [0, 0], [5, 4]]
    out_m, aux = ME.backend.GlobalPoolingForwardGPU(f.detach(), _modes(ME)["max"], key,
                                                    ME.CoordinateMapKey(4), mgr._manager)
    assert out_m.cpu().tolist() == [[2, 3], [0, 0], [4, 5]]
    assert aux.cpu().tolist() == [[0, 1], [-1, -1], [2, 5]]
    _, cnt = ME.backend.GlobalPoolingForwardGPU(f.detach(), _modes(ME)["avg"], key,
                                                ME.CoordinateMapKey(4), mgr._manager)
    assert cnt.cpu().tolist() == [1, 0, 2]
    ya = ME.MinkowskiGlobalAvgPooling()(xs)
    ya.F.sum().backward()
    assert f.grad.cpu().tolist() == [[1, 1], [0.5, 0.5], [0.5, 0.5]]
    # a batch index the origin map does not hold
    bad, _ = mgr.insert_and_map(torch.tensor([[5, 0, 0, 0]], dtype=torch.int32, device=cuda), 1,
                                "bad")
    with pytest.raises(RuntimeError):
        fn.apply(torch.ones(1, 2, device=cuda), _modes(ME)["sum"], bad, None, mgr)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_low_precision_within_one_output_rounding(ME, cuda, dtype):
    coords = _clouds(3000, 3)
    g = torch.Generator().manual_seed(11)
    feats = torch.randn(len(coords), 64, generator=g).to(dtype)
    # half an ulp, relative; tiny is half the fp16 subnormal spacing (results near zero)
    eps = 2.0 ** -8 if dtype == torch.bfloat16 else 2.0 ** -11
    tiny = 2.0 ** -25
    x32 = _tensor(ME, coords, feats.float(), cuda, requires_grad=True)
    xl = _tensor(ME, coords, feats, cuda, requires_grad=True)
    gout = torch.randn(len(coords), 64, generator=g).to(dtype)
    for name in ("sum", "avg", "max"):
        a = ME.MinkowskiGlobalPooling(_modes(ME)[name])(x32).F
        b = ME.MinkowskiGlobalPooling(_modes(ME)[name])(xl).F
        assert b.dtype == dtype
        assert ((b.float() - a).abs() <= eps * a.abs() + tiny).all(), name
    gl = torch.rand(3, 64, generator=g).to(dtype)
    for layer in (ME.MinkowskiBroadcastAddition(), ME.MinkowskiBroadcastMultiplication()):
        glob32 = ME.SparseTensor(gl.float().to(cuda), coordinate_map_key=x32.coordinate_manager.origin(),
                                 coordinate_manager=x32.coordinate_manager)
        globl = ME.SparseTensor(gl.to(cuda), coordinate_map_key=xl.coordinate_manager.origin(),
                                coordinate_manager=xl.coordinate_manager)
        a, b = layer(x32, glob32).F, layer(xl, globl).F
        assert ((b.float() - a).abs() <= eps * a.abs() + tiny).all()
    n32, nl = ME.MinkowskiInstanceNorm(64).to(cuda), ME.MinkowskiInstanceNorm(64).to(cuda)
    a, b = n32(x32).F, nl(xl).F
    assert b.dtype == dtype
    assert ((b.float() - a).abs() <= eps * a.abs() + 1e-4).all()
    a.backward(gout.float().to(cuda))
    b.backward(gout.to(cuda))
    ga, gb = x32.F.grad, xl.F.grad.float()
    # the gradient's inputs are the rounded normalised features: a few roundings, not one
    assert ((gb - ga).abs() <= 4 * eps * ga.abs().max()).all()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_multi_tile_segments_are_bitwise_deterministic(ME, cuda, dtype):
    """8 clouds x 100k rows x 96 channels: every segment spans ~200 row tiles."""
    n, B, C = 100_000, 8, 96
    g = torch.Generator(device=cuda).manual_seed(3)
    b = torch.arange(B, device=cuda, dtype=torch.int32).repeat_interleave(n)
    xyz = torch.arange(n, device=cuda, dtype=torch.int32).repeat(B)
    coords = torch.stack([b, xyz % 97, (xyz // 97) % 101, xyz // 9797], 1).int().contiguous()
    feats = torch.randn(B * n, C, device=cuda, generator=g).to(dtype)
    gout = torch.randn(B * n, C, device=cuda, generator=g).to(dtype)
    outs = []
    for _ in range(2):
        x = ME.SparseTensor(feats.clone(), coords, requires_grad=True)
        y = [ME.MinkowskiGlobalPooling(m)(x).F for m in _modes(ME).values()]
        z = ME.MinkowskiInstanceNorm(C).to(cuda)(x).F
        z.backward(gout)
        yb = ME.MinkowskiBroadcastMultiplication()(x, ME.SparseTensor(
            y[1].detach().requires_grad_(True), coordinate_map_key=x.coordinate_manager.origin(),
            coordinate_manager=x.coordinate_manager)).F
        outs.append([t.detach().clone() for t in y + [z, x.F.grad, yb]])
    for a, c in zip(*outs):
        assert torch.equal(a, c)
    ref = feats.double().view(B, n, C).sum(1)
    assert rel_err(outs[0][0].double().cpu(), ref.cpu()) < (1e-6 if dtype == torch.float32 else 4e-3)


# ---- networks ----------------------------------------------------------------------------------
def test_resnet14_fp32_matches_reference(ME, cuda):
    from examples.resnet import resnet
    G = golden("ref_resnet.npz")
    torch.manual_seed(0)
    net = resnet("ResNet14", ME, 3, 40, 3, dropout=0.0)
    assert (state_digest(net) == G["resnet/init_digest"]).all(), \
        "seeded initial weights differ from the reference's"
    out, loss = _resnet_step(ME, net, cuda)
    assert (out.C.cpu().numpy() == G["resnet/out_coords"]).all()
    F, R = out.F.detach().cpu().numpy(), G["resnet/logits"]
    assert np.abs(F - R).max() / np.abs(R).max() < 1e-3
    assert abs(loss - float(G["resnet/loss"])) / abs(float(G["resnet/loss"])) < 1e-3
    # as in test_gpu_network.py: the layers next to the loss tightly; below them fp32 round-off is
    # amplified by the train-mode batch norms (observed 2.6e-2 of the max at layer2, direction
    # unchanged), so the deep layers are asserted to point the same way
    params = dict(net.named_parameters())
    for p in ("conv1.0.kernel", "layer2.0.conv1.kernel", "conv5.1.kernel", "final.linear.weight"):
        gg = params[p].grad.cpu().numpy().ravel()[G[f"resnet/{p}/idx"]].astype(np.float64)
        gr = G[f"resnet/{p}/grad"].astype(np.float64)
        if p in ("conv5.1.kernel", "final.linear.weight"):
            assert np.abs(gg - gr).max() / float(G[f"resnet/{p}/absmax"]) < 2e-3, p
        else:
            cos = float(gg @ gr / (np.linalg.norm(gg) * np.linalg.norm(gr)))
            assert cos > 0.9995 and np.abs(gg - gr).max() / float(G[f"resnet/{p}/absmax"]) < 5e-2, p


def test_se_block_matches_reference(ME, cuda):
    from examples.resnet import se_basic_block
    G = golden("ref_resnet.npz")
    torch.manual_seed(1)
    blk = se_basic_block(ME, 32, 32, dimension=3)
    assert (state_digest(blk) == G["se/init_digest"]).all()
    y, x = _se_step(ME, blk, cuda)
    assert rel_err(y.F.detach().cpu(), G["se/out_feats"]) < 1e-4
    assert rel_err(x.F.grad.cpu(), G["se/grad_in"]) < 1e-3
    for p, t in blk.named_parameters():
        if f"se/{p}/grad" in G:
            assert rel_err(t.grad.cpu(), G[f"se/{p}/grad"]) < 1e-3, p
