"""Pruning, union and arithmetic between sparse tensors on different coordinate maps on the GPU,
through the public API and the native kernels (csrc/union.cu), against the compiled reference's
fixtures (tests/golden/ref_prune, ref_union, ref_binary_*, ref_completion, written by
tests/golden/make_generative_fixtures.py) and torch autograd."""
import numpy as np
import pytest
import torch

from helpers import golden, rel_err, state_digest

pytestmark = pytest.mark.gpu

COMPLETION_SEED = 3
COMPLETION_CHANNELS = (8, 16, 32, 64)      # 3 levels: tensor strides 1, 2, 4, 8
# The classifiers start with bias -1.5 (a prior of "mostly empty", about 3 standard deviations of
# the initial logits, which have a spread of about 0.5): zero is crossed only in the tail of the
# logit distribution, where few logits lie.  With this seed and bias, every level still keeps
# some voxels by prediction, and no logit lies within 1e-2 of zero.  That is far above the fp32
# rounding error of a logit, which does not depend on the bias.  So a different summation order
# cannot flip a pruning decision.  (Scaling weight and bias together would not help: it scales
# each logit and its error alike.)
COMPLETION_CLS_BIAS = -1.5


def canon(coords):
    c = np.asarray(coords)
    return np.lexsort(c.T[::-1])


def _to_ours(g_canon, coords, dev):
    """A gradient stored in canonical row order, in the row order of `coords`."""
    perm = canon(coords)
    g = torch.empty(g_canon.shape, dtype=torch.float32)
    g[torch.as_tensor(perm)] = torch.as_tensor(g_canon)
    return g.to(dev)


def _sorted(y):
    c = y.C.cpu().numpy()
    perm = canon(c)
    return c[perm], y.F.detach().float().cpu().numpy()[perm]


def _inputs(ME, dev, coords_list, feats_list, dtype=torch.float32):
    xs, mgr = [], None
    for c, f in zip(coords_list, feats_list):
        x = ME.SparseTensor(torch.as_tensor(f).to(dtype).to(dev), torch.as_tensor(c).to(dev),
                            coordinate_manager=mgr, requires_grad=True)
        mgr = x.coordinate_manager
        xs.append(x)
    return xs


# ---- shared with tests/golden/make_generative_fixtures.py (run there on the reference) ----------
def _completion_step(MEh, net, dev):
    from examples.completion import completion_loss, shell_pair
    pairs = [shell_pair(12.6, seed=60 + b, batch=b) for b in range(2)]
    partial = torch.cat([p for p, _ in pairs])
    full = torch.cat([f for _, f in pairs])
    net = net.to(dev).train()
    with torch.no_grad():
        for cls in net.dec_cls:
            cls.bias.fill_(COMPLETION_CLS_BIAS)
    x = MEh.SparseTensor(torch.ones(len(partial), 1).to(dev), partial.to(dev))
    target_key, _ = x.coordinate_manager.insert_and_map(full.to(dev), string_id="target")
    out_cls, targets, final = net(x, target_key)
    loss = completion_loss(out_cls, targets)
    loss.backward()
    return out_cls, targets, final, float(loss)


# ---- fixtures of the compiled reference --------------------------------------------------------
def test_pruning_matches_reference(ME, cuda):
    G = golden("ref_prune.npz")
    x = _inputs(ME, cuda, [G["in_coords"]], [G["in_feats"]])[0]
    keep = torch.as_tensor(G["keep"]).to(cuda)
    y = ME.MinkowskiPruning()(x, keep)
    # rows of the pruned map: the kept rows in ascending input order
    assert torch.equal(y.C, x.C[keep])
    c, f = _sorted(y)
    assert (c == G["out_coords"]).all()
    assert rel_err(f, G["out_feats"]) < 1e-5
    y.F.backward(_to_ours(G["grad_out"], y.C.cpu().numpy(), cuda))
    assert rel_err(x.F.grad.cpu(), G["grad_in"]) < 1e-5


def test_union_matches_reference(ME, cuda):
    G = golden("ref_union.npz")
    xs = _inputs(ME, cuda, [G[f"in_coords_{i}"] for i in range(3)],
                 [G[f"in_feats_{i}"] for i in range(3)])
    y = ME.MinkowskiUnion()(*xs)
    c, f = _sorted(y)
    assert (c == G["out_coords"]).all()
    assert rel_err(f, G["out_feats"]) < 1e-5
    y.F.backward(_to_ours(G["grad_out"], y.C.cpu().numpy(), cuda))
    for i, x in enumerate(xs):
        assert rel_err(x.F.grad.cpu(), G[f"grad_in_{i}"]) < 1e-5, i


@pytest.mark.parametrize("name", ["add", "sub", "mul", "div"])
def test_binary_on_different_maps_matches_reference(ME, cuda, name):
    G = golden(f"ref_binary_{name}.npz")
    a, b = _inputs(ME, cuda, [G["in_coords_0"], G["in_coords_1"]],
                   [G["in_feats_0"], G["in_feats_1"]])
    assert a.coordinate_map_key != b.coordinate_map_key
    y = {"add": lambda p, q: p + q, "sub": lambda p, q: p - q, "mul": lambda p, q: p * q,
         "div": lambda p, q: p / q}[name](a, b)
    c, f = _sorted(y)
    assert (c == G["out_coords"]).all()
    assert rel_err(f, G["out_feats"]) < 1e-5
    y.F.backward(_to_ours(G["grad_out"], y.C.cpu().numpy(), cuda))
    assert rel_err(a.F.grad.cpu(), G["grad_in_0"]) < 1e-5
    assert rel_err(b.F.grad.cpu(), G["grad_in_1"]) < 1e-5


# ---- our definition: row order, caching, edge cases, errors -------------------------------------
def _two(ME, cuda, C=4):
    ca = torch.tensor([[0, 0, 0, 0], [0, 1, 0, 0], [1, 2, 2, 2], [0, 3, 0, 0]], dtype=torch.int32)
    cb = torch.tensor([[0, 5, 5, 5], [0, 1, 0, 0], [1, 2, 2, 2], [1, 7, 7, 7]], dtype=torch.int32)
    g = torch.Generator().manual_seed(5)
    return _inputs(ME, cuda, [ca, cb], [torch.randn(4, C, generator=g) + 3,
                                        torch.randn(4, C, generator=g) + 3])


def test_union_row_order_map_and_cache(ME, cuda):
    a, b = _two(ME, cuda)
    mgr = a.coordinate_manager
    y = a + b
    want = torch.tensor([[0, 0, 0, 0], [0, 1, 0, 0], [1, 2, 2, 2], [0, 3, 0, 0], [0, 5, 5, 5],
                         [1, 7, 7, 7]], dtype=torch.int32)
    assert torch.equal(y.C.cpu(), want)
    assert y.tensor_stride == [1, 1, 1]
    out_key = ME.CoordinateMapKey(4)
    maps = mgr.union_map([a.coordinate_map_key, b.coordinate_map_key], out_key)
    assert out_key == y.coordinate_map_key          # cached per ordered tuple of keys
    assert maps[0].dtype == torch.int64
    assert maps[0].cpu().tolist() == [[0, 1, 2, 3], [0, 1, 2, 3]]
    assert maps[1].cpu().tolist() == [[0, 1, 2, 3], [4, 1, 2, 5]]
    assert (a + b).coordinate_map_key == y.coordinate_map_key
    assert (b + a).coordinate_map_key != y.coordinate_map_key
    # piecewise semantics: self-only rows keep a, other-only rows op(0, b), shared rows op(a, b)
    A, B = a.F.detach(), b.F.detach()
    for op in (lambda p, q: p + q, lambda p, q: p - q, lambda p, q: p * q, lambda p, q: p / q):
        F = op(a, b).F.detach()
        assert torch.equal(F[0], A[0]) and torch.equal(F[3], A[3])
        assert torch.equal(F[1], op(A[1], B[1])) and torch.equal(F[2], op(A[2], B[2]))
        assert torch.equal(F[4], op(torch.zeros_like(B[0]), B[0]))
        assert torch.equal(F[5], op(torch.zeros_like(B[3]), B[3]))
    # the same-key path is unchanged
    z = a + a
    assert z.coordinate_map_key == a.coordinate_map_key
    assert torch.equal(z.F, a.F + a.F)


@pytest.mark.parametrize("name", ["add", "sub", "mul", "div"])
def test_binary_gradients_match_autograd(ME, cuda, name):
    a, b = _two(ME, cuda, C=8)
    op = {"add": lambda p, q: p + q, "sub": lambda p, q: p - q, "mul": lambda p, q: p * q,
          "div": lambda p, q: p / q}[name]
    y = op(a, b)
    g = torch.randn(y.F.shape, generator=torch.Generator().manual_seed(9)).to(cuda)
    y.F.backward(g)
    # the reference's torch composition (MinkowskiTensor.py:522-540) on the same union map
    maps = a.coordinate_manager.union_map([a.coordinate_map_key, b.coordinate_map_key],
                                          ME.CoordinateMapKey(4))
    fa = a.F.detach().clone().requires_grad_(True)
    fb = b.F.detach().clone().requires_grad_(True)
    out = torch.zeros(y.F.shape, device=cuda)
    out[maps[0][1]] = fa[maps[0][0]]
    out[maps[1][1]] = op(out[maps[1][1]], fb[maps[1][0]])
    out.backward(g)
    assert torch.allclose(y.F.detach(), out.detach(), rtol=1e-6, atol=0)
    assert torch.allclose(a.F.grad, fa.grad, rtol=1e-6, atol=0)
    assert torch.allclose(b.F.grad, fb.grad, rtol=1e-6, atol=0)


def test_empty_keep_all_and_zero_row_inputs(ME, cuda):
    a, b = _two(ME, cuda)
    prune = ME.MinkowskiPruning()
    with pytest.warns(UserWarning):
        e = prune(a, torch.zeros(4, dtype=torch.bool, device=cuda))
    assert e.F.shape == (0, 4) and e.C.shape == (0, 4)
    e.F.sum().backward()
    assert torch.equal(a.F.grad, torch.zeros_like(a.F))
    a.F.grad = None
    k = prune(a, torch.ones(4, dtype=torch.uint8, device=cuda))
    assert k.coordinate_map_key != a.coordinate_map_key
    assert torch.equal(k.C, a.C) and torch.equal(k.F, a.F)
    # a union with a 0-row input, and a pruned-away tensor added to a full one
    u = ME.MinkowskiUnion()(a, e, b)
    v = ME.MinkowskiUnion()(a, b)
    assert torch.equal(u.C, v.C) and torch.equal(u.F, v.F)
    w = e + b
    assert torch.equal(w.C, b.C) and torch.equal(w.F, b.F)
    w.F.sum().backward()
    assert torch.equal(b.F.grad, torch.ones_like(b.F))
    # an empty map can be pruned again and is empty
    assert prune(e, torch.zeros(0, dtype=torch.bool, device=cuda)).F.shape == (0, 4)


def test_argument_errors(ME, cuda):
    a, b = _two(ME, cuda)
    mgr = a.coordinate_manager._manager
    key = lambda: ME.CoordinateMapKey(4)
    fwd = ME.backend.PruningForwardGPU
    keep = torch.ones(4, dtype=torch.bool, device=cuda)
    with pytest.raises(RuntimeError, match="boolean"):
        fwd(a.F.detach(), keep.float(), a.coordinate_map_key, key(), mgr)
    with pytest.raises(RuntimeError, match="keep.dim"):
        fwd(a.F.detach(), keep.view(2, 2), a.coordinate_map_key, key(), mgr)
    with pytest.raises(RuntimeError, match="keep size mismatch"):
        fwd(a.F.detach(), keep[:3], a.coordinate_map_key, key(), mgr)
    with pytest.raises(RuntimeError, match="device"):
        fwd(a.F.detach(), keep.cpu(), a.coordinate_map_key, key(), mgr)
    with pytest.raises(RuntimeError, match="in_feat.dim"):
        fwd(a.F.detach()[:, 0].contiguous(), keep, a.coordinate_map_key, key(), mgr)
    with pytest.raises(RuntimeError, match="Invalid in_feat size"):
        fwd(b.F.detach()[:3].contiguous(), keep[:3], a.coordinate_map_key, key(), mgr)
    # a union needs one tensor stride
    s = ME.MinkowskiConvolution(4, 4, kernel_size=2, stride=2, dimension=3).to(cuda)(a)
    with pytest.raises(RuntimeError, match="tensor stride"):
        a + s
    with pytest.raises(RuntimeError, match="tensor stride"):
        a.coordinate_manager.union_map([a.coordinate_map_key, s.coordinate_map_key],
                                       ME.CoordinateMapKey(4))


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_low_precision_within_one_output_rounding(ME, cuda, dtype):
    eps = 2.0 ** -8 if dtype == torch.bfloat16 else 2.0 ** -11
    G = golden("ref_binary_div.npz")
    coords = [G["in_coords_0"], G["in_coords_1"]]
    feats = [torch.as_tensor(G["in_feats_0"]).to(dtype), torch.as_tensor(G["in_feats_1"]).to(dtype)]
    lo = _inputs(ME, cuda, coords, feats, dtype)
    hi = _inputs(ME, cuda, coords, [f.float() for f in feats])
    g = torch.randn(4096, feats[0].shape[1], generator=torch.Generator().manual_seed(3)).to(dtype)
    for name, op in (("add", lambda p, q: p + q), ("sub", lambda p, q: p - q),
                     ("mul", lambda p, q: p * q), ("div", lambda p, q: p / q),
                     ("union", lambda p, q: ME.MinkowskiUnion()(p, q)),
                     ("prune", lambda p, q: ME.MinkowskiPruning()(p, p.F[:, 0].detach() > 0))):
        for x in lo + hi:
            x.F.grad = None
        yl, yh = op(*lo), op(*hi)
        assert yl.F.dtype == dtype and torch.equal(yl.C, yh.C), name
        a = yh.F.detach()
        assert ((yl.F.detach().float() - a).abs() <= eps * a.abs()).all(), name
        gg = g[:len(yl.F)].to(cuda)
        yl.F.backward(gg)
        yh.F.backward(gg.float())
        for xl, xh in zip(lo, hi):
            if xh.F.grad is None:
                continue
            # the fp32 gradient of the same rounded inputs and output gradient, rounded once
            ref = xh.F.grad
            assert ((xl.F.grad.float() - ref).abs() <= eps * ref.abs()).all(), name


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_bitwise_determinism_at_scale(ME, cuda, dtype):
    """8 clouds x 100k rows x 96 channels: prune, union and mul on different maps, twice."""
    n, B, C = 100_000, 8, 96
    g = torch.Generator(device=cuda).manual_seed(3)
    b = torch.arange(B, device=cuda, dtype=torch.int32).repeat_interleave(n)
    xyz = torch.arange(n, device=cuda, dtype=torch.int32).repeat(B)
    ca = torch.stack([b, xyz % 97, (xyz // 97) % 101, xyz // 9797], 1).int().contiguous()
    cb = ca.clone()
    cb[:, 1] += 48                                       # about half the rows shared
    fa = torch.randn(B * n, C, device=cuda, generator=g).to(dtype)
    fb = (torch.rand(B * n, C, device=cuda, generator=g) + 0.5).to(dtype)
    keep = torch.rand(B * n, device=cuda, generator=g) < 0.5
    outs = []
    for _ in range(2):
        x, y = _inputs(ME, cuda, [ca, cb], [fa.clone(), fb.clone()], dtype)
        p = ME.MinkowskiPruning()(x, keep)
        u = ME.MinkowskiUnion()(x, y)
        m = x * y
        res = [p.F, u.F, m.F]
        for t in res:
            t.backward(torch.ones_like(t) * 0.5, retain_graph=False)
        outs.append([t.detach().clone() for t in res] + [x.F.grad.clone(), y.F.grad.clone()])
    for a, c in zip(*outs):
        assert torch.equal(a, c)
    assert outs[0][1].shape[0] > B * n                   # the union is larger than either input


# ---- the completion network ------------------------------------------------------------------
def test_completion_net_matches_reference(ME, cuda):
    from examples.completion import completion_net
    G = golden("ref_completion.npz")
    torch.manual_seed(COMPLETION_SEED)
    net = completion_net(ME, COMPLETION_CHANNELS, COMPLETION_CHANNELS)
    assert (state_digest(net) == G["init_digest"]).all(), \
        "seeded initial weights differ from the reference's"
    out_cls, targets, final, loss = _completion_step(ME, net, cuda)
    for j, (o, t) in enumerate(zip(out_cls, targets)):
        c = o.C.cpu().numpy()
        perm = canon(c)
        assert (c[perm] == G[f"level{j}/coords"]).all(), j
        assert (t.cpu().numpy()[perm] == G[f"level{j}/target"]).all(), j
        F, R = o.F.detach().cpu().numpy()[perm, 0], G[f"level{j}/logits"]
        assert np.abs(F - R).max() / np.abs(R).max() < 1e-3, j
        # no pruning decision can have flipped: every logit is closer to the reference's than
        # the reference's logits are to the threshold
        assert np.abs(F - R).max() < np.abs(R).min(), j
        keep = o.F.detach().cpu().numpy()[:, 0] > 0
        if j < len(out_cls) - 1:
            keep |= t.cpu().numpy()
        kc = c[keep]
        assert (kc[canon(kc)] == G[f"level{j}/kept_coords"]).all(), j
    fc = final.C.cpu().numpy()
    assert (fc[canon(fc)] == G["final_coords"]).all()
    assert abs(loss - float(G["loss"])) / abs(float(G["loss"])) < 1e-3
    params = dict(net.named_parameters())
    for p in ("enc_block_s1.0.kernel", "enc_blocks.1.0.kernel", "dec_blocks.0.0.kernel",
              "dec_blocks.2.3.kernel", "dec_cls.2.kernel", "dec_cls.2.bias"):
        gg = params[p].grad.cpu().numpy().ravel()[G[f"{p}/idx"]].astype(np.float64)
        gr = G[f"{p}/grad"].astype(np.float64)
        cos = float(gg @ gr / (np.linalg.norm(gg) * np.linalg.norm(gr)))
        assert cos > 0.9995 and np.abs(gg - gr).max() / float(G[f"{p}/absmax"]) < 5e-2, p


def test_completion_net_trains_in_bf16(ME, cuda):
    from examples.completion import completion_loss, completion_net, shell_pair
    torch.manual_seed(0)
    net = completion_net(ME, (16, 32, 64, 128, 256), (16, 32, 64, 128, 256)).to(cuda).train()
    opt = torch.optim.SGD(net.parameters(), lr=0.1, momentum=0.9)
    pairs = [shell_pair(20.0, seed=70 + b, batch=b) for b in range(4)]
    partial = torch.cat([p for p, _ in pairs]).to(cuda)
    full = torch.cat([f for _, f in pairs]).to(cuda)
    for _ in range(3):
        opt.zero_grad()
        x = ME.SparseTensor(torch.ones(len(partial), 1, dtype=torch.bfloat16, device=cuda), partial)
        target_key, _ = x.coordinate_manager.insert_and_map(full, string_id="target")
        out_cls, targets, final = net(x, target_key)
        assert all(o.F.dtype == torch.bfloat16 for o in out_cls)
        loss = completion_loss(out_cls, targets)
        loss.backward()
        assert torch.isfinite(loss)
        opt.step()


@pytest.mark.parametrize("name", ["add", "sub", "mul", "div"])
def test_mixed_dtypes_are_promoted(ME, cuda, name):
    """bf16 self with an fp32 other (and fp32 with fp16): computed in the promoted dtype, the result
    in self's dtype.  Compared with the reference's composition, zeros(self.dtype) + index
    assignment, with the cast to self's dtype written out (torch's index assignment no longer
    casts implicitly)."""
    op = {"add": lambda p, q: p + q, "sub": lambda p, q: p - q, "mul": lambda p, q: p * q,
          "div": lambda p, q: p / q}[name]
    for da, db in ((torch.bfloat16, torch.float32), (torch.float32, torch.float16)):
        a, b = _two(ME, cuda, C=8)
        a = ME.SparseTensor(a.F.detach().to(da).requires_grad_(True),
                            coordinate_map_key=a.coordinate_map_key,
                            coordinate_manager=a.coordinate_manager)
        b = ME.SparseTensor(b.F.detach().to(db).requires_grad_(True),
                            coordinate_map_key=b.coordinate_map_key,
                            coordinate_manager=b.coordinate_manager)
        y = op(a, b)
        assert y.F.dtype == da
        maps = a.coordinate_manager.union_map([a.coordinate_map_key, b.coordinate_map_key],
                                              ME.CoordinateMapKey(4))
        fa = a.F.detach().clone().requires_grad_(True)
        fb = b.F.detach().clone().requires_grad_(True)
        out = torch.zeros(y.F.shape, dtype=da, device=cuda)
        out[maps[0][1]] = fa[maps[0][0]]
        out[maps[1][1]] = op(out[maps[1][1]], fb[maps[1][0]]).to(da)
        assert torch.equal(y.F.detach(), out.detach())
        g = torch.randn(y.F.shape, generator=torch.Generator().manual_seed(4)).to(da).to(cuda)
        y.F.backward(g)
        out.backward(g)
        assert a.F.grad.dtype == da and b.F.grad.dtype == db
        for got, want in ((a.F.grad, fa.grad), (b.F.grad, fb.grad)):
            eps = 2.0 ** -8 if got.dtype == torch.bfloat16 else 2.0 ** -10
            assert ((got.float() - want.float()).abs() <= eps * want.float().abs() + 1e-6).all()
    # MinkowskiUnion: the first input's dtype
    a, b = _two(ME, cuda, C=8)
    bl = ME.SparseTensor(b.F.detach().bfloat16(), coordinate_map_key=b.coordinate_map_key,
                         coordinate_manager=b.coordinate_manager)
    u = ME.MinkowskiUnion()(a, bl)
    assert u.F.dtype == torch.float32
    ref = ME.MinkowskiUnion()(a, ME.SparseTensor(bl.F.float(), coordinate_map_key=b.coordinate_map_key,
                                                 coordinate_manager=b.coordinate_manager))
    assert torch.equal(u.F, ref.F)
