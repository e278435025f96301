"""Dense-tensor interop on the GPU: SparseTensor.dense, to_sparse, to_sparse_all, dense_coordinates
and the dense-head example, element-exact against the compiled reference's fixtures
(tests/golden/ref_dense_*.npz, written by tests/golden/make_dense_fixtures.py from the case tables
below), against the torch composition dense() used to be, and against the numpy restatement."""
import numpy as np
import pytest
import torch

import dense_oracle as O
from examples.dense_head import dense_head
from helpers import golden, state_digest

pytestmark = pytest.mark.gpu

C_DENSE = 3
# name -> (D, tensor stride, min_coordinate given, shape given, contract_stride)
DENSE_CASES = {
    "d2_plain": (2, 1, False, False, True),
    "d2_min_shape": (2, 1, True, True, True),
    "d3_plain": (3, 1, False, False, True),
    "d3_min": (3, 1, True, False, True),
    "d3_shape": (3, 1, False, True, True),
    "d3_s2": (3, 2, False, False, True),
    "d3_s2_nocontract": (3, 2, True, False, False),
    "d4_plain": (4, 1, False, False, True),
    "d4_s2_min_shape": (4, 2, True, True, True),
}
# name -> (format, shape of x)
TO_SPARSE_CASES = {"bcxx": ("BCXX", (2, 3, 6, 7)), "bxxxc": ("BXXXC", (2, 4, 5, 6, 3)),
                   "default": (None, (2, 3, 4, 5, 6))}
ALL_SHAPE = (2, 3, 4, 5)
COORD_SHAPE = (2, 3, 4, 5, 2)
HEAD_PARAMS = ("encoder.0.kernel", "encoder.6.kernel", "head.weight")


def dense_case(name):
    """(stride-1 cloud, coordinates at the case's tensor stride, features in sorted-coordinate
    order, min_coordinate or None, shape or None) of a DENSE_CASES entry.  Without a
    min_coordinate the cloud holds the origin, where the reference's grid starts."""
    D, s, use_min, use_shape, contract = DENSE_CASES[name]
    g = np.random.default_rng(sorted(DENSE_CASES).index(name))
    ext = {2: 9, 3: 6, 4: 4}[D] * s
    lo = -ext if use_min else 0
    base = np.concatenate([g.integers(0, 2, (150, 1)), g.integers(lo, ext, (150, D))], 1)
    base = np.unique(np.concatenate([np.zeros((1, D + 1), np.int64), base]), axis=0)
    base = base[g.permutation(len(base))].astype(np.int32)
    coords = np.unique(np.concatenate([base[:, :1], base[:, 1:] // s * s], 1), axis=0)
    feats = g.standard_normal((len(coords), C_DENSE)).astype(np.float32)
    min_c = [lo - s] * D if use_min else None
    shape = None
    if use_shape:
        step = s if contract else 1
        shape = [3, 7] + [int(v) for v in (coords[:, 1:].max(0) - (min_c or [0] * D)[0]) // step + 3]
    return base, coords.astype(np.int32), feats, min_c, shape


def to_sparse_volume(name):
    """A volume with all-zero cells, and one cell whose channels cancel in sum but not in abs-sum."""
    fmt, shape = TO_SPARSE_CASES[name]
    g = np.random.default_rng(50 + sorted(TO_SPARSE_CASES).index(name))
    ch = 1 if fmt is None else fmt.find("C")
    cells = list(shape)
    cells[ch] = 1
    x = g.standard_normal(shape).astype(np.float32) * (g.uniform(size=cells) < 0.3)
    xc = np.moveaxis(x, ch, -1)
    cell = (1,) + (2,) * (x.ndim - 2)
    xc[cell] = 0
    xc[cell][:2] = (1.5, -1.5)
    return x


def head_volume(seed=7, shape=(2, 2, 12, 10, 8)):
    g = np.random.default_rng(seed)
    x = g.standard_normal(shape).astype(np.float32) * (g.uniform(size=(shape[0], 1) + shape[2:]) < 0.3)
    x[0, :, 0, 0, 0] = 1.0        # the grid of MinkowskiToDenseTensor starts at the origin
    return x


def head_step(MEh, net, dev):
    """One forward + backward of the dense-head example -> (volume with its gradient, output)."""
    v = torch.from_numpy(head_volume()).to(dev).requires_grad_()
    out = net(v)
    g = np.random.default_rng(8).standard_normal(tuple(out.shape)).astype(np.float32)
    out.backward(torch.from_numpy(g).to(dev))
    return v, out


def _sorted_rows(st):
    c = st.C.cpu().numpy()
    p = O.canon(c)
    return c[p], st.F.detach().float().cpu().numpy()[p], p


def _old_dense(x, shape=None, min_coordinate=None, contract_stride=True):
    """The torch composition SparseTensor.dense was before it ran on the native kernel."""
    ts = torch.tensor(x.tensor_stride, device=x.device, dtype=torch.int64)
    coords = x.C.long()
    b, xyz = coords[:, 0], coords[:, 1:]
    if min_coordinate is None:
        min_coordinate = xyz.min(0).values
    else:
        min_coordinate = torch.as_tensor(min_coordinate, device=x.device).long().flatten()
    xyz = xyz - min_coordinate
    if contract_stride:
        xyz = xyz // ts
    nb, spatial = int(b.max().item()) + 1, (xyz.max(0).values + 1).tolist()
    if shape is not None:
        nb, spatial = shape[0], list(shape[2:])
    dense = torch.zeros([nb, x.F.size(1)] + spatial, dtype=x.dtype, device=x.device)
    idx = (b,) + tuple(xyz[:, i] for i in range(x.D))
    dense.permute(0, *range(2, 2 + x.D), 1)[idx] = x.F
    return dense, min_coordinate.int(), torch.tensor(x.tensor_stride, dtype=torch.int32)


# ---- the compiled reference's fixtures ---------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("name", list(DENSE_CASES))
def test_dense_matches_reference(ME, cuda, name, dtype):
    D, s, use_min, use_shape, contract = DENSE_CASES[name]
    G = golden(f"ref_dense_{name}.npz")
    _, coords, feats, min_c, shape = dense_case(name)
    assert (coords == G["coords"]).all() and (feats == G["feats"]).all()
    f = torch.from_numpy(feats).to(cuda, dtype).requires_grad_()
    x = ME.SparseTensor(f, torch.from_numpy(coords).to(cuda), tensor_stride=s)
    d, mn, st = x.dense(shape=None if shape is None else torch.Size(shape),
                        min_coordinate=None if min_c is None else torch.IntTensor(min_c),
                        contract_stride=contract)
    want = torch.from_numpy(G["dense"]).to(dtype)
    assert d.dtype == dtype and d.is_contiguous() and tuple(d.shape) == tuple(want.shape)
    assert torch.equal(d.detach().cpu(), want)
    assert mn.dtype == torch.int32 and mn.cpu().tolist() == G["min_coordinate"].tolist()
    assert st.dtype == torch.int32 and st.tolist() == [s] * D
    go = torch.from_numpy(G["grad_out"]).to(dtype)
    d.backward(go.to(cuda))
    assert torch.equal(f.grad.cpu(), torch.from_numpy(G["grad_feats"]).to(dtype))


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("name", list(TO_SPARSE_CASES))
def test_to_sparse_matches_reference(ME, cuda, name, dtype):
    fmt, _ = TO_SPARSE_CASES[name]
    G = golden(f"ref_dense_to_sparse_{name}.npz")
    x = torch.from_numpy(to_sparse_volume(name)).to(cuda, dtype).requires_grad_()
    st = ME.to_sparse(x, fmt)
    # torch.where order, which the insert keeps: rows are distinct
    assert (st.C.cpu().numpy() == G["coords"]).all()
    assert torch.equal(st.F.detach().cpu(), torch.from_numpy(G["feats"]).to(dtype))
    st.F.backward(torch.from_numpy(G["grad_out"]).to(cuda, dtype))
    assert torch.equal(x.grad.cpu(), torch.from_numpy(G["grad_x"]).to(dtype))


def test_to_sparse_all_and_dense_coordinates_match_reference(ME, cuda):
    G = golden("ref_dense_all.npz")
    x = torch.from_numpy(G["x"]).to(cuda).requires_grad_()
    st = ME.to_sparse_all(x)
    assert (st.C.cpu().numpy() == G["coords"]).all()
    assert torch.equal(st.F.detach().cpu(), torch.from_numpy(G["feats"]))
    st.F.backward(torch.from_numpy(G["grad_out"]).to(cuda))
    assert torch.equal(x.grad.cpu(), torch.from_numpy(G["grad_x"]))
    c = ME.dense_coordinates(COORD_SHAPE, cuda)
    assert c.is_cuda and c.dtype == torch.int32
    assert (c.cpu().numpy() == G["dense_coordinates"]).all()
    # cached coordinates, and the module's three branches
    cached = ME.dense_coordinates(x.shape, cuda)
    a = ME.MinkowskiToSparseTensor(coordinates=cached)(x.detach())
    b = ME.MinkowskiToSparseTensor(remove_zeros=False)(x.detach())
    assert torch.equal(a.C, st.C) and torch.equal(b.F, st.F.detach())
    z = x.detach().clone()
    z[:, :, 0] = 0
    kept = ME.MinkowskiToSparseTensor()(z)
    assert len(kept) == z.abs().sum(1).ne(0).sum().item() and (kept.C[:, 1] > 0).all()


def test_dense_head_matches_reference(ME, cuda):
    G = golden("ref_dense_head.npz")
    torch.manual_seed(0)
    net = dense_head(ME)
    assert (state_digest(net) == G["init_digest"]).all(), \
        "seeded initial weights differ from the reference's"
    net = net.to(cuda)
    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False     # the Conv3d head in fp32, as the reference ran it
    try:
        v, out = head_step(ME, net, cuda)
    finally:
        torch.backends.cudnn.allow_tf32 = tf32
    a, b = out.detach().cpu().numpy(), G["out"]
    assert a.shape == b.shape and np.abs(a - b).max() / np.abs(b).max() < 1e-3
    a, b = v.grad.cpu().numpy(), G["grad_volume"]
    assert ((a != 0) <= (head_volume() != 0).any(1, keepdims=True)).all()   # zero cells get none
    assert np.abs(a - b).max() / np.abs(b).max() < 2e-2
    params = dict(net.named_parameters())
    for p in HEAD_PARAMS:
        a, b = params[p].grad.cpu().numpy(), G[f"{p}/grad"]
        assert np.abs(a - b).max() / np.abs(b).max() < 2e-2, p


# ---- the torch composition dense() used to be ---------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("C", [1, 3, 20, 32])
@pytest.mark.parametrize("D,stride", [(2, 1), (3, 1), (3, 2), (3, (1, 2, 4)), (4, 2)])
def test_dense_equals_old_composition(ME, cuda, D, stride, C, dtype):
    g = torch.Generator().manual_seed(D * 100 + C)
    ts = torch.tensor([stride] * D if isinstance(stride, int) else list(stride))
    n = 3000
    xyz = torch.randint(-12, 12, (n, D), generator=g) * ts
    coords = torch.unique(torch.cat([torch.randint(0, 3, (n, 1), generator=g), xyz], 1), dim=0).int()
    coords = coords[torch.randperm(len(coords), generator=g)]
    f = torch.randn(len(coords), C, generator=g).to(cuda, dtype)
    x = ME.SparseTensor(f, coords.to(cuda), tensor_stride=ts.tolist())
    lo = coords[:, 1:].min(0).values
    big = [4, C] + ((coords[:, 1:].max(0).values - lo + ts) // ts + 2).tolist()
    for kw in ({}, {"contract_stride": False}, {"min_coordinate": lo - 2 * ts},
               {"min_coordinate": lo - ts, "shape": torch.Size(big)}):
        got, want = x.dense(**kw), _old_dense(x, **kw)
        assert torch.equal(got[0], want[0]), kw
        assert got[1].dtype == want[1].dtype and torch.equal(got[1], want[1]), kw
        assert got[2].dtype == want[2].dtype and torch.equal(got[2], want[2]), kw


# ---- gradients, cropping, layouts ---------------------------------------------------------------
def _cloud(cuda, n=2000, C=8, dtype=torch.float32, seed=0):
    g = torch.Generator().manual_seed(seed)
    coords = torch.unique(torch.cat([torch.randint(0, 2, (n, 1), generator=g),
                                     torch.randint(-8, 8, (n, 3), generator=g)], 1), dim=0).int()
    return coords.to(cuda), torch.randn(len(coords), C, generator=g).to(cuda, dtype)


@pytest.mark.parametrize("C", [3, 8])
def test_dense_backward_gathers_and_crops(ME, cuda, C):
    coords, f = _cloud(cuda, C=C)
    f.requires_grad_()
    x = ME.SparseTensor(f, coords)
    shape = torch.Size([1, C, 10, 12, 9])          # batch 1 and everything past the box is cropped
    d, _, _ = x.dense(shape=shape, min_coordinate=torch.IntTensor([-4, -5, -3]))
    c = coords.cpu().numpy()
    want = O.rows_to_dense(c, f.detach().cpu().numpy(), list(shape), [-4, -5, -3], [1, 1, 1])
    assert (d.detach().cpu().numpy() == want).all()
    go = torch.randn(d.shape, device=cuda)
    d.backward(go)
    gw = O.dense_to_rows(go.cpu().numpy(), c, [-4, -5, -3], [1, 1, 1])
    assert (f.grad.cpu().numpy() == gw).all()
    inside = (c[:, 0] < 1) & (c[:, 1] >= -4) & (c[:, 1] < 6) & (c[:, 2] >= -5) & (c[:, 2] < 7) & \
        (c[:, 3] >= -3) & (c[:, 3] < 6)
    assert 0 < inside.sum() < len(c) and (f.grad.cpu().numpy()[~inside] == 0).all()
    # a channel-last upstream gradient (what a cudnn head may hand back) is read where it lies
    f.grad = None
    d2, _, _ = x.dense(shape=shape, min_coordinate=torch.IntTensor([-4, -5, -3]))
    d2.backward(go.permute(0, 2, 3, 4, 1).contiguous().permute(0, 4, 1, 2, 3))
    assert (f.grad.cpu().numpy() == gw).all()


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("C", [1, 5, 8])
def test_to_sparse_layouts_and_gradient(ME, cuda, C, dtype):
    g = torch.Generator().manual_seed(C)
    x = (torch.randn(2, C, 9, 6, 7, generator=g) *
         (torch.rand(2, 1, 9, 6, 7, generator=g) < 0.25)).to(cuda, dtype)
    ref = ME.to_sparse(x)
    xn = x.cpu().float().numpy()
    assert (ref.C.cpu().numpy() == O.nonzero_coordinates(xn)).all()
    assert (ref.F.float().cpu().numpy() == O.dense_to_rows(xn, ref.C.cpu().numpy(), [0] * 3, [1] * 3)).all()
    go = torch.randn(ref.F.shape, generator=g).to(cuda, dtype)
    want = torch.from_numpy(O.rows_to_dense(ref.C.cpu().numpy(), go.float().cpu().numpy(),
                                            list(x.shape), [0] * 3, [1] * 3)).to(dtype)
    # the same volume: channel-last, a strided view of a larger buffer, and an offset view
    last = x.permute(0, 2, 3, 4, 1).contiguous()
    buf = torch.zeros(2, C, 9, 12, 9, device=cuda, dtype=dtype)
    view = buf[:, :, :, ::2, 1:8]
    view.copy_(x)
    for t, fmt in ((x, None), (last, "BXXXC"), (view, None), (last.permute(0, 4, 1, 2, 3), None)):
        t = t.detach().requires_grad_()
        st = ME.to_sparse(t, fmt)
        assert torch.equal(st.C, ref.C) and torch.equal(st.F, ref.F)
        st.F.backward(go)
        gx = t.grad if fmt is None else t.grad.permute(0, 4, 1, 2, 3)
        assert torch.equal(gx.cpu(), want)


def test_dense_into_views_and_64_bit_offsets(ME, cuda):
    """Strides far above 2^31 elements over a small allocation: a [2, C, 3, 2, 2] view whose batch
    stride is 2^31 + 8 elements (expanded axes make the span without the memory)."""
    import minkowskiengine_b200.dense as MD
    C = 4
    coords, f = _cloud(cuda, C=C)
    x = ME.SparseTensor(f, coords)
    cmap = x.coordinate_manager._manager._get(x.coordinate_map_key)
    # channel-last target and a strided channel-first target give the contiguous result
    want = x.dense(shape=torch.Size([2, C, 16, 16, 16]), min_coordinate=torch.IntTensor([-8] * 3))[0]
    last = torch.empty(2, 16, 16, 16, C, device=cuda).permute(0, 4, 1, 2, 3)
    MD.rows_to_dense(f, cmap, last, 1, [-8] * 3)
    assert torch.equal(last, want)
    buf = torch.full((2, C, 16, 32, 17), 7.0, device=cuda)
    MD.rows_to_dense(f, cmap, buf[:, :, :, ::2, :16], 1, [-8] * 3)
    assert torch.equal(buf[:, :, :, ::2, :16], want) and (buf[:, :, :, 1::2] == 7).all()
    # 64-bit offsets: batch 1 of the view lies 2^31 + 8 elements after batch 0 (4 GiB of fp16)
    big = 2 ** 31 + 8
    if torch.cuda.mem_get_info()[0] < 12 * 2 ** 30:
        pytest.skip("not enough free memory beside other work for the 2^31-element view")
    h = torch.zeros(big + 4096, device=cuda, dtype=torch.float16)
    hv = h.as_strided((2, 3, 2, 2, 2), (big, 1, 256, 32, 4))
    hv.copy_(torch.randint(1, 100, (2, 3, 2, 2, 2), device=cuda).half())
    st = ME.to_sparse(hv)
    assert len(st) == 16 and torch.equal(st.F, hv.permute(0, 2, 3, 4, 1).reshape(-1, 3))
    h.zero_()
    MD.rows_to_dense(st.F, st.coordinate_manager._manager._get(st.coordinate_map_key), hv, 1)
    assert torch.equal(hv.permute(0, 2, 3, 4, 1).reshape(-1, 3), st.F)
    assert torch.count_nonzero(h).item() == 48


def test_round_trip_empty_single_and_errors(ME, cuda):
    coords, f = _cloud(cuda, C=6)
    f[::5] = 0                                     # all-zero rows do not come back
    x = ME.SparseTensor(f, coords)
    d, mn, _ = x.dense()
    back = ME.to_sparse(d)
    keep = f.abs().sum(1) != 0
    c = torch.cat([coords[keep][:, :1], coords[keep][:, 1:] - mn], 1).cpu().numpy()
    p = O.canon(c)
    bc, bf, _ = _sorted_rows(back)
    assert (bc == c[p]).all() and (bf == f[keep].cpu().numpy()[p]).all()
    # NaN counts as non-zero, -0.0 does not
    z = torch.zeros(1, 2, 3, 3, device=cuda)
    z[0, 0, 1, 1], z[0, 1, 2, 0] = float("nan"), -0.0
    assert ME.to_sparse(z).C.tolist() == [[0, 1, 1]]
    assert len(ME.to_sparse(torch.zeros(1, 2, 3, 3, device=cuda))) == 0
    # a single voxel; an empty tensor
    one = ME.SparseTensor(torch.ones(1, 2, device=cuda), torch.tensor([[1, -3, 5]], device=cuda).int())
    d, mn, _ = one.dense()
    assert tuple(d.shape) == (2, 2, 1, 1) and d[1].eq(1).all() and d[0].eq(0).all()
    assert mn.tolist() == [-3, 5]
    empty = ME.SparseTensor(torch.zeros(0, 2, device=cuda), torch.zeros(0, 3, device=cuda).int())
    d, mn, _ = empty.dense(shape=torch.Size([2, 9, 4, 4]))
    assert tuple(d.shape) == (2, 2, 4, 4) and d.eq(0).all() and mn.tolist() == [0, 0]
    with pytest.raises(AssertionError, match="shape is required to densify an empty tensor"):
        empty.dense()
    s2 = ME.SparseTensor(torch.ones(1, 2, device=cuda), torch.tensor([[0, 2, 4]], device=cuda).int(),
                         tensor_stride=2)
    with pytest.raises(AssertionError, match="must be divisible by the tensor stride"):
        s2.dense(min_coordinate=torch.IntTensor([1, 0]))
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        ME.to_sparse(torch.ones(1, 2, 3, 3))
    with pytest.raises(ME._lib.BackendError, match="unsupported feature dtype"):
        ME.to_sparse(torch.ones(1, 2, 3, 3, device=cuda, dtype=torch.float64))
    assert ME.MinkowskiToDenseTensor(torch.Size([1, 2, 4, 4]))(s2).shape == (1, 2, 4, 4)
