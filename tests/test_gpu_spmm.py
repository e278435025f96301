"""ME.spmm, spmm_average, MinkowskiSPMMFunction, MinkowskiSPMMAverageFunction and
MinkowskiDirectMaxPoolingFunction on the GPU: against the compiled reference's fixtures (fp32),
element by element against the float64 restatement (tests/spmm_oracle.py) in fp32 / bf16 / fp16,
the adjoint identity of the autograd functions, bit-identical repeats on the native library, and
the errors."""
import os

import numpy as np
import pytest
import torch

import spmm_oracle as O
from helpers import assert_one_rounding

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
DTYPES = [torch.float32, torch.bfloat16, torch.float16]


def _load(name):
    return np.load(os.path.join(GOLDEN, name))


def _t(a, dev, dtype=None):
    t = torch.from_numpy(np.asarray(a)).to(dev)
    return t if dtype is None else t.to(dtype)


def _coo(P, n_rows, n_cols, seed, dev, itype=torch.int32):
    """Unsorted entries with repeated pairs, empty rows (the last two) and an unused column 0."""
    g = torch.Generator().manual_seed(seed)
    rows = torch.randint(0, max(n_rows - 2, 1), (P,), generator=g)
    cols = torch.randint(1 if n_cols > 1 else 0, n_cols, (P,), generator=g)
    k = P // 8
    if k:
        rows[-k:], cols[-k:] = rows[:k].clone(), cols[:k].clone()
    perm = torch.randperm(P, generator=g)
    return rows[perm].to(itype).to(dev), cols[perm].to(itype).to(dev)


def _feats(n, C, seed, dev, dtype):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(n, C, generator=g) * 2 - 1).to(dtype).to(dev)


# ---- against the reference's fixtures (fp32) ------------------------------------------------------
@pytest.mark.parametrize("name", ["small", "cloud"])
def test_spmm_matches_reference(ME, cuda, name):
    z = _load(f"ref_spmm_{name}.npz")
    n_rows, n_cols = (int(v) for v in z["shape"])
    r, c, v = _t(z["rows"], cuda), _t(z["cols"], cuda), _t(z["vals"], cuda)
    mat = _t(z["mat"], cuda).requires_grad_()
    size = torch.Size([n_rows, n_cols])
    out = ME.MinkowskiSPMMFunction.apply(r, c, v, size, mat)
    np.testing.assert_allclose(out.detach().cpu().numpy(), z["out"], rtol=1e-5, atol=1e-5)
    out.backward(_t(z["grad_out"], cuda))
    np.testing.assert_allclose(mat.grad.cpu().numpy(), z["grad"], rtol=1e-5, atol=1e-5)
    mat.grad = None
    avg, coo, vals = ME.spmm_average(r, c, size, mat.detach())
    np.testing.assert_allclose(avg.cpu().numpy(), z["avg"], rtol=1e-5, atol=1e-5)
    ref_coo, _ = O.average_coo(z["rows"], z["cols"], n_rows)
    assert coo.dtype == torch.int64 and (coo.cpu() == ref_coo).all()   # stably sorted by row
    np.testing.assert_allclose(vals.cpu().numpy(), z["avg_vals"], rtol=1e-7)
    out = ME.MinkowskiSPMMAverageFunction.apply(r, c, size, mat)
    out.backward(_t(z["grad_out"], cuda))
    np.testing.assert_allclose(mat.grad.cpu().numpy(), z["avg_grad"], rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("name", ["small", "cloud"])
def test_direct_max_matches_reference(ME, cuda, name):
    z = _load(f"ref_direct_max_{name}.npz")
    n_out = int(z["n_out"])
    im, om = _t(z["in_map"], cuda), _t(z["out_map"], cuda)
    x = _t(z["feats"], cuda)
    out, mask = ME.backend.direct_max_pool_fw(im, om, x, n_out)
    assert (out.cpu().numpy() == z["out"]).all()
    assert mask.dtype == torch.int32 and (mask.cpu().numpy() == z["mask"]).all()
    xg = x.clone().requires_grad_()
    y = ME.MinkowskiDirectMaxPoolingFunction.apply(im, om, xg, n_out)
    y.backward(_t(z["grad_out"], cuda))
    np.testing.assert_allclose(xg.grad.cpu().numpy(), z["grad"], rtol=1e-5, atol=1e-5)
    # int64 maps give an int64 mask with the same values
    _, mask64 = ME.backend.direct_max_pool_fw(im.long(), om.long(), x, n_out)
    assert mask64.dtype == torch.int64 and (mask64.cpu().numpy() == z["mask"]).all()


# ---- against float64, element by element ----------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("C", [1, 3, 7, 8, 64])
@pytest.mark.parametrize("itype", [torch.int32, torch.int64])
def test_spmm_float64(ME, cuda, dtype, C, itype):
    n_rows, n_cols, P = 300, 200, 2500
    r, c = _coo(P, n_rows, n_cols, 10 + C, cuda, itype)
    vals = _feats(P, 1, 20 + C, cuda, dtype).view(-1)
    mat = _feats(n_cols, C, 30 + C, cuda, dtype).requires_grad_()
    size = torch.Size([n_rows, n_cols])
    out = ME.MinkowskiSPMMFunction.apply(r, c, vals, size, mat)
    assert out.dtype == dtype and out.shape == (n_rows, C)
    ref, A = O.spmm(r, c, vals, n_rows, mat.detach())
    assert_one_rounding(out.detach(), ref, A, f"spmm {dtype} C={C}")
    assert (out[-2:] == 0).all()
    g = _feats(n_rows, C, 40 + C, cuda, dtype)
    out.backward(g)
    ref, A = O.spmm(c, r, vals, n_cols, g)
    assert_one_rounding(mat.grad, ref, A, f"spmm grad {dtype} C={C}")
    # the average and its backward
    mat.grad = None
    avg = ME.MinkowskiSPMMAverageFunction.apply(r, c, size, mat)
    ref, A = O.spmm_average(r, c, n_rows, mat.detach())
    assert_one_rounding(avg.detach(), ref, A, f"spmm_average {dtype} C={C}")
    avg.backward(g)
    coo, w = O.average_coo(r.cpu(), c.cpu(), n_rows)
    w = w.to(dtype).to(cuda)                      # the 1 / count values in mat's dtype
    ref, A = O.spmm(coo[1], coo[0], w, n_cols, g)
    assert_one_rounding(mat.grad, ref, A, f"spmm_average grad {dtype} C={C}")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("C", [1, 3, 7, 8, 64])
@pytest.mark.parametrize("itype", [torch.int32, torch.int64])
def test_direct_max_float64(ME, cuda, dtype, C, itype):
    n_in, n_out, P = 500, 300, 3000
    out_map, in_map = _coo(P, n_out, n_in, 50 + C, cuda, itype)
    g = torch.Generator().manual_seed(60 + C)
    x = ((torch.randint(-8, 8, (n_in, C), generator=g).float()) / 4).to(dtype).to(cuda)  # ties
    x[: n_in // 4] = -x[: n_in // 4].abs() - 1                 # all-negative inputs
    x = x.requires_grad_()
    y = ME.MinkowskiDirectMaxPoolingFunction.apply(in_map, out_map, x, n_out)
    ref, ref_mask = O.direct_max(in_map, out_map, x.detach(), n_out)
    assert y.dtype == dtype and (y.detach().double() == ref).all()
    _, mask = ME.backend.direct_max_pool_fw(in_map, out_map, x.detach(), n_out)
    assert mask.dtype == itype and (mask.long() == ref_mask).all()
    assert (mask[-2:] == -1).all() and (y[-2:] == 0).all()    # rows without pairs
    gout = _feats(n_out, C, 70 + C, cuda, dtype)
    y.backward(gout)
    ref = O.direct_max_backward(gout, ref_mask, n_in)
    A = O.direct_max_backward(gout.abs(), ref_mask, n_in)
    assert_one_rounding(x.grad, ref, A, f"direct max grad {dtype} C={C}")
    # the reference's entry point, from the flat mask alone
    gi = ME.backend.direct_max_pool_bw(gout, mask, n_in)
    assert_one_rounding(gi, ref, A, f"direct_max_pool_bw {dtype} C={C}")


def test_direct_max_semantics(ME, cuda):
    """All-negative channels give the true maximum, the first pair wins a tie, a row without pairs
    is 0 with mask -1 and sends nothing, a repeated pair counts once."""
    x = torch.tensor([[-3.0, 1.0], [-1.0, 1.0], [-2.0, 0.5]], device=cuda, requires_grad=True)
    im = torch.tensor([0, 1, 1, 2], device=cuda)
    om = torch.tensor([0, 0, 0, 2], device=cuda)
    out, mask = ME.backend.direct_max_pool_fw(im, om, x.detach(), 3)
    assert out.tolist() == [[-1.0, 1.0], [0.0, 0.0], [-2.0, 0.5]]
    assert mask.tolist() == [[2, 1], [-1, -1], [4, 5]] and mask.dtype == torch.int64
    y = ME.MinkowskiDirectMaxPoolingFunction.apply(im, om, x, 3)
    y.backward(torch.ones(3, 2, device=cuda))
    assert x.grad.tolist() == [[0.0, 1.0], [1.0, 0.0], [1.0, 1.0]]


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_points_to_voxels_large(ME, cuda, dtype):
    """8 clouds x 250k points onto voxels: the sizes profiles/spmm_bench.py times."""
    n, C = 8 * 250_000, 32
    g = torch.Generator().manual_seed(5)
    n_vox = 600_000
    vox = torch.randint(0, n_vox, (n,), generator=g).to(cuda)
    pts = torch.arange(n, device=cuda)
    x = _feats(n, C, 6, cuda, dtype)
    w = _feats(n, 1, 7, cuda, dtype).view(-1)
    out = ME.spmm(vox, pts, w, torch.Size([n_vox, n]), x)
    ref, A = O.spmm(vox, pts, w, n_vox, x)
    assert_one_rounding(out, ref, A, "spmm 8x250k")
    avg, _, _ = ME.spmm_average(vox, pts, torch.Size([n_vox, n]), x)
    ref, A = O.spmm_average(vox, pts, n_vox, x)
    assert_one_rounding(avg, ref, A, "spmm_average 8x250k")
    y, mask = ME.backend.direct_max_pool_fw(pts, vox, x, n_vox)
    ref, ref_mask = O.direct_max(pts, vox, x, n_vox)
    assert (y.double() == ref).all() and (mask.long() == ref_mask).all()
    gout = _feats(n_vox, C, 8, cuda, dtype)
    gi = ME.backend.direct_max_pool_bw(gout, mask, n)
    assert (gi.double() == O.direct_max_backward(gout, ref_mask, n)).all()   # one term each


# ---- adjoint identity ---------------------------------------------------------------------------
def test_adjoint_identities(ME, cuda):
    """<spmm(A, x), g> = <x, spmm(A^T, g)> through the autograd functions, in float64 arithmetic
    on the fp32 results."""
    n_rows, n_cols, P, C = 400, 300, 5000, 16
    r, c = _coo(P, n_rows, n_cols, 80, cuda)
    vals = _feats(P, 1, 81, cuda, torch.float32).view(-1)
    x = _feats(n_cols, C, 82, cuda, torch.float32).requires_grad_()
    g = _feats(n_rows, C, 83, cuda, torch.float32)
    size = torch.Size([n_rows, n_cols])
    for fn in (lambda m: ME.MinkowskiSPMMFunction.apply(r, c, vals, size, m),
               lambda m: ME.MinkowskiSPMMAverageFunction.apply(r, c, size, m)):
        x.grad = None
        y = fn(x)
        y.backward(g)
        lhs = (y.detach().double() * g.double()).sum()
        rhs = (x.detach().double() * x.grad.double()).sum()
        scale = (y.detach().double().abs() * g.double().abs()).sum()
        assert abs(float(lhs - rhs)) <= 2 ** -20 * float(scale), (float(lhs), float(rhs))


# ---- native path, repeats --------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
def test_bit_identical_on_native_path(ME, cuda, dtype):
    from minkowskiengine_b200 import _lib
    n_rows, n_cols, P, C = 2000, 3000, 40_000, 24
    r, c = _coo(P, n_rows, n_cols, 90, cuda)
    vals = _feats(P, 1, 91, cuda, dtype).view(-1)
    x = _feats(n_cols, C, 92, cuda, dtype)
    g = _feats(n_rows, C, 93, cuda, dtype)
    size = torch.Size([n_rows, n_cols])

    def run():
        n0 = _lib.launch_count()
        res = []
        for fn in (lambda m: ME.MinkowskiSPMMFunction.apply(r, c, vals, size, m),
                   lambda m: ME.MinkowskiSPMMAverageFunction.apply(r, c, size, m),
                   lambda m: ME.MinkowskiDirectMaxPoolingFunction.apply(c, r, m, n_rows)):
            m = x.clone().requires_grad_()
            n1 = _lib.launch_count()
            y = fn(m)
            n2 = _lib.launch_count()
            y.backward(g)
            assert n2 > n1 and _lib.launch_count() > n2, "forward and backward run on the library"
            res += [y.detach().clone(), m.grad.clone()]
        assert _lib.launch_count() > n0
        return res

    a, b = run(), run()
    for u, v in zip(a, b):
        assert torch.equal(u.view(torch.uint8) if u.dtype != torch.float32 else u.view(torch.int32),
                           v.view(torch.uint8) if v.dtype != torch.float32 else v.view(torch.int32))


# ---- empty cases and errors ----------------------------------------------------------------------
def test_empty_cases(ME, cuda):
    from minkowskiengine_b200 import _lib
    e = torch.zeros(0, dtype=torch.int32, device=cuda)
    x = _feats(5, 4, 1, cuda, torch.float32)
    n0 = _lib.launch_count()
    out = ME.spmm(e, e, torch.zeros(0, device=cuda), torch.Size([3, 5]), x)
    assert out.shape == (3, 4) and (out == 0).all()
    avg, coo, vals = ME.spmm_average(e, e, torch.Size([3, 5]), x)
    assert (avg == 0).all() and coo.shape == (2, 0) and vals.numel() == 0
    y, mask = ME.backend.direct_max_pool_fw(e, e, x, 3)
    assert (y == 0).all() and (mask == -1).all()
    assert ME.spmm(e, e, torch.zeros(0, device=cuda), torch.Size([0, 5]), x).shape == (0, 4)
    assert _lib.launch_count() == n0
    # C = 0 checks the indices (one launch) and reduces nothing
    r = torch.tensor([0, 1], device=cuda)
    assert ME.spmm(r, r, torch.ones(2, device=cuda), torch.Size([2, 5]),
                   x[:, :0]).shape == (2, 0)
    assert _lib.launch_count() == n0 + 1


def test_errors(ME, cuda):
    r = torch.tensor([0, 1, 2], device=cuda)
    v = torch.ones(3, device=cuda)
    x = torch.ones(4, 2, device=cuda)
    s = torch.Size([3, 4])
    with pytest.raises(AssertionError):
        ME.spmm(r, r[:2], v, s, x)                                   # lengths
    with pytest.raises(AssertionError):
        ME.spmm(r, r, v[:2], s, x)
    with pytest.raises(AssertionError):
        ME.spmm(r, r, v.half(), s, x)                                # vals / mat dtype
    with pytest.raises(AssertionError):
        ME.spmm(r, r, v.cpu(), s, x)                                 # devices
    with pytest.raises(AssertionError):
        ME.spmm(r.cpu(), r, v, s, x)
    with pytest.raises(RuntimeError):
        ME.spmm(r, r, v.double(), s, x.double())                     # fp64
    with pytest.raises(RuntimeError, match="column"):
        ME.spmm(r, torch.tensor([0, 4, 1], device=cuda), v, s, x)    # cols out of range
    with pytest.raises(RuntimeError, match="column"):
        ME.spmm(r, torch.tensor([0, -1, 1], device=cuda), v, s, x)
    with pytest.raises(RuntimeError, match="column"):
        ME.spmm(r, torch.tensor([0, 2 ** 32, 1], device=cuda), v, s, x)   # would wrap to 0
    with pytest.raises(RuntimeError, match="row"):
        ME.spmm(torch.tensor([0, 3, 1], device=cuda), r, v, s, x)    # rows out of range
    with pytest.raises(RuntimeError, match="row"):
        ME.spmm_average(torch.tensor([-1, 0, 1], device=cuda), r, s, x)
    xm = torch.ones(3, 2, device=cuda)
    with pytest.raises(RuntimeError, match="column"):
        ME.MinkowskiDirectMaxPoolingFunction.apply(torch.tensor([0, 3], device=cuda),
                                                   torch.tensor([0, 1], device=cuda), xm, 2)
    with pytest.raises(RuntimeError, match="row"):
        ME.MinkowskiDirectMaxPoolingFunction.apply(torch.tensor([0, 1], device=cuda),
                                                   torch.tensor([0, 2], device=cuda), xm, 2)
    with pytest.raises(RuntimeError):
        ME.MinkowskiDirectMaxPoolingFunction.apply(r, r, xm.cpu(), 3)
    with pytest.raises(RuntimeError):
        ME.MinkowskiDirectMaxPoolingFunction.apply(r, r, xm.double(), 3)
    # an int32 flat mask cannot hold n_in * C - 1 = 2^31 + 31: a [2^26 + 1, 32] input (expanded,
    # no storage; the check comes before any copy)
    big = torch.zeros(1, 32, device=cuda).expand(2 ** 26 + 1, 32)
    one = torch.tensor([0], dtype=torch.int32, device=cuda)
    with pytest.raises(RuntimeError, match="flat mask"):
        ME.backend.direct_max_pool_fw(one, one, big, 1)
    with pytest.raises(RuntimeError, match="flat mask"):
        ME.backend.direct_max_pool_bw(torch.ones(1, 32, device=cuda),
                                      torch.zeros(1, 32, dtype=torch.int32, device=cuda), 2 ** 26)


# ---- the caller's index tensors ---------------------------------------------------------------------
def test_int64_indices_not_written(ME, cuda):
    """int64 (and float) indices are converted out of place: values outside int32 stay in the
    caller's tensor and its autograd version does not move."""
    r = torch.tensor([0, 2, 1, 2], device=cuda)
    c = torch.tensor([1, 0, 1, 2], device=cuda)
    bad = torch.tensor([0, 2 ** 40, 1, 2], device=cuda)
    neg = torch.tensor([0, -2 ** 40, 1, 2], device=cuda)
    v = torch.ones(4, device=cuda)
    x = _feats(3, 4, 1, cuda, torch.float32)
    size = torch.Size([3, 3])
    tensors = (r, c, bad, neg)
    before = [(t.clone(), t._version) for t in tensors]
    ME.spmm(r, c, v, size, x)
    ME.spmm_average(r, c, size, x)
    _, mask = ME.backend.direct_max_pool_fw(c, r, x, 3)
    for t in (bad, neg):
        with pytest.raises(RuntimeError, match="column"):
            ME.spmm(r, t, v, size, x)
        with pytest.raises(RuntimeError, match="row"):
            ME.spmm(t, c, v, size, x)
    m0, v0 = mask.clone(), mask._version
    ME.backend.direct_max_pool_bw(torch.ones(3, 4, device=cuda), mask, 3)
    assert torch.equal(mask, m0) and mask._version == v0
    for t, (t0, ver) in zip(tensors, before):
        assert torch.equal(t, t0) and t._version == ver


def test_index_reused_by_autograd(ME, cuda):
    """An int64 index a graph saved earlier (x[inv]) can go to spmm without breaking backward."""
    inv = torch.tensor([0, 2, 1, 2, 0], device=cuda)
    pts = torch.arange(5, device=cuda)
    x = _feats(3, 4, 2, cuda, torch.float32).requires_grad_()
    y = x[inv]                                   # saves inv for its backward
    z = ME.MinkowskiSPMMFunction.apply(inv, pts, torch.ones(5, device=cuda), torch.Size([3, 5]), y)
    z.sum().backward()
    ref, _ = O.spmm(pts, inv, torch.ones(5), 5, torch.ones(3, 4, device=cuda))
    ref_x, _ = O.spmm(inv, pts, torch.ones(5), 3, ref)
    assert torch.equal(x.grad.double(), ref_x)


@pytest.mark.parametrize("itype", [torch.int32, torch.int64])
def test_second_backward_with_retain_graph(ME, cuda, itype):
    r, c = _coo(400, 60, 50, 3, cuda, itype)
    vals = _feats(400, 1, 4, cuda, torch.float32).view(-1)
    x = _feats(50, 8, 5, cuda, torch.float32).requires_grad_()
    g = _feats(60, 8, 6, cuda, torch.float32)
    size = torch.Size([60, 50])
    for fn in (lambda m: ME.MinkowskiSPMMFunction.apply(r, c, vals, size, m),
               lambda m: ME.MinkowskiSPMMAverageFunction.apply(r, c, size, m),
               lambda m: ME.MinkowskiDirectMaxPoolingFunction.apply(c, r, m, 60)):
        x.grad = None
        y = fn(x)
        y.backward(g, retain_graph=True)
        first = x.grad.clone()
        y.backward(g)
        assert torch.equal(x.grad, 2 * first)
