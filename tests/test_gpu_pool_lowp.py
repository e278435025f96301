"""Local pooling (sum / avg / max) in fp32, bf16 and fp16 against the numpy oracle, element by
element.

- The max forward involves no rounding: the output must equal the oracle's bit for bit, and the
  arg-max (`max_index`) must be the oracle's exactly (ascending k, strict '<': the first of equal
  maxima wins).  Inputs are drawn from a few values, so that ties are common.
- An empty window (kernel < stride, or an output coordinate given by the caller with no input in
  reach) holds the lowest finite value of the dtype, as the reference CPU kernel fills it, and
  passes no gradient.
- Sum, avg and the max backward are accumulated in fp32 and rounded once (tests/helpers.py), also
  where windows overlap and one input is the arg-max of many windows."""
import numpy as np
import pytest
import torch

from helpers import assert_one_rounding, random_cloud, unique_cloud
from oracle import oracle_np as O

pytestmark = pytest.mark.gpu

D = 3
DTYPES = {"fp32": torch.float32, "bf16": torch.bfloat16, "fp16": torch.float16}
MODES = {"sum": O.POOL_SUM, "avg": O.POOL_AVG, "max": O.POOL_MAX}


def _layer(ME, mode, k, s):
    cls = {"sum": ME.MinkowskiSumPooling, "avg": ME.MinkowskiAvgPooling,
           "max": ME.MinkowskiMaxPooling}[mode]
    return cls(kernel_size=k, stride=s, dimension=D)


def _features(n, C, mode, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    if mode == "max":       # few distinct values: many ties
        f = torch.randint(-3, 4, (n, C), generator=g).float() * 0.75
    else:
        f = torch.rand(n, C, generator=g) - 0.5
    return f.to(dtype)


def _stride_map_by_cell(in_c, out_c, s):
    """The reference's stride-map shortcut (kernel == stride) as one group per position in the
    stride cell, axis 0 fastest: the order in which this package visits a cell, so that max ties
    resolve alike.  The reference's single group follows its hash map's iteration order, which is
    implementation-defined."""
    (i,), (o,) = O.stride_map(in_c, out_c, [s] * D)
    off = in_c[i, 1:] - out_c[o, 1:]                 # in [0, s) per axis
    cell = sum(off[:, d] * s ** d for d in range(D))
    return [i[cell == c] for c in range(s ** D)], [o[cell == c] for c in range(s ** D)]


def _run_and_check(ME, cuda, mode, k, s, C, dtype, coords, out_coords=None, seed=0):
    feats = _features(len(coords), C, mode, dtype, seed)
    x = ME.SparseTensor(feats, coords, device=cuda, requires_grad=True)
    y = _layer(ME, mode, k, s)(x, coordinates=out_coords) if out_coords is not None \
        else _layer(ME, mode, k, s)(x)
    aux = y.F.grad_fn.num_nonzero
    g = torch.Generator().manual_seed(seed + 1)
    gout = (torch.rand(y.F.shape, generator=g) - 0.5).to(dtype)
    y.F.backward(gout.to(cuda))

    in_c, out_c = x.C.cpu().numpy(), y.C.cpu().numpy()
    if k == s and out_coords is None:
        im, om = _stride_map_by_cell(in_c, out_c, s)
    else:
        im, om = O.kernel_map(in_c, out_c, O.region_offsets(O.HYPER_CUBE, [k] * D, [1] * D, [1] * D))
    n_in, n_out = len(in_c), len(out_c)
    cnt = np.zeros(n_out)
    for o in om:
        np.add.at(cnt, o, 1)
    empty = torch.as_tensor(cnt == 0, device=cuda)
    f64 = feats.double().numpy()
    ref, ref_aux = O.pool_forward(f64, im, om, n_out, MODES[mode])
    ref = torch.as_tensor(ref, device=cuda)
    yF = y.F.detach()
    assert yF.dtype == dtype
    if mode == "max":
        ref[empty] = torch.finfo(dtype).min
        assert bool(torch.isfinite(yF).all()), "an empty max window gave a non-finite value"
        assert torch.equal(yF.double(), ref), "max forward is not exact"
        assert torch.equal(aux.cpu(), torch.as_tensor(ref_aux)), "arg-max differs from the oracle"
    else:
        A, _ = O.pool_forward(np.abs(f64), im, om, n_out, MODES[mode])
        assert_one_rounding(yF, ref, torch.as_tensor(A, device=cuda), f"{mode} forward")
        if mode == "avg":
            assert torch.equal(aux.double().cpu(), torch.as_tensor(ref_aux))
    g64 = gout.double().numpy()
    gi_ref = O.pool_backward(g64, n_in, im, om, MODES[mode], ref_aux)
    gi_A = O.pool_backward(np.abs(g64), n_in, im, om, MODES[mode], ref_aux)
    assert x.F.grad.dtype == dtype
    assert_one_rounding(x.F.grad, torch.as_tensor(gi_ref, device=cuda),
                        torch.as_tensor(gi_A, device=cuda), f"{mode} backward")
    return int(empty.sum())


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("C", [6, 32, 96])
@pytest.mark.parametrize("k,s", [(2, 2), (3, 1), (3, 2), (2, 3), (3, 4)])
@pytest.mark.parametrize("mode", list(MODES))
def test_local_pooling_vs_oracle(ME, cuda, mode, k, s, C, dtype):
    coords = unique_cloud(3000, 9, seed=31 + k * 10 + s, allow_negative=True)
    n_empty = _run_and_check(ME, cuda, mode, k, s, C, DTYPES[dtype], coords, seed=k * 7 + s + C)
    if k < s and k == 2:
        assert n_empty > 0, "expected empty windows with kernel < stride"


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("k,s", [(3, 2), (3, 1), (2, 3)])
def test_local_pooling_onto_given_coordinates(ME, cuda, mode, k, s, dtype):
    """Pooling onto caller-given output coordinates, some with no input in reach."""
    coords = unique_cloud(2500, 10, seed=41, allow_negative=True)
    far = coords[::5].clone()
    far[:, 1:] += 1000
    out = torch.cat([coords[::3], far]).to(cuda)
    n_empty = _run_and_check(ME, cuda, mode, k, s, 32, DTYPES[dtype], coords, out_coords=out,
                             seed=5)
    assert n_empty >= len(far)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
def test_max_pool_backward_bitwise_at_scale(ME, cuda, dtype):
    """k = 3, s = 1 (every input in up to 27 windows), > 500k rows: two backward passes agree bit
    for bit."""
    coords = torch.unique(random_cloud(900_000, 60, seed=3, allow_negative=True), dim=0)
    assert len(coords) >= 500_000
    feats = _features(len(coords), 32, "max", dtype, seed=4).to(cuda)
    x = ME.SparseTensor(feats, coords.to(cuda))
    pool = _layer(ME, "max", 3, 1)
    gout = None
    grads = []
    for _ in range(2):
        f = x.F.detach().clone().requires_grad_(True)
        y = pool(ME.SparseTensor(f, coordinate_map_key=x.coordinate_map_key,
                                 coordinate_manager=x.coordinate_manager))
        if gout is None:
            g = torch.Generator().manual_seed(6)
            gout = (torch.rand(y.F.shape, generator=g) - 0.5).to(dtype).to(cuda)
        y.F.backward(gout)
        grads.append(f.grad)
    assert torch.equal(grads[0], grads[1])
