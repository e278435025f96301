"""COO sparse-times-dense products and direct max pooling without a GPU: the float64 restatement
(tests/spmm_oracle.py) pinned to the compiled reference's fixtures, and the public names."""
import os

import numpy as np
import pytest
import torch

import spmm_oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _load(name):
    return np.load(os.path.join(GOLDEN, name))


@pytest.mark.parametrize("name", ["small", "cloud"])
def test_spmm_oracle_matches_reference(name):
    z = _load(f"ref_spmm_{name}.npz")
    n_rows, n_cols = (int(v) for v in z["shape"])
    out, _ = O.spmm(z["rows"], z["cols"], z["vals"], n_rows, z["mat"])
    np.testing.assert_allclose(out.numpy(), z["out"], rtol=1e-5, atol=1e-5)
    grad, _ = O.spmm(z["cols"], z["rows"], z["vals"], n_cols, z["grad_out"])
    np.testing.assert_allclose(grad.numpy(), z["grad"], rtol=1e-5, atol=1e-5)
    avg, _ = O.spmm_average(z["rows"], z["cols"], n_rows, z["mat"])
    np.testing.assert_allclose(avg.numpy(), z["avg"], rtol=1e-5, atol=1e-5)
    coo, vals = O.average_coo(z["rows"], z["cols"], n_rows)
    # the reference sorts by row only (not stably): compare each row's entries as a multiset
    ref = z["avg_coo"]
    assert (coo[0].numpy() == ref[0]).all()
    key = lambda c: np.lexsort((c[1], c[0]))                                     # noqa: E731
    assert (coo.numpy()[:, key(coo.numpy())] == ref[:, key(ref)]).all()
    np.testing.assert_allclose(vals.numpy(), z["avg_vals"], rtol=1e-7)
    agrad, _ = O.spmm(coo[1], coo[0], vals, n_cols, z["grad_out"])
    np.testing.assert_allclose(agrad.numpy(), z["avg_grad"], rtol=1e-5, atol=1e-5)
    # the fixture covers duplicates, rows without entries and an unused column
    pairs = set(zip(z["rows"].tolist(), z["cols"].tolist()))
    assert len(pairs) < len(z["rows"])
    assert (np.bincount(z["rows"], minlength=n_rows) == 0).any()
    assert (np.bincount(z["cols"], minlength=n_cols) == 0).any()


@pytest.mark.parametrize("name", ["small", "cloud"])
def test_direct_max_oracle_matches_reference(name):
    z = _load(f"ref_direct_max_{name}.npz")
    n_out, n_in = int(z["n_out"]), len(z["feats"])
    out, mask = O.direct_max(z["in_map"], z["out_map"], z["feats"], n_out)
    assert (out.numpy() == z["out"]).all()
    assert (mask.numpy() == z["mask"]).all()
    grad = O.direct_max_backward(z["grad_out"], mask, n_in)
    np.testing.assert_allclose(grad.numpy(), z["grad"], rtol=1e-5, atol=1e-5)
    pairs = set(zip(z["in_map"].tolist(), z["out_map"].tolist()))
    assert len(pairs) < len(z["in_map"])                              # repeated pairs
    assert (np.bincount(z["in_map"], minlength=n_in) == 0).any()      # inputs no pair reads


def test_direct_max_oracle_semantics():
    """All-negative channels give the true maximum, the first pair wins a tie, an output row
    without pairs is 0 with mask -1, and a repeated pair sends its gradient once."""
    x = torch.tensor([[-3.0, 1.0], [-1.0, 1.0], [-2.0, 0.5]])
    in_map, out_map = [0, 1, 1, 2], [0, 0, 0, 2]
    out, mask = O.direct_max(in_map, out_map, x, 3)
    assert out.tolist() == [[-1.0, 1.0], [0.0, 0.0], [-2.0, 0.5]]
    assert mask.tolist() == [[2, 1], [-1, -1], [4, 5]]
    g = O.direct_max_backward(torch.ones(3, 2), mask, 3)
    assert g.tolist() == [[0.0, 1.0], [1.0, 0.0], [1.0, 1.0]]


def test_public_names(ME):
    for name in ("spmm", "spmm_average", "MinkowskiSPMMFunction", "MinkowskiSPMMAverageFunction",
                 "MinkowskiDirectMaxPoolingFunction"):
        assert hasattr(ME, name), name
    for name in ("coo_spmm_int32", "coo_spmm_average_int32", "direct_max_pool_fw",
                 "direct_max_pool_bw"):
        assert callable(getattr(ME.backend, name)), name


def test_cpu_tensors_raise(ME):
    r = torch.tensor([0, 1])
    v = torch.ones(2)
    with pytest.raises(AssertionError):
        ME.spmm(r, r, v, torch.Size([2, 2]), torch.ones(2, 3))
    with pytest.raises(RuntimeError):
        ME.MinkowskiDirectMaxPoolingFunction.apply(r, r, torch.ones(2, 3), 2)
