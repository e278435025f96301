"""The numpy restatement of the TensorField operations (tests/field_oracle.py) against the compiled
reference's fixtures (tests/golden/make_field_fixtures.py), and the host plumbing that needs no GPU."""
import os

import numpy as np
import pytest

import field_oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _load(name):
    return np.load(os.path.join(GOLDEN, name))


@pytest.mark.parametrize("stride", [1, 2])
@pytest.mark.parametrize("mode", [O.SUM, O.AVG, O.SUBSAMPLE, O.MAX])
def test_quantisation_oracle_matches_reference(mode, stride):
    z = _load("ref_field_quantize.npz")
    pts, feats = z["coords"], z["feats"]
    tag = f"{mode}_s{stride}"
    uniq, uidx, inv = O.insert(O.quantize(pts, stride))
    perm = O.canon(uniq)
    assert (uniq[perm] == z[f"{tag}_out_coords"]).all()
    out, _ = O.reduce(feats, inv, len(uniq), mode)
    np.testing.assert_allclose(out[perm], z[f"{tag}_out"], rtol=1e-5, atol=1e-5)
    g = np.empty_like(z[f"{tag}_grad_out"])
    g[perm] = z[f"{tag}_grad_out"]
    grad = O.reduce_backward(g, feats, inv, len(uniq), mode)
    np.testing.assert_allclose(grad, z[f"{tag}_grad_in"], rtol=1e-5, atol=1e-5)
    if mode == O.SUBSAMPLE:
        assert (uidx == np.array([np.nonzero(inv == r)[0][0] for r in range(len(uniq))])).all()


def test_slice_oracle_matches_reference():
    stride = 1
    z = _load("ref_field_slice.npz")
    coords = z[f"s{stride}_coords"]
    inv = O.find(coords, O.quantize(z["coords"], stride))
    assert (inv >= 0).all()
    np.testing.assert_allclose(O.slice_forward(z[f"s{stride}_feats"], inv), z[f"s{stride}_out"],
                               rtol=0, atol=0)
    grad = O.slice_backward(z[f"s{stride}_grad_out"], inv, len(coords))
    np.testing.assert_allclose(grad, z[f"s{stride}_grad_feats"], rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("D", [3, 4])
def test_interpolation_oracle_matches_reference(D):
    z = _load("ref_field_interp.npz")
    coords, feats, q = z[f"d{D}_coords"], z[f"d{D}_feats"], z[f"d{D}_query"]
    rows, w = O.interp_map(q, coords, 2)
    hits = (rows >= 0).sum(1)
    K = 1 << D
    assert ((hits > 0) & (hits < K)).any() and (hits == 0).any()
    np.testing.assert_allclose(O.interp_forward(feats, rows, w), z[f"d{D}_out"], rtol=1e-5,
                               atol=1e-5)
    np.testing.assert_allclose(O.interp_backward(z[f"d{D}_grad_out"], rows, w, len(coords)),
                               z[f"d{D}_grad_feats"], rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("stride", [2, 4])
def test_reference_slice_onto_a_pooled_map_is_not_the_points_voxel(stride):
    """The reference composes the field's stride-1 map with the stride map by indexing the stride
    map's (in, out) pairs, which come in hash-table order, with stride-1 rows
    (MinkowskiTensorField.py:437-441): almost no point receives its own voxel's features.  Here a
    point receives the features of the voxel that holds it at that stride (DESIGN.md §7); the GPU
    tests check that against the restatement."""
    z = _load("ref_field_slice.npz")
    inv = O.find(z[f"s{stride}_coords"], O.quantize(z["coords"], stride))
    assert (inv >= 0).all()
    own = np.all(O.slice_forward(z[f"s{stride}_feats"], inv) == z[f"s{stride}_out"], axis=1)
    assert own.mean() < 0.05
    feats = {tuple(r) for r in z[f"s{stride}_feats"].tolist()}
    assert all(tuple(r) in feats for r in z[f"s{stride}_out"].tolist())


def test_fixture_cases_cover_the_quantisation_range():
    z = _load("ref_field_quantize.npz")
    _, _, inv = O.insert(O.quantize(z["coords"], 1))
    cnt = np.bincount(inv)
    assert cnt.min() == 1 and cnt.max() >= 25
    assert len(np.unique(np.round(z["coords"][:, 0]))) == 3
    assert (z["feats"] > 0).all()    # MAX_POOL: the reference's max pool starts from zero


def test_public_names_and_splat_without_gpu():
    import minkowskiengine_b200 as ME
    for name in ("TensorField", "MinkowskiInterpolation", "MinkowskiInterpolationFunction",
                 "MinkowskiToSparseTensor"):
        assert hasattr(ME, name)
    for name in ("slice", "cat_slice", "interpolate", "features_at_coordinates"):
        assert callable(getattr(ME.SparseTensor, name))
    for name in ("insert_field", "get_coordinate_field", "field_to_sparse_insert_and_map",
                 "field_to_sparse_map", "exists_field_to_sparse", "get_field_to_sparse_map",
                 "field_to_sparse_keys", "interpolation_map_weight"):
        assert callable(getattr(ME.CoordinateManager, name))
        assert callable(getattr(ME.backend.CoordinateMapManagerGPU_c10, name))
    import torch
    with pytest.raises(NotImplementedError, match="SPLAT"):
        ME.TensorField(torch.zeros(1, 1), torch.zeros(1, 4),
                       quantization_mode=ME.SparseTensorQuantizationMode.SPLAT_LINEAR_INTERPOLATION)
    with pytest.raises(RuntimeError, match="CUDA"):
        ME.TensorField(torch.zeros(1, 1), torch.zeros(1, 4))
