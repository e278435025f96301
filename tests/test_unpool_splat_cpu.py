"""Unpooling and splatting without a GPU: the float64 restatement (tests/unpool_splat_oracle.py)
pinned to the compiled reference's fixtures, the public names, and the unpooling's sum."""
import os

import numpy as np
import pytest

import unpool_splat_oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
UNPOOL = {"k2s2_d3": (2, 2), "k3s2_d2": (3, 2), "k2s2_expand": (2, 2), "k2s2_d4": (2, 2)}


def _load(name):
    return np.load(os.path.join(GOLDEN, name))


@pytest.mark.parametrize("name", list(UNPOOL))
def test_unpool_oracle_matches_reference(name):
    k, s = UNPOOL[name]
    z = _load(f"ref_unpool_{name}.npz")
    out_c = z["out_coords"]
    if name.endswith("expand"):
        assert (O.expand_coords(z["in_coords"], 2, k, s) == out_c).all()
    else:
        # without expansion the output is the existing stride-1 map
        assert (z["coords"][O.canon(z["coords"])] == out_c).all()
    pairs = O.unpool_pairs(z["in_coords"], 2, out_c, k, s)
    np.testing.assert_allclose(O.unpool_forward(z["in_feats"], pairs, len(out_c)), z["out"],
                               rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(O.unpool_backward(z["grad_out"], pairs, len(z["in_coords"])),
                               z["grad_in"], rtol=1e-6, atol=1e-6)
    if k == s:   # the stride map: every fine row has at most one parent
        assert len(np.unique(pairs[1])) == len(pairs[1])


def _check_splat(z, tag):
    coords, rows, w = O.splat_map(z[f"{tag}coords"])
    perm = O.canon(coords)
    assert (coords[perm] == z[f"{tag}out_coords"]).all()
    rank = np.empty_like(perm)
    rank[perm] = np.arange(len(perm))
    out = O.splat_forward(z[f"{tag}feats"], rows, w, len(coords))
    np.testing.assert_allclose(out[perm], z[f"{tag}out"], rtol=1e-5, atol=1e-6)
    g = z[f"{tag}grad_out"][rank]                 # canonical -> first-occurrence row order
    np.testing.assert_allclose(O.splat_backward(g, rows, w), z[f"{tag}grad_in"], rtol=1e-5,
                               atol=1e-6)
    return coords, rows, w, perm, rank


@pytest.mark.parametrize("tag", ["small_", "small2_"])
def test_splat_oracle_matches_reference_small(tag):
    z = _load("ref_splat_small.npz")
    coords, _, w, _, _ = _check_splat(z, tag)
    D = coords.shape[1] - 1
    assert len(coords) == 2 * 2 ** D - 1   # the two cells share one corner
    assert np.allclose(w.sum(1), 1.0)


def test_splat_oracle_matches_reference_cloud():
    z = _load("ref_splat_cloud.npz")
    coords, rows, w, perm, rank = _check_splat(z, "")
    # points on integer coordinates: corners of weight 0 are rows as well
    assert (w == 0).any()
    # interpolate from the splat map: the same corners and weights
    f = z["interp_feats"][rank]
    np.testing.assert_allclose(O.splat_backward(f, rows, w), z["interp_out"], rtol=1e-5,
                               atol=1e-6)
    gf = O.splat_forward(z["interp_grad_out"], rows, w, len(coords))
    np.testing.assert_allclose(gf[perm], z["interp_grad_feats"], rtol=1e-5, atol=1e-6)


def test_public_names():
    import minkowskiengine_b200 as ME
    for name in ("MinkowskiPoolingTranspose", "MinkowskiLocalPoolingTransposeFunction",
                 "MinkowskiStackCat", "MinkowskiStackSum", "MinkowskiStackMean",
                 "MinkowskiStackVar", "MinkowskiToFeature", "sum", "mean", "var", "cat"):
        assert hasattr(ME, name), name
    assert callable(ME.TensorField.splat)
    assert callable(ME.backend.LocalPoolingTransposeForwardGPU)
    assert callable(ME.backend.LocalPoolingTransposeBackwardGPU)
    assert "meb200_splat_coords" in ME._lib.PROTOTYPES


def test_pooling_transpose_sums_whatever_the_mode():
    """The layer's pooling_mode is the base class's default (average); the native call is the sum
    in every case, as both reference backends compute it."""
    import inspect

    import minkowskiengine_b200 as ME
    layer = ME.MinkowskiPoolingTranspose(kernel_size=2, stride=2, dimension=3)
    assert layer.is_transpose and layer.pooling is ME.MinkowskiLocalPoolingTransposeFunction
    assert layer.pooling_mode == ME.PoolingMode.LOCAL_AVG_POOLING
    src = inspect.getsource(ME.backend.LocalPoolingTransposeForwardGPU)
    assert "_lib.POOL_SUM" in src and "_POOL_CODE" not in src
    src = inspect.getsource(ME.backend.LocalPoolingTransposeBackwardGPU)
    assert "_lib.POOL_SUM" in src and "_POOL_CODE" not in src
    assert layer.kernel_generator.expand_coordinates is False
    assert ME.MinkowskiPoolingTranspose(2, 2, expand_coordinates=True,
                                        dimension=3).kernel_generator.expand_coordinates
