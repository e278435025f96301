"""Dense-tensor interop without a GPU: the numpy restatement (tests/dense_oracle.py) pinned to the
compiled reference's fixtures, the public names, the argument checks of to_sparse, and
dense_coordinates on the CPU."""
import os

import numpy as np
import pytest
import torch

import dense_oracle as O
import test_gpu_dense as T

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _load(name):
    return np.load(os.path.join(GOLDEN, name))


@pytest.mark.parametrize("name", list(T.DENSE_CASES))
def test_dense_oracle_matches_reference(name):
    D, s, use_min, use_shape, contract = T.DENSE_CASES[name]
    z = _load(f"ref_dense_{name}.npz")
    _, coords, feats, min_c, shape = T.dense_case(name)
    assert (coords == z["coords"]).all() and (feats == z["feats"]).all()
    origin, step, extent = O.dense_extent(coords, [s] * D, T.C_DENSE, min_c, contract)
    if shape is not None:
        extent = [shape[0], T.C_DENSE] + shape[2:]      # the channel count of `shape` is replaced
    assert (origin == z["min_coordinate"]).all()
    assert tuple(extent) == z["dense"].shape
    assert (O.rows_to_dense(coords, feats, extent, origin, step) == z["dense"]).all()
    assert (O.dense_to_rows(z["grad_out"], coords, origin, step) == z["grad_feats"]).all()


@pytest.mark.parametrize("name", list(T.TO_SPARSE_CASES))
def test_to_sparse_oracle_matches_reference(name):
    fmt, _ = T.TO_SPARSE_CASES[name]
    z = _load(f"ref_dense_to_sparse_{name}.npz")
    x = np.moveaxis(T.to_sparse_volume(name), 1 if fmt is None else fmt.find("C"), 1)
    coords = O.nonzero_coordinates(x)
    D = x.ndim - 2
    assert (coords == z["coords"]).all()
    assert 0 < len(coords) < x.size // x.shape[1]       # all-zero cells were dropped
    cancel = (coords == np.array([1] + [2] * D)).all(1)
    assert cancel.sum() == 1 and z["feats"][cancel].sum() == 0      # kept by its abs-sum
    assert (O.dense_to_rows(x, coords, [0] * D, [1] * D) == z["feats"]).all()
    gx = O.rows_to_dense(coords, z["grad_out"], x.shape, [0] * D, [1] * D)
    assert (np.moveaxis(gx, 1, 1 if fmt is None else fmt.find("C")) == z["grad_x"]).all()


def test_to_sparse_all_and_dense_coordinates_match_reference(ME):
    z = _load("ref_dense_all.npz")
    coords = O.dense_coordinates(T.ALL_SHAPE)
    assert (coords == z["coords"]).all()
    assert (O.dense_to_rows(z["x"], coords, [0, 0], [1, 1]) == z["feats"]).all()
    assert (O.rows_to_dense(coords, z["grad_out"], T.ALL_SHAPE, [0, 0], [1, 1]) == z["grad_x"]).all()
    assert (O.dense_coordinates(T.COORD_SHAPE) == z["dense_coordinates"]).all()
    got = ME.dense_coordinates(T.COORD_SHAPE)
    assert got.dtype == torch.int32 and not got.is_cuda
    assert (got.numpy() == z["dense_coordinates"]).all()
    with pytest.raises(AssertionError, match="Invalid shape"):
        ME.dense_coordinates((2, 3))


def test_public_names(ME):
    for name in ("to_sparse", "to_sparse_all", "dense_coordinates", "MinkowskiToDenseTensor",
                 "MinkowskiToSparseTensor", "MinkowskiToDenseFunction",
                 "MinkowskiDenseToRowsFunction"):
        assert hasattr(ME, name), name
    m = ME.MinkowskiToSparseTensor(remove_zeros=False, coordinates=None)
    assert m.remove_zeros is False and m.coordinates is None
    assert ME.MinkowskiToDenseTensor(torch.Size([1, 2, 3, 3])).shape == (1, 2, 3, 3)
    from examples.dense_head import dense_head
    assert len(list(dense_head(ME).parameters())) == 9


def test_to_sparse_format_checks(ME):
    x = torch.zeros(2, 3, 4, 4)
    with pytest.raises(AssertionError, match="Input has 0 spatial dimension."):
        ME.to_sparse(torch.zeros(2, 3))
    with pytest.raises(AssertionError, match=r"Invalid format: BCX. len\(format\) != x.ndim"):
        ME.to_sparse(x, "BCX")
    for fmt in ("CBXX", "XCXX", "BBCX"):
        with pytest.raises(AssertionError, match="The input must have the batch axis and the format "
                           "must include 'B' indicating the batch axis."):
            ME.to_sparse(x, fmt)
    for fmt in ("BXXX", "BCCX"):
        with pytest.raises(AssertionError, match="The format must indicate the channel axis"):
            ME.to_sparse(x, fmt)
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        ME.to_sparse(x, "BCXX")
    with pytest.raises(AssertionError, match="Invalid shape"):
        ME.to_sparse_all(torch.zeros(2, 3))
