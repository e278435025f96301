"""TEST INFRASTRUCTURE — numpy restatement of the dense-tensor interop (csrc/dense.cu,
minkowskiengine_b200/dense.py).  Dense arrays are [B, C, X1..XD]; coordinate rows int32 [n, D+1]
with the batch index first.  Everything is data movement, so results are exact."""
import numpy as np


def canon(coords):
    """Permutation that sorts coordinate rows lexicographically."""
    return np.lexsort(coords.T[::-1])


def rows_to_dense(coords, feats, shape, origin, step):
    """dense[b, :, i] = feats[r] for the row r at coordinate origin + i * step; rows outside the
    volume or off the step lattice are cropped; every other cell is zero."""
    dense = np.zeros(shape, feats.dtype)
    rel = coords[:, 1:].astype(np.int64) - np.asarray(origin, np.int64)
    step = np.asarray(step, np.int64)
    idx = rel // step
    ok = (rel % step == 0).all(1) & (idx >= 0).all(1) & (idx < np.asarray(shape[2:])).all(1) & \
        (coords[:, 0] >= 0) & (coords[:, 0] < shape[0])
    cell = (coords[ok, 0],) + tuple(idx[ok].T)
    np.moveaxis(dense, 1, -1)[cell] = feats[ok]
    return dense


def dense_to_rows(dense, coords, origin, step):
    """out[r] = the cell of coordinate row r, zero for a row outside the volume or off the
    lattice: the transpose of rows_to_dense."""
    shape = dense.shape
    out = np.zeros((len(coords), shape[1]), dense.dtype)
    rel = coords[:, 1:].astype(np.int64) - np.asarray(origin, np.int64)
    step = np.asarray(step, np.int64)
    idx = rel // step
    ok = (rel % step == 0).all(1) & (idx >= 0).all(1) & (idx < np.asarray(shape[2:])).all(1) & \
        (coords[:, 0] >= 0) & (coords[:, 0] < shape[0])
    cell = (coords[ok, 0],) + tuple(idx[ok].T)
    out[ok] = np.moveaxis(dense, 1, -1)[cell]
    return out


def nonzero_coordinates(dense):
    """int32 [M, D+1] cells with a non-zero channel (NaN counts), row-major."""
    keep = (np.moveaxis(dense, 1, -1) != 0).any(-1)
    return np.stack(np.nonzero(keep), 1).astype(np.int32)


def dense_coordinates(shape):
    """int32 [B * prod(X), D+1]: every cell of a [B, C, X1..XD] tensor, row-major."""
    sizes = (shape[0], *shape[2:])
    return np.stack([g.reshape(-1) for g in np.meshgrid(*(np.arange(s) for s in sizes),
                                                        indexing="ij")], 1).astype(np.int32)


def dense_extent(coords, tensor_stride, channels, min_coordinate, contract_stride):
    """(origin, step, shape) SparseTensor.dense uses when `shape` is None."""
    ts = np.asarray(tensor_stride, np.int64)
    origin = coords[:, 1:].min(0).astype(np.int64) if min_coordinate is None \
        else np.asarray(min_coordinate, np.int64)
    step = ts if contract_stride else np.ones_like(ts)
    spatial = (coords[:, 1:].max(0) - origin) // step + 1
    return origin, step, [int(coords[:, 0].max()) + 1, channels] + [int(s) for s in spatial]
