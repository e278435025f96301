"""Generates sparse-matrix and direct max pooling results of the COMPILED REFERENCE (oracle/_ref,
built by oracle/build_ref.py) on seeded inputs.  Run where the reference is available:

    python tests/golden/make_spmm_fixtures.py

Writes
  tests/golden/ref_spmm_small.npz       spmm and spmm_average (the reference's CPU path,
  tests/golden/ref_spmm_cloud.npz       torch.sparse), forward and the backward spmm over the
                                        transposed matrix, on unsorted entries with duplicate
                                        pairs, rows without entries and unused columns
  tests/golden/ref_direct_max_small.npz direct_max_pool_fw / _bw of the compiled reference on
  tests/golden/ref_direct_max_cloud.npz unsorted pairs with repeated pairs and input rows no pair
                                        reads; every output row has pairs and a positive value
                                        in each channel (the reference starts its maximum from 0
                                        with mask 0, which this package does not)

Each file stores the inputs, the forward values and the gradient of a seeded output gradient.
The script runs on one thread so that it rewrites the committed files bit for bit."""
import os
import sys

os.environ["OMP_NUM_THREADS"] = "1"     # before torch and the reference load libgomp

import numpy as np  # noqa: E402
import torch  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

# name -> (entries, rows, columns, channels, seed)
SPMM_CASES = {"small": (40, 9, 7, 3, 1), "cloud": (3000, 700, 500, 8, 2)}
MAX_CASES = {"small": (40, 12, 6, 3, 3), "cloud": (4000, 900, 600, 7, 4)}


def coo_entries(P, n_rows, n_cols, rng):
    """Unsorted (rows, cols) with a block of repeated pairs; rows >= n_rows - 2 and column 0 never
    appear (empty output rows, an unused column)."""
    rows = rng.integers(0, n_rows - 2, P)
    cols = rng.integers(1, n_cols, P)
    k = P // 8
    rows[-k:], cols[-k:] = rows[:k], cols[:k]           # duplicates
    perm = rng.permutation(P)
    return rows[perm].astype(np.int32), cols[perm].astype(np.int32)


def spmm_case(ME, name):
    P, n_rows, n_cols, C, seed = SPMM_CASES[name]
    rng = np.random.default_rng(seed)
    rows, cols = coo_entries(P, n_rows, n_cols, rng)
    vals = rng.standard_normal(P).astype(np.float32)
    mat = rng.standard_normal((n_cols, C)).astype(np.float32)
    g = rng.standard_normal((n_rows, C)).astype(np.float32)
    size = torch.Size([n_rows, n_cols])
    r, c, v = torch.from_numpy(rows), torch.from_numpy(cols), torch.from_numpy(vals)
    out = ME.spmm(r, c, v, size, torch.from_numpy(mat))
    grad = ME.spmm(c, r, v, torch.Size([n_cols, n_rows]), torch.from_numpy(g))
    from sparse_matrix_functions import spmm_average
    avg, coo, avals = spmm_average(r, c, size, torch.from_numpy(mat))
    avg_grad = ME.spmm(coo[1], coo[0], avals, torch.Size([n_cols, n_rows]), torch.from_numpy(g))
    return dict(rows=rows, cols=cols, vals=vals, mat=mat, grad_out=g, shape=np.array([n_rows, n_cols]),
                out=out.numpy(), grad=grad.numpy(), avg=avg.numpy(), avg_coo=coo.numpy(),
                avg_vals=avals.numpy(), avg_grad=avg_grad.numpy())


def max_case(name):
    import MinkowskiEngineBackend._C as _C
    P, n_in, n_out, C, seed = MAX_CASES[name]
    rng = np.random.default_rng(seed)
    # every output row gets pairs; input rows >= n_in - 3 are never read
    out_map = np.concatenate([np.arange(n_out), rng.integers(0, n_out, P - n_out)])
    in_map = rng.integers(0, n_in - 3, P)
    k = P // 8
    in_map[-k:], out_map[-k:] = in_map[:k], out_map[:k]     # repeated pairs
    perm = rng.permutation(P)
    in_map, out_map = in_map[perm].astype(np.int32), out_map[perm].astype(np.int32)
    x = rng.standard_normal((n_in, C)).astype(np.float32)
    x[x == 0] = 1.0
    x = np.round(x * 4) / 4                                   # ties between distinct inputs
    # a positive value in every channel of every output row: the row's first pair's input
    first = np.unique(out_map, return_index=True)[1]
    x[in_map[first]] = np.abs(x[in_map[first]]) + 0.25
    g = rng.standard_normal((n_out, C)).astype(np.float32)
    out, mask = _C.direct_max_pool_fw(torch.from_numpy(in_map), torch.from_numpy(out_map),
                                      torch.from_numpy(x), n_out, False)
    grad = _C.direct_max_pool_bw(torch.from_numpy(g), mask, n_in)
    return dict(in_map=in_map, out_map=out_map, feats=x, grad_out=g, n_out=np.array(n_out),
                out=out.numpy(), mask=mask.numpy(), grad=grad.numpy())


def main():
    from oracle import ref
    ME = ref.import_reference()
    torch.manual_seed(0)
    for name in SPMM_CASES:
        np.savez(os.path.join(HERE, f"ref_spmm_{name}.npz"), **spmm_case(ME, name))
    for name in MAX_CASES:
        np.savez(os.path.join(HERE, f"ref_direct_max_{name}.npz"), **max_case(name))
    print("wrote", ", ".join([f"ref_spmm_{n}.npz" for n in SPMM_CASES] +
                             [f"ref_direct_max_{n}.npz" for n in MAX_CASES]))


if __name__ == "__main__":
    main()
