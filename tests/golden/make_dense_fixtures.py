"""Generates dense-tensor interop results of the COMPILED REFERENCE (oracle/_ref, built by
oracle/build_ref.py, CPU path) on the seeded cases of tests/test_gpu_dense.py.  Run where the
reference is available:

    python tests/golden/make_dense_fixtures.py

Writes
  tests/golden/ref_dense_<case>.npz            SparseTensor.dense for every DENSE_CASES entry:
                                               D = 2, 3, 4, with and without min_coordinate and
                                               shape, contract_stride=False, at tensor stride 1 and
                                               on the map a stride-2 convolution made
  tests/golden/ref_dense_to_sparse_<case>.npz  to_sparse for formats "BCXX", "BXXXC" and the
                                               default, with all-zero cells and a cell whose
                                               channels cancel in sum but not in abs-sum
  tests/golden/ref_dense_all.npz               to_sparse_all and dense_coordinates
  tests/golden/ref_dense_head.npz              one fp32 forward + backward of
                                               examples/dense_head.py, with the gradient of the
                                               dense input

Every case stores its inputs, the forward values and the gradient of a seeded output gradient.
dense() cases store their rows in sorted-coordinate order (a dense tensor does not depend on the
row order); to_sparse rows are in the reference's own order, torch.where's."""
import os
import sys

os.environ["OMP_NUM_THREADS"] = "1"     # before torch and the reference load libgomp

import numpy as np  # noqa: E402
import torch  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

import dense_oracle as O  # noqa: E402
import test_gpu_dense as T  # noqa: E402


def dense_case(ME, name):
    D, s, use_min, use_shape, contract = T.DENSE_CASES[name]
    base, coords, feats, min_c, shape = T.dense_case(name)
    x = ME.SparseTensor(torch.ones(len(base), 1), torch.from_numpy(base))
    if s > 1:   # the map a strided convolution makes
        x = ME.MinkowskiConvolution(1, 1, kernel_size=2, stride=s, dimension=D)(x)
    c = x.C.numpy()
    perm = O.canon(c)
    assert (c[perm] == coords).all()
    f = np.empty_like(feats)
    f[perm] = feats
    leaf = torch.from_numpy(f).requires_grad_()
    y = ME.SparseTensor(leaf, coordinate_map_key=x.coordinate_map_key,
                        coordinate_manager=x.coordinate_manager)
    d, mn, st = y.dense(shape=None if shape is None else torch.Size(shape),
                        min_coordinate=None if min_c is None else torch.IntTensor(min_c),
                        contract_stride=contract)
    assert st.tolist() == [s] * D
    g = np.random.default_rng(1000).standard_normal(tuple(d.shape)).astype(np.float32)
    d.backward(torch.from_numpy(g))
    np.savez_compressed(os.path.join(HERE, f"ref_dense_{name}.npz"), coords=coords, feats=feats,
                        dense=d.detach().numpy(),
                        min_coordinate=np.asarray(mn).reshape(-1).astype(np.int32),
                        grad_out=g, grad_feats=leaf.grad.numpy()[perm])
    print("dense", name, len(coords), "rows ->", tuple(d.shape), flush=True)


def to_sparse_case(ME, name):
    fmt, _ = T.TO_SPARSE_CASES[name]
    x = torch.from_numpy(T.to_sparse_volume(name)).requires_grad_()
    st = ME.to_sparse(x, fmt)
    g = np.random.default_rng(2000).standard_normal(tuple(st.F.shape)).astype(np.float32)
    st.F.backward(torch.from_numpy(g))
    np.savez_compressed(os.path.join(HERE, f"ref_dense_to_sparse_{name}.npz"),
                        coords=st.C.numpy(), feats=st.F.detach().numpy(), grad_out=g,
                        grad_x=x.grad.numpy())
    print("to_sparse", name, tuple(x.shape), "->", len(st), "rows", flush=True)


def all_case(ME):
    rng = np.random.default_rng(3000)
    x = torch.from_numpy(rng.standard_normal(T.ALL_SHAPE).astype(np.float32)).requires_grad_()
    st = ME.to_sparse_all(x)
    g = rng.standard_normal(tuple(st.F.shape)).astype(np.float32)
    st.F.backward(torch.from_numpy(g))
    np.savez_compressed(os.path.join(HERE, "ref_dense_all.npz"), x=x.detach().numpy(),
                        coords=st.C.numpy(), feats=st.F.detach().numpy(), grad_out=g,
                        grad_x=x.grad.numpy(),
                        dense_coordinates=ME.dense_coordinates(T.COORD_SHAPE).numpy())


def head_case(ME):
    from examples.dense_head import dense_head
    from helpers import state_digest
    torch.manual_seed(0)
    net = dense_head(ME)
    out = {"init_digest": state_digest(net)}
    v, y = T.head_step(ME, net, "cpu")
    out["out"] = y.detach().numpy()
    out["grad_volume"] = v.grad.numpy()
    params = dict(net.named_parameters())
    for p in T.HEAD_PARAMS:
        out[f"{p}/grad"] = params[p].grad.numpy()
    np.savez_compressed(os.path.join(HERE, "ref_dense_head.npz"), **out)
    print("dense head", tuple(v.shape), "->", tuple(y.shape), flush=True)


def main():
    from oracle.ref import import_reference
    ME = import_reference()
    for name in T.DENSE_CASES:
        dense_case(ME, name)
    for name in T.TO_SPARSE_CASES:
        to_sparse_case(ME, name)
    all_case(ME)
    head_case(ME)
    print("wrote tests/golden/ref_dense_*.npz")


if __name__ == "__main__":
    main()
