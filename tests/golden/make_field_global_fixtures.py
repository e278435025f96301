"""Generates global pooling over TensorField points and a MinkowskiPointNet step with the COMPILED
REFERENCE (oracle/_ref, built by oracle/build_ref.py) on seeded inputs.  Run where the reference is
available:

    python tests/golden/make_field_global_fixtures.py

Writes
  tests/golden/ref_field_global_{sum,avg,max}.npz  3 or 4 clouds of shuffled float points with
                        integer batch values: points, features, output, output gradient and input
                        gradient.  Max goes through MinkowskiGlobalMaxPooling(field); sum and avg go
                        through MinkowskiGlobalPoolingFunction.apply with the field key in the
                        _KERNEL modes (the reference's Python layer routes only max to a field, and
                        its _PYTORCH_INDEX sum / avg write cloud b to row batch_index[b])
  tests/golden/ref_field_pointnet.npz  one fp32 training step of examples/pointnet.py (small
                        widths, no dropout) on the inputs of tests/test_gpu_field_global.py:
                        initial-weight digest, logits, loss and sampled gradients

The reference's origin-map row order is implementation-defined, so per-cloud rows are stored in
ascending batch order, the order this package defines."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

SAMPLE_ELEMS = 2048


def field_points(seed, batches, n, C):
    g = np.random.default_rng(seed)
    b = np.concatenate([np.asarray(batches), g.choice(batches, n - len(batches))])
    g.shuffle(b)
    xyz = g.uniform(-10, 10, (n, 3))
    pts = np.concatenate([b[:, None], xyz], 1).astype(np.float32)
    return pts, g.standard_normal((n, C)).astype(np.float32)


def _origin_perm(y):
    """perm with (reference origin rows)[perm] in ascending batch order."""
    return np.argsort(y.C.numpy()[:, 0], kind="stable")


def global_case(ME, mode, seed, batches):
    pts, feats = field_points(seed, batches, 1400, 6)
    x = ME.TensorField(torch.from_numpy(feats).requires_grad_(True), torch.from_numpy(pts))
    if mode == "max":
        y = ME.MinkowskiGlobalMaxPooling()(x)
    else:
        pm = {"sum": ME.PoolingMode.GLOBAL_SUM_POOLING_KERNEL,
              "avg": ME.PoolingMode.GLOBAL_AVG_POOLING_KERNEL}[mode]
        out_key = ME.CoordinateMapKey(x.coordinate_field_map_key.get_coordinate_size())
        F = ME.MinkowskiGlobalPoolingFunction.apply(x.F, pm, x.coordinate_field_map_key, out_key,
                                                     x._manager)
        y = ME.SparseTensor(F, coordinate_map_key=out_key, coordinate_manager=x._manager)
    perm = _origin_perm(y)
    gout = torch.rand(y.F.shape, generator=torch.Generator().manual_seed(seed))
    g_ref = torch.empty_like(gout)
    g_ref[perm] = gout                         # reference row perm[k] = canonical row k
    y.F.backward(g_ref)
    np.savez_compressed(os.path.join(HERE, f"ref_field_global_{mode}.npz"), pts=pts, feats=feats,
                        out_coords=y.C.numpy()[perm], out_feats=y.F.detach().numpy()[perm],
                        grad_out=gout.numpy(), grad_in=x.F.grad.numpy())
    print("wrote field global", mode, flush=True)


def pointnet_case(REF):
    import test_gpu_field_global as T
    from helpers import state_digest
    net = T.pointnet_net(REF)
    out = {"init_digest": state_digest(net)}
    y, loss = T.pointnet_step(REF, net, "cpu")
    perm = _origin_perm(y)
    out["out_coords"] = y.C.numpy()[perm]
    out["logits"] = y.F.detach().numpy()[perm]
    out["loss"] = np.float64(loss)
    params = dict(net.named_parameters())
    rng = np.random.default_rng(5)
    for p in T.POINTNET_PARAMS:
        gr = params[p].grad.numpy().ravel()
        idx = np.sort(rng.choice(gr.size, min(gr.size, SAMPLE_ELEMS), replace=False))
        out[f"{p}/idx"] = idx.astype(np.int64)
        out[f"{p}/grad"] = gr[idx].astype(np.float32)
        out[f"{p}/absmax"] = np.float64(np.abs(gr).max())
    print("pointnet loss", loss, flush=True)
    np.savez_compressed(os.path.join(HERE, "ref_field_pointnet.npz"), **out)


def main():
    from oracle.ref import import_reference
    ME = import_reference()
    torch.set_num_threads(os.cpu_count() or 1)
    global_case(ME, "sum", 40, [0, 1, 2])
    global_case(ME, "avg", 41, [0, 1, 2, 3])
    global_case(ME, "max", 42, [0, 2, 3])
    pointnet_case(ME)


if __name__ == "__main__":
    main()
