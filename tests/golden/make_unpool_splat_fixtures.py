"""Generates unpooling and splatting results of the COMPILED REFERENCE (oracle/_ref, built by
oracle/build_ref.py) on seeded inputs.  Run where the reference is available:

    python tests/golden/make_unpool_splat_fixtures.py

Writes
  tests/golden/ref_unpool_k2s2_d3.npz      MinkowskiPoolingTranspose k2s2 onto the stride-1 map, after
                                           a k2s2 max pool of it (the stride-map path), D = 3
  tests/golden/ref_unpool_k3s2_d2.npz      k3s2 after a k3s2 sum pool (the kernel-map path), D = 2
  tests/golden/ref_unpool_k2s2_expand.npz  k2s2 with expand_coordinates=True (new coordinates), D = 3
  tests/golden/ref_unpool_k2s2_d4.npz      k2s2 at D = 4
  tests/golden/ref_splat_small.npz         the reference's test_small / test_small2 points (D = 1, 2)
  tests/golden/ref_splat_cloud.npz         a D = 3 cloud with negative coordinates, points on integer
                                           coordinates and many points per corner; splat, and
                                           interpolate from the splat map back onto the points
  tests/golden/ref_unpool_stack_unet.npz   one fp32 training step of examples/stack_unet.py
  tests/golden/ref_splat_fcnn.npz          one fp32 training step of examples/fcnn.py (splat=True)

Every case stores its input and output coordinates, forward values and the gradient of a seeded
output gradient.  Rows of every map are stored in canonical (sorted coordinate) order and output
gradients are drawn in that order, so the fixtures do not depend on the reference's hash-table row
order.  The reference's CPU sums are added in an order that depends on its OpenMP threads, so the
script runs on one thread: it then rewrites the committed files bit for bit."""
import os
import sys

os.environ["OMP_NUM_THREADS"] = "1"     # before torch and the reference load libgomp

import numpy as np  # noqa: E402
import torch  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

from make_field_fixtures import SAMPLE_ELEMS, canon  # noqa: E402

# name -> (D, pooling before the unpool, kernel size, stride, expand_coordinates, seed)
UNPOOL_CASES = {
    "k2s2_d3": (3, "max", 2, 2, False, 1),
    "k3s2_d2": (2, "sum", 3, 2, False, 2),
    "k2s2_expand": (3, "max", 2, 2, True, 3),
    "k2s2_d4": (4, "max", 2, 2, False, 4),
}
C_UNPOOL = 4


def unpool_cloud(D, seed):
    g = np.random.default_rng(seed)
    n = {2: 300, 3: 600, 4: 700}[D]
    ext = {2: 12, 3: 8, 4: 5}[D]
    c = np.concatenate([g.integers(0, 2, (n, 1)), g.integers(-ext, ext, (n, D))], 1)
    return np.unique(c, axis=0).astype(np.int32)[g.permutation(len(np.unique(c, axis=0)))]


def _leaf_on(ME, y, f_canon):
    """A leaf SparseTensor on y's map with features given in canonical row order."""
    perm = canon(y.C.numpy())
    f = np.empty_like(f_canon)
    f[perm] = f_canon
    leaf = torch.from_numpy(f).requires_grad_()
    return leaf, ME.SparseTensor(leaf, coordinate_map_key=y.coordinate_map_key,
                                 coordinate_manager=y.coordinate_manager), perm


def unpool_case(ME, name):
    D, pool, k, s, expand, seed = UNPOOL_CASES[name]
    coords = unpool_cloud(D, seed)
    rng = np.random.default_rng(100 + seed)
    x = ME.SparseTensor(torch.ones(len(coords), 1), torch.from_numpy(coords))
    P = ME.MinkowskiMaxPooling if pool == "max" else ME.MinkowskiSumPooling
    y = P(kernel_size=k, stride=s, dimension=D)(x)
    f = rng.standard_normal((len(y), C_UNPOOL)).astype(np.float32)
    leaf, ys, pin = _leaf_on(ME, y, f)
    out = ME.MinkowskiPoolingTranspose(kernel_size=k, stride=s, expand_coordinates=expand,
                                       dimension=D)(ys)
    c = out.C.numpy()
    po = canon(c)
    g = rng.standard_normal(out.F.shape).astype(np.float32)
    g_ref = np.empty_like(g)
    g_ref[po] = g
    out.F.backward(torch.from_numpy(g_ref))
    np.savez_compressed(os.path.join(HERE, f"ref_unpool_{name}.npz"),
                        coords=coords, in_coords=y.C.numpy()[pin], in_feats=f,
                        out_coords=c[po], out=out.F.detach().numpy()[po], grad_out=g,
                        grad_in=leaf.grad.numpy()[pin])
    print("unpool", name, len(coords), "->", len(y), "->", len(c), flush=True)


def _splat(ME, pts, feats, seed, tag, out):
    rng = np.random.default_rng(seed)
    x = torch.from_numpy(feats).clone().requires_grad_()
    tf = ME.TensorField(x, torch.from_numpy(pts))
    st = tf.splat()
    c = st.C.numpy()
    perm = canon(c)
    g = rng.standard_normal(st.F.shape).astype(np.float32)
    g_ref = np.empty_like(g)
    g_ref[perm] = g
    st.F.backward(torch.from_numpy(g_ref))
    out[f"{tag}coords"] = pts
    out[f"{tag}feats"] = feats
    out[f"{tag}out_coords"] = c[perm]
    out[f"{tag}out"] = st.F.detach().numpy()[perm]
    out[f"{tag}grad_out"] = g
    out[f"{tag}grad_in"] = x.grad.numpy()
    return tf, st, rng


def splat_small(ME):
    out = {}
    for tag, pts in (("small_", [[0, 0.1], [0, 1.1]]), ("small2_", [[0, 0.1, 0.1], [0, 1.1, 1.1]])):
        _splat(ME, np.array(pts, np.float32), np.array([[1], [2]], np.float32), 9, tag, out)
    np.savez_compressed(os.path.join(HERE, "ref_splat_small.npz"), **out)


def splat_cloud_points(seed=5, C=3):
    """D = 3, two clouds: points across [-4, 4) (negative coordinates), points on integer
    coordinates (corners of weight 0) and a cluster of many points inside one cell."""
    g = np.random.default_rng(seed)
    wide = np.concatenate([g.integers(0, 2, (400, 1)), g.uniform(-4, 4, (400, 3))], 1)
    ints = np.concatenate([g.integers(0, 2, (30, 1)), g.integers(-4, 4, (30, 3))], 1)
    half = np.concatenate([g.integers(0, 2, (20, 1)), g.integers(-4, 4, (20, 3)) +
                           np.array([0.5, 0, 0])], 1)           # integer on two axes
    cluster = np.concatenate([np.zeros((60, 1)), -1.5 + g.uniform(-0.4, 0.4, (60, 3))], 1)
    pts = np.concatenate([wide, ints, half, cluster]).astype(np.float32)
    pts = pts[g.permutation(len(pts))]
    feats = g.standard_normal((len(pts), C)).astype(np.float32)
    return pts, feats


def splat_cloud(ME):
    pts, feats = splat_cloud_points()
    out = {}
    tf, st, rng = _splat(ME, pts, feats, 6, "", out)
    # interpolate from the splat map back onto the points: a leaf on the splat map
    f = rng.standard_normal((len(st), 5)).astype(np.float32)
    leaf, ys, perm = _leaf_on(ME, st, f)
    y = ys.interpolate(tf)
    g = rng.standard_normal(y.F.shape).astype(np.float32)
    y.F.backward(torch.from_numpy(g))
    out["interp_feats"] = f
    out["interp_out"] = y.F.detach().numpy()
    out["interp_grad_out"] = g
    out["interp_grad_feats"] = leaf.grad.numpy()[perm]
    np.savez_compressed(os.path.join(HERE, "ref_splat_cloud.npz"), **out)
    print("splat cloud", len(pts), "points ->", len(st), "voxels", flush=True)


def _sampled_grads(net, names, seed, out):
    params = dict(net.named_parameters())
    rng = np.random.default_rng(seed)
    for p in names:
        gr = params[p].grad.numpy().ravel()
        idx = np.sort(rng.choice(gr.size, min(gr.size, SAMPLE_ELEMS), replace=False))
        out[f"{p}/idx"] = idx.astype(np.int64)
        out[f"{p}/grad"] = gr[idx].astype(np.float32)
        out[f"{p}/absmax"] = np.float64(np.abs(gr).max())


def networks(REF):
    import test_gpu_unpool_splat as T
    from helpers import state_digest
    net = T.stack_unet_net(REF)
    out = {"init_digest": state_digest(net)}
    logits, loss = T.stack_unet_step(REF, net, "cpu")
    out["logits"] = logits.detach().numpy()
    out["loss"] = np.float64(loss)
    _sampled_grads(net, T.STACK_PARAMS, 5, out)
    print("stack_unet loss", loss, flush=True)
    np.savez_compressed(os.path.join(HERE, "ref_unpool_stack_unet.npz"), **out)

    net = T.splat_fcnn_net(REF)
    out = {"init_digest": state_digest(net)}
    y, loss = T.splat_fcnn_step(REF, net, "cpu")
    perm = np.argsort(y.C.numpy()[:, 0], kind="stable")
    out["out_coords"] = y.C.numpy()[perm]
    out["logits"] = y.F.detach().numpy()[perm]
    out["loss"] = np.float64(loss)
    _sampled_grads(net, T.FCNN_PARAMS, 5, out)
    print("splat fcnn loss", loss, flush=True)
    np.savez_compressed(os.path.join(HERE, "ref_splat_fcnn.npz"), **out)


def main():
    from oracle.ref import import_reference
    ME = import_reference()
    torch.manual_seed(0)
    for name in UNPOOL_CASES:
        unpool_case(ME, name)
    splat_small(ME)
    splat_cloud(ME)
    networks(ME)
    print("wrote tests/golden/ref_unpool_*.npz and ref_splat_*.npz")


if __name__ == "__main__":
    main()
