"""Generates TensorField results of the COMPILED REFERENCE (oracle/_ref, built by
oracle/build_ref.py) on seeded inputs.  Run where the reference is available:

    python tests/golden/make_field_fixtures.py

Writes
  tests/golden/ref_field_quantize.npz  a 3-cloud float cloud with 1-30 points per voxel, quantised
                                       at strides 1 and 2 in the four modes: output and gradient
                                       (MAX_POOL on positive features only: the reference's max pool
                                       starts from zero)
  tests/golden/ref_field_slice.npz     slice of the stride-1 voxels and of stride-2 / stride-4 maps
                                       made by max pooling back onto the points, with gradients
  tests/golden/ref_field_interp.npz    features_at_coordinates on a stride-2 map, D = 3 and D = 4,
                                       with queries whose corners are all, partly or not present
  tests/golden/ref_field_fcnn.npz      one fp32 training step of examples/fcnn.py (small channels,
                                       no dropout) on the inputs of tests/test_gpu_field.py:
                                       initial-weight digest, logits, loss and sampled gradients

MinkowskiFCNN slices maps at strides 2-16 back onto the points.  The reference composes the field's
stride-1 map with the stride map by indexing the stride map's (in, out) pairs, which come in
hash-table order, with stride-1 rows (MinkowskiTensorField.py:437-441), so a point does not receive
its own voxel (tests/test_field_cpu.py shows it on ref_field_slice.npz).  For the network run that
one step is corrected: the pairs are put in input-row order before they are indexed.  Everything
else is the reference's code.

Rows of every map are stored in canonical (sorted coordinate) order and output gradients are drawn
in that order, so the fixtures do not depend on the reference's hash-table row order."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

MODES = ("UNWEIGHTED_SUM", "UNWEIGHTED_AVERAGE", "RANDOM_SUBSAMPLE", "MAX_POOL")


def canon(coords):
    c = np.asarray(coords)
    return np.lexsort(c.T[::-1])


def field_cloud(seed, clouds=3, voxels=120, extent=8, max_pts=30, C=5):
    """Float points: `voxels` voxels per cloud, 1..max_pts points each, in shuffled order."""
    g = np.random.default_rng(seed)
    pts = []
    for b in range(clouds):
        vox = np.unique(g.integers(-extent, extent, (voxels, 3)), axis=0)
        cnt = g.integers(1, max_pts + 1, len(vox))
        rep = np.repeat(vox, cnt, axis=0).astype(np.float64)
        rep += g.uniform(0.02, 0.98, rep.shape)
        pts.append(np.concatenate([np.full((len(rep), 1), b, np.float64), rep], 1))
    pts = np.concatenate(pts).astype(np.float32)
    pts = pts[g.permutation(len(pts))]
    feats = g.uniform(0.1, 2.0, (len(pts), C)).astype(np.float32)
    return pts, feats


def quantize(ME):
    pts, feats = field_cloud(0)
    out = {"coords": pts, "feats": feats}
    for s in (1, 2):
        for mode in MODES:
            x = torch.from_numpy(feats).clone().requires_grad_()
            tf = ME.TensorField(x, torch.from_numpy(pts),
                                quantization_mode=getattr(ME.SparseTensorQuantizationMode, mode))
            st = tf.sparse(tensor_stride=s)
            c = st.C.numpy()
            perm = canon(c)
            g = np.random.default_rng(100 + s).standard_normal(st.F.shape).astype(np.float32)
            g_ref = np.empty_like(g)
            g_ref[perm] = g
            st.F.backward(torch.from_numpy(g_ref))
            tag = f"{mode}_s{s}"
            out[f"{tag}_out_coords"] = c[perm]
            out[f"{tag}_out"] = st.F.detach().numpy()[perm]
            out[f"{tag}_grad_out"] = g
            out[f"{tag}_grad_in"] = x.grad.numpy()
    np.savez_compressed(os.path.join(HERE, "ref_field_quantize.npz"), **out)


def slicing(ME):
    pts, feats = field_cloud(1, C=4)
    tf = ME.TensorField(torch.from_numpy(feats), torch.from_numpy(pts))
    st = tf.sparse()
    pool = ME.MinkowskiMaxPooling(kernel_size=2, stride=2, dimension=3)
    levels = {1: st, 2: pool(st)}
    levels[4] = pool(levels[2])
    out = {"coords": pts, "feats": feats}
    rng = np.random.default_rng(7)
    for s, y in levels.items():
        c = y.C.numpy()
        perm = canon(c)
        f = rng.standard_normal(y.F.shape).astype(np.float32)   # canonical order
        f_ref = np.empty_like(f)
        f_ref[perm] = f
        leaf = torch.from_numpy(f_ref).requires_grad_()
        ys = ME.SparseTensor(leaf, coordinate_map_key=y.coordinate_map_key,
                             coordinate_manager=y.coordinate_manager)
        sl = ys.slice(tf)
        g = rng.standard_normal(sl.F.shape).astype(np.float32)
        sl.F.backward(torch.from_numpy(g))
        out[f"s{s}_coords"] = c[perm]
        out[f"s{s}_feats"] = f
        out[f"s{s}_out"] = sl.F.detach().numpy()
        out[f"s{s}_grad_out"] = g
        out[f"s{s}_grad_feats"] = leaf.grad.numpy()[perm]
    np.savez_compressed(os.path.join(HERE, "ref_field_slice.npz"), **out)


def interpolation(ME):
    out = {}
    for D in (3, 4):
        rng = np.random.default_rng(20 + D)
        vox = np.unique(rng.integers(-6, 6, (300 if D == 3 else 500, D)), axis=0) * 2
        b = rng.integers(0, 2, (len(vox), 1))
        coords = np.unique(np.concatenate([b, vox], 1), axis=0).astype(np.int32)
        feats = rng.standard_normal((len(coords), 6)).astype(np.float32)
        # queries: near voxels (most corners present), across the region (some present) and far
        # outside (none present)
        near = coords[rng.integers(0, len(coords), 200)].astype(np.float64)
        near[:, 1:] += rng.uniform(-1.9, 1.9, (200, D))
        wide = np.concatenate([rng.integers(0, 2, (150, 1)),
                               rng.uniform(-14, 14, (150, D))], 1)
        far = np.concatenate([rng.integers(0, 2, (30, 1)), rng.uniform(40, 60, (30, D))], 1)
        q = np.concatenate([near, wide, far]).astype(np.float32)
        x = torch.from_numpy(feats).clone().requires_grad_()
        st = ME.SparseTensor(x, torch.from_numpy(coords), tensor_stride=2)
        assert len(st) == len(coords)
        y = st.features_at_coordinates(torch.from_numpy(q))
        g = rng.standard_normal(y.shape).astype(np.float32)
        y.backward(torch.from_numpy(g))
        out[f"d{D}_coords"] = coords
        out[f"d{D}_feats"] = feats
        out[f"d{D}_query"] = q
        out[f"d{D}_out"] = y.detach().numpy()
        out[f"d{D}_grad_out"] = g
        out[f"d{D}_grad_feats"] = x.grad.numpy()
    np.savez_compressed(os.path.join(HERE, "ref_field_interp.npz"), **out)


SAMPLE_ELEMS = 2048


def _ordered_inverse_mapping(REF):
    """The reference's TensorField.inverse_mapping with the stride map indexed by input row."""
    def inverse_mapping(self, key):
        if key not in self._inverse_mapping:
            mgr, fk = self._manager, self.coordinate_field_map_key
            if mgr.exists_field_to_sparse(fk, key):
                self._inverse_mapping[key] = mgr.get_field_to_sparse_map(fk, key)[1]
            else:
                one = [k for k in mgr.field_to_sparse_keys(fk)
                       if np.prod(k.get_tensor_stride()) == 1][0]
                base = self.inverse_mapping(one)
                in_rows, out_rows = mgr.stride_map(one, key)
                by_row = torch.empty(mgr.size(one), dtype=torch.int64)
                by_row[in_rows.long()] = out_rows.long()
                self._inverse_mapping[key] = by_row[base.long()]
        return self._inverse_mapping[key]
    return inverse_mapping


def fcnn_case(REF):
    sys.path.insert(0, os.path.dirname(HERE))
    import test_gpu_field as T
    from helpers import state_digest
    REF.TensorField.inverse_mapping = _ordered_inverse_mapping(REF)
    net = T.fcnn_net(REF)
    out = {"init_digest": state_digest(net)}
    y, loss = T.fcnn_step(REF, net, "cpu")
    perm = np.argsort(y.C.numpy()[:, 0], kind="stable")
    out["out_coords"] = y.C.numpy()[perm]
    out["logits"] = y.F.detach().numpy()[perm]
    out["loss"] = np.float64(loss)
    params = dict(net.named_parameters())
    rng = np.random.default_rng(5)
    for p in T.FCNN_PARAMS:
        gr = params[p].grad.numpy().ravel()
        idx = np.sort(rng.choice(gr.size, min(gr.size, SAMPLE_ELEMS), replace=False))
        out[f"{p}/idx"] = idx.astype(np.int64)
        out[f"{p}/grad"] = gr[idx].astype(np.float32)
        out[f"{p}/absmax"] = np.float64(np.abs(gr).max())
    print("fcnn loss", loss, flush=True)
    np.savez_compressed(os.path.join(HERE, "ref_field_fcnn.npz"), **out)


def main():
    from oracle.ref import import_reference
    ME = import_reference()
    torch.manual_seed(0)
    quantize(ME)
    slicing(ME)
    interpolation(ME)
    fcnn_case(ME)
    print("wrote tests/golden/ref_field_{quantize,slice,interp,fcnn}.npz")


if __name__ == "__main__":
    main()
