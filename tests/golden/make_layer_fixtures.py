"""Generates tests/golden/ref_layer_*.npz: one layer per file, run by the COMPILED REFERENCE
(oracle/_ref, built from the reference's sources by oracle/build_ref.py) at the layer shapes the
other fixtures leave out — coordinate widths 2 and 6..8, coordinates near 2^30, non-cubic,
per-axis, even and dilated kernels, inputs at tensor stride 2 and 4, HYPER_CROSS regions,
transposed and generative layers, expanded and caller-given output coordinates, and pooling maps
of strided inputs.  Run where the reference is available:

    python oracle/build_ref.py && python tests/golden/make_layer_fixtures.py

Every file holds the layer's input map as inserted (`raw_coords` at tensor stride `ts_in`, with
duplicates, and the insert's `unique_index` / `inverse_map`), the layer's input coordinates and
features, its weight, the output coordinates, features and `grad_out`, the reference's
`grad_in` / `grad_weight`, and its kernel map as sorted (k, in coordinate, out coordinate) triples.
Derived-map row order is implementation-defined, so every coordinate set is stored in
lexicographic order with its feature rows permuted to match.  `meta` is a JSON record of the
layer's arguments.  Convolution features, weights and `grad_out` are multiples of 2^-7 / 2^-9,
exact in bf16 and fp16, so that a low-precision run reads the same values; pooling features are
all different, so that a max pooling has no ties."""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import oracle_np as O  # noqa: E402
from oracle import ref  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))


def cloud(n, extent, seed, D, ts=1, base=0):
    """n rows (with duplicates) of two batches, spatial coordinates base + ts * [-extent, extent)."""
    g = torch.Generator().manual_seed(seed)
    c = torch.randint(-extent, extent, (n, D), generator=g, dtype=torch.int64) * ts + base
    b = torch.randint(0, 2, (n, 1), generator=g, dtype=torch.int64)
    return torch.cat([b, c], 1).int()


def dyadic(shape, seed, scale):
    """Values k * scale, |k| <= 64: exact in fp32, bf16 and fp16."""
    g = torch.Generator().manual_seed(seed)
    return torch.randint(-64, 65, shape, generator=g).float() * scale


def triples(cm, in_key, out_key, K, **kw):
    kd = cm.kernel_map(in_key, out_key, **kw)
    im = [kd[k][0].numpy().astype(np.int64) if k in kd else np.zeros(0, np.int64) for k in range(K)]
    om = [kd[k][1].numpy().astype(np.int64) if k in kd else np.zeros(0, np.int64) for k in range(K)]
    return O.kernel_map_triples(cm.get_coordinates(in_key).numpy(),
                                cm.get_coordinates(out_key).numpy(), im, om)


def leaf_features(cm, key, cin, seed, distinct=False):
    """Features of map `key` drawn in canonical row order, as a leaf in the map's own row order;
    `distinct`: all different (multiples of 2^-12), so that a max pooling has no ties."""
    c = cm.get_coordinates(key).numpy()
    p = O.lexsort_rows(c)
    f = torch.empty(len(c), cin)
    if distinct:
        g = torch.Generator().manual_seed(seed)
        v = (torch.randperm(len(c) * cin, generator=g) - len(c) * cin // 2).float() * 2.0 ** -12
        f[torch.from_numpy(p)] = v.reshape(len(c), cin)
    else:
        f[torch.from_numpy(p)] = dyadic((len(c), cin), seed, 2.0 ** -7)
    return f.requires_grad_(True), c, p


def case(ME, name, D, n, extent, seed, kind="conv", cin=4, cout=4, ks=3, stride=1, dil=1,
         ts_in=1, region="cube", pre_stride=None, given=None, pool=None, extra_stride=None,
         base=0):
    """One layer.  kind: conv | transpose | generative | pool.  pre_stride: the layer reads the
    map `stride(inserted, pre_stride)` (so that the inserted, finer map exists for a transpose).
    given: None | 'tensor' | 'key' — output coordinates passed to the layer, or 'expand' —
    a forward convolution with expand_coordinates=True.  extra_stride: also
    store the strided map of the inserted one at this stride (coordinates and stride map)."""
    ks_l, st_l, dl_l, ts_l = ([v] * D if np.isscalar(v) else list(v)
                              for v in (ks, stride, dil, ts_in))
    rt = {"cube": ME.RegionType.HYPER_CUBE, "cross": ME.RegionType.HYPER_CROSS}[region]
    torch.manual_seed(seed)
    raw = cloud(n, extent, seed, D, ts_l[0], base)
    cm = ME.CoordinateManager(D=D, coordinate_map_type=ME.CoordinateMapType.CPU)
    key0, (uidx, inv) = cm.insert_and_map(raw, ts_l)
    assert len(uidx) < n, f"{name}: the cloud must hold duplicates"
    out = {"raw_coords": raw.numpy(), "unique_index": uidx.numpy().astype(np.int64),
           "inverse_map": inv.numpy().astype(np.int64)}
    if extra_stride is not None:
        ks_key = cm.stride(key0, extra_stride)
        sc = cm.get_coordinates(ks_key).numpy()
        i, o = cm.stride_map(key0, ks_key)
        c0 = cm.get_coordinates(key0).numpy()
        out["xs_coords"] = O.canonical_rows(sc)[0]
        out["xs_pairs"] = O.kernel_map_triples(c0, sc, [i.numpy().astype(np.int64)],
                                               [o.numpy().astype(np.int64)])[:, 1:].astype(np.int32)
    in_key = key0 if pre_stride is None else cm.stride(key0, pre_stride)
    feats, in_c, in_p = leaf_features(cm, in_key, cin, seed + 1, distinct=kind == "pool")
    x = ME.SparseTensor(feats, coordinate_map_key=in_key, coordinate_manager=cm)
    kg = ME.KernelGenerator(kernel_size=ks_l, stride=st_l, dilation=dl_l, region_type=rt,
                            expand_coordinates=kind == "generative" or given == "expand",
                            dimension=D)
    K = kg.kernel_volume
    w = None
    if kind == "pool":
        layer = {"max": ME.MinkowskiMaxPooling, "avg": ME.MinkowskiAvgPooling}[pool](
            kernel_size=ks_l, stride=st_l, dilation=dl_l, dimension=D)
    else:
        cls = {"conv": ME.MinkowskiConvolution, "transpose": ME.MinkowskiConvolutionTranspose,
               "generative": ME.MinkowskiGenerativeConvolutionTranspose}[kind]
        kw = {"expand_coordinates": True} if given == "expand" else {}
        layer = cls(cin, cout, kernel_generator=kg, dimension=D, **kw)
        w = dyadic(tuple(layer.kernel.shape), seed + 2, 2.0 ** -9)
        with torch.no_grad():
            layer.kernel.copy_(w)
    if given in ("tensor", "key"):
        gc = cloud(n // 2, extent + 3, seed + 3, D)       # partly out of the input's reach
        out["given_coords"] = gc.numpy()
        y = layer(x, gc if given == "tensor" else cm.insert_and_map(gc, 1, "given")[0])
    else:
        y = layer(x)
    out_c = y.C.numpy()
    oc, of, op = O.canonical_rows(out_c, y.F.detach().numpy())
    gout = torch.empty(y.F.shape)
    gout[torch.from_numpy(op)] = dyadic(tuple(y.F.shape), seed + 4, 2.0 ** -7)
    y.F.backward(gout)
    kmap_kw = dict(stride=st_l, kernel_size=ks_l, dilation=dl_l, region_type=rt,
                   is_transpose=kind in ("transpose", "generative"), is_pool=kind == "pool")
    out.update(in_coords=in_c[in_p], in_feats=feats.detach().numpy()[in_p],
               out_coords=oc, out_feats=of, grad_out=gout.numpy()[op],
               grad_in=feats.grad.numpy()[in_p],
               kmap=triples(cm, in_key, y.coordinate_map_key, K, **kmap_kw).astype(np.int32))
    if w is not None:
        out.update(weight=w.numpy(), grad_weight=layer.kernel.grad.numpy())
    meta = {"kind": kind, "D": D, "cin": cin, "cout": cout, "kernel_size": ks_l, "stride": st_l,
            "dilation": dl_l, "ts_in": ts_l, "region": region, "pre_stride": pre_stride,
            "given": given, "pool": pool, "extra_stride": extra_stride, "K": K,
            "out_ts": list(y.tensor_stride)}
    out["meta"] = np.array(json.dumps(meta, sort_keys=True))
    np.savez_compressed(os.path.join(HERE, f"ref_layer_{name}.npz"), **out)
    print(f"{name:24s} K={K:5d} in {len(in_c):5d} -> out {len(oc):5d} pairs {len(out['kmap']):7d}")


def main():
    ME = ref.import_reference()
    # coordinate widths 2 and 6..8 (D = 1, 5, 6, 7), each with its insert and a stride-3 map
    case(ME, "d1_k3s1", 1, 400, 200, 10, cin=16, cout=16, extra_stride=3)
    case(ME, "d1_k2s2", 1, 400, 200, 11, cin=5, cout=7, ks=2, stride=2, extra_stride=3)
    case(ME, "d5_k3s1", 5, 500, 3, 12, cin=3, cout=5, extra_stride=3)          # K = 243
    case(ME, "d5_k2s2", 5, 500, 3, 13, cin=16, cout=16, ks=2, stride=2, extra_stride=3)
    case(ME, "d6_k2s2", 6, 500, 2, 14, cin=16, cout=16, ks=2, stride=2, extra_stride=3)  # K = 64
    case(ME, "d7_k3s1", 7, 150, 1, 15, cin=2, cout=3, extra_stride=3)          # K = 2187
    # coordinates near +-2^30 (the reference strides through float32: every coordinate here is a
    # multiple of the tensor stride 64, so its quotients are exact in float32 as well)
    case(ME, "large_k3s2", 3, 400, 6, 16, cin=8, cout=12, stride=2, ts_in=64,
         base=-(2 ** 30) + 2 ** 10, extra_stride=4)
    case(ME, "large_pos_k3s2", 3, 400, 6, 17, cin=16, cout=16, stride=2, ts_in=64,
         base=2 ** 30 - 2 ** 10, extra_stride=4)
    # kernel shapes
    case(ME, "k315_s1", 3, 400, 6, 20, cin=16, cout=16, ks=[3, 1, 5])
    case(ME, "k231_s212", 3, 400, 6, 21, cin=5, cout=7, ks=[2, 3, 1], stride=[2, 1, 2])
    case(ME, "k2s1", 3, 400, 6, 22, cin=16, cout=16, ks=2)
    case(ME, "k4s1", 3, 400, 6, 23, cin=6, cout=10, ks=4)
    case(ME, "k3s2_dil2", 3, 400, 7, 24, cin=16, cout=16, stride=2, dil=2)
    case(ME, "k3s1_dil123", 3, 400, 7, 25, cin=3, cout=5, dil=[1, 2, 3])
    # inputs at tensor stride 2 and 4 (offsets scale with the input's tensor stride)
    case(ME, "ts2_k3s2", 3, 400, 6, 30, cin=16, cout=16, stride=2, ts_in=2)
    case(ME, "ts2_k3s1", 3, 400, 6, 31, cin=8, cout=12, ts_in=2)
    case(ME, "ts4_k3s2", 3, 400, 6, 32, cin=5, cout=16, stride=2, ts_in=4)
    case(ME, "ts4_k3s1", 3, 400, 6, 33, cin=16, cout=32, ts_in=4)
    # HYPER_CROSS regions at input tensor stride 2
    case(ME, "cross_k5s1_ts2", 3, 400, 6, 40, cin=16, cout=16, ks=5, ts_in=2, region="cross")
    case(ME, "cross_k5s2_ts2", 3, 400, 6, 41, cin=6, cout=7, ks=5, stride=2, ts_in=2,
         region="cross")
    # transposed convolutions onto an existing finer map, and one onto a map made from regions
    case(ME, "tr_k3s2_2to1", 3, 400, 6, 50, kind="transpose", cin=16, cout=16, stride=2,
         pre_stride=2)
    case(ME, "tr_k3s2_4to2", 3, 400, 6, 51, kind="transpose", cin=7, cout=5, stride=2,
         ts_in=2, pre_stride=2)
    case(ME, "tr_k4s2", 3, 400, 6, 52, kind="transpose", cin=16, cout=16, ks=4, stride=2,
         pre_stride=2)
    case(ME, "tr_k313s2", 3, 400, 6, 53, kind="transpose", cin=8, cout=16, ks=[3, 1, 3],
         stride=2, pre_stride=2)
    case(ME, "tr_k3s2_regions", 3, 150, 6, 54, kind="transpose", cin=5, cout=3, stride=2,
         ts_in=2)
    # generative transposes and expanded forward coordinates
    case(ME, "gen_k2s2_4to2", 3, 250, 6, 60, kind="generative", cin=16, cout=16, ks=2, stride=2,
         ts_in=4)
    case(ME, "gen_k3s2_4to2", 3, 150, 4, 61, kind="generative", cin=5, cout=6, stride=2, ts_in=4)
    case(ME, "expand_k3s1", 3, 250, 6, 62, cin=6, cout=5, given="expand")
    case(ME, "expand_k3s2", 3, 250, 6, 63, cin=16, cout=16, stride=2, given="expand")
    # output coordinates given by the caller, as a tensor and as a key
    case(ME, "given_tensor", 3, 400, 6, 70, cin=16, cout=16, given="tensor")
    case(ME, "given_key", 3, 400, 6, 71, cin=6, cout=5, given="key")
    # pooling maps of an input at tensor stride 2.  A dilated window at a strided input can hold
    # no input row at all; the reference's CPU max pooling leaves such a row's max index at -1 and
    # its backward then adds into grad_in[-1] (pooling_max_kernel.hpp:72-115), which corrupts its
    # heap.  So the dilated map is recorded by average pooling; a pooling map does not depend on
    # the mode, and the tests run both modes on both maps.
    case(ME, "maxpool_k2s2_ts2", 3, 400, 6, 80, kind="pool", cin=5, ks=2, stride=2, ts_in=2,
         pool="max")
    case(ME, "avgpool_k3s2_dil2_ts2", 3, 400, 6, 83, kind="pool", cin=16, stride=2, dil=2,
         ts_in=2, pool="avg")


if __name__ == "__main__":
    main()
