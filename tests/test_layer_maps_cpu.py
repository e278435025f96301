"""The numpy oracle (oracle/oracle_np.py) against the compiled reference, one layer per fixture
(tests/golden/ref_layer_*.npz, written by tests/golden/make_layer_fixtures.py): the insert, the
strided, region and caller-given output coordinates, the kernel map as (k, in coordinate, out
coordinate) triples, and the float64 features and gradients within 1e-5 relative.

The fixtures cover what the other reference fixtures leave out: coordinate widths 2 and 6..8,
coordinates near 2^30, non-cubic, per-axis, even and dilated kernels, inputs at tensor stride 2
and 4, HYPER_CROSS regions, transposed and generative layers, expanded and caller-given output
coordinates, and pooling maps.  The oracle's offset tables restate `kernel_generator`'s, so a
convention error shared by both (offset order, centring, which tensor stride scales the offsets,
the transposed direction, the aligned-only filter) fails here first, on a machine without a GPU."""
import glob
import json
import os

import numpy as np
import pytest

from helpers import layer_out_ts
from oracle import oracle_np as O

GOLD = os.path.join(os.path.dirname(__file__), "golden")
FIXTURES = sorted(glob.glob(os.path.join(GOLD, "ref_layer_*.npz")))
REGION = {"cube": O.HYPER_CUBE, "cross": O.HYPER_CROSS}


def _id(path):
    return os.path.basename(path)[len("ref_layer_"):-len(".npz")]


def load(path):
    f = np.load(path)
    return f, json.loads(str(f["meta"]))


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30)) if b.size else 0.0


def oracle_layer(f, m):
    """The oracle's (in coordinates, in tensor stride, out coordinates, out tensor stride,
    in_maps, out_maps) of the fixture's layer, from its inserted coordinates alone."""
    D, ts = m["D"], m["ts_in"]
    ui, _ = O.insert_and_map(f["raw_coords"])
    inserted = f["raw_coords"][ui]
    if m["pre_stride"] is not None:
        in_c, in_ts = O.stride_map_coords(inserted, ts, [m["pre_stride"]] * D)
    else:
        in_c, in_ts = O.unique_rows(inserted), list(ts)
    ks, st, dl, rt = m["kernel_size"], m["stride"], m["dilation"], REGION[m["region"]]
    if m["kind"] in ("transpose", "generative"):
        out_ts = [t // s for t, s in zip(in_ts, st)]
        offs = O.region_offsets(rt, ks, dl, out_ts)
        if m["kind"] == "transpose" and m["pre_stride"] is not None:
            out_c = O.unique_rows(inserted)          # the finer map exists: the inserted one
        else:
            out_c = O.stride_region_coords(in_c, offs, out_ts, is_transpose=True)
        im, om = O.transposed_kernel_map(in_c, out_c, offs)
        return in_c, in_ts, out_c, out_ts, im, om
    out_ts = [t * s for t, s in zip(in_ts, st)]
    if m["given"] in ("tensor", "key"):
        out_c, out_ts = O.unique_rows(f["given_coords"]), [1] * D
    elif m["given"] == "expand":
        out_c = O.stride_region_coords(in_c, O.region_offsets(rt, ks, dl, in_ts), out_ts,
                                       is_transpose=False)
    else:
        out_c, _ = O.stride_map_coords(in_c, in_ts, st)
    if m["kind"] == "pool" and ks == st:
        im, om = O.stride_map(in_c, out_c, out_ts)
    else:
        im, om = O.kernel_map(in_c, out_c, O.region_offsets(rt, ks, dl, in_ts))
    return in_c, in_ts, out_c, out_ts, im, om


@pytest.mark.parametrize("path", FIXTURES, ids=_id)
def test_insert_and_strides(path):
    f, m = load(path)
    ui, inv = O.insert_and_map(f["raw_coords"])
    assert np.array_equal(ui, f["unique_index"]) and np.array_equal(inv, f["inverse_map"])
    if m["extra_stride"] is not None:
        c0 = f["raw_coords"][ui]
        sc, _ = O.stride_map_coords(c0, m["ts_in"], [m["extra_stride"]] * m["D"])
        assert np.array_equal(sc, f["xs_coords"])
        im, om = O.stride_map(c0, sc, [t * m["extra_stride"] for t in m["ts_in"]])
        pairs = O.kernel_map_triples(c0, sc, im, om)[:, 1:]
        assert np.array_equal(pairs, f["xs_pairs"])


@pytest.mark.parametrize("path", FIXTURES, ids=_id)
def test_layer_map(path):
    f, m = load(path)
    in_c, _, out_c, out_ts, im, om = oracle_layer(f, m)
    assert np.array_equal(in_c, f["in_coords"])
    assert out_ts == layer_out_ts(m)
    assert out_c.shape == f["out_coords"].shape and np.array_equal(out_c, f["out_coords"])
    if m["kind"] == "pool" and m["kernel_size"] == m["stride"]:
        assert np.array_equal(im[0], np.arange(len(in_c)))    # every input row has its parent
    tri = O.kernel_map_triples(in_c, out_c, im, om)
    assert tri.shape == f["kmap"].shape and np.array_equal(tri, f["kmap"])


@pytest.mark.parametrize("path", FIXTURES, ids=_id)
def test_layer_features(path):
    f, m = load(path)
    _, _, out_c, _, im, om = oracle_layer(f, m)
    if m["kind"] == "pool":
        mode = {"max": O.POOL_MAX, "avg": O.POOL_AVG}[m["pool"]]
        y, aux = O.pool_forward(f["in_feats"], im, om, len(out_c), mode)
        gi = O.pool_backward(f["grad_out"], len(f["in_feats"]), im, om, mode, aux)
        assert _rel(y, f["out_feats"]) < 1e-5 and _rel(gi, f["grad_in"]) < 1e-5
        return
    y = O.conv_forward(f["in_feats"], f["weight"], im, om, len(out_c))
    gi, gw = O.conv_backward(f["in_feats"], f["grad_out"], f["weight"], im, om)
    assert _rel(y, f["out_feats"]) < 1e-5
    assert _rel(gi, f["grad_in"]) < 1e-5
    assert _rel(gw, f["grad_weight"]) < 1e-5
    if m["given"] in ("tensor", "key"):
        reached = np.zeros(len(out_c), bool)
        for o in om:
            reached[o] = True
        assert (~reached).any() and not f["out_feats"][~reached].any(), \
            "given rows out of the input's reach must exist and be zero"


def test_fixture_coverage():
    """Every group of layer shapes has a fixture, and each convolution group has a layer on the
    16-channel grid (the tensor-core route in bf16 / fp16) and one off it."""
    metas = {_id(p): load(p)[1] for p in FIXTURES}
    assert {m["D"] for m in metas.values()} >= {1, 5, 6, 7}
    groups = {"d": lambda n: n[0] == "d" and n[1].isdigit(), "large": lambda n: "large" in n,
              "k": lambda n: n[0] == "k", "ts": lambda n: n.startswith("ts"),
              "cross": lambda n: "cross" in n, "tr": lambda n: n.startswith("tr_"),
              "gen": lambda n: n.startswith(("gen", "expand")),
              "given": lambda n: n.startswith("given")}
    for g, sel in groups.items():
        grid = [m["cin"] % 16 == 0 and m["cout"] % 16 == 0
                for n, m in metas.items() if sel(n)]
        assert any(grid) and not all(grid), g
