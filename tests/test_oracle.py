"""CPU tests pinning the numpy oracle (oracle/oracle_np.py):
  1. against the reference's own golden vectors (tests/golden/reference_goldens.json,
     transcribed from the reference's tests, file:line in each entry);
  2. against outputs of the compiled reference stored as fixtures (tests/golden/ref_*.npz,
     produced by tests/golden/make_fixtures.py);
  3. against one strided convolution of the compiled reference on seeded inputs
     (tests/golden/ref_live_conv.npz, produced by tests/golden/make_reference_runs.py)."""
import glob
import json
import os

import numpy as np
import pytest

from oracle import oracle_np as O

GOLD = os.path.join(os.path.dirname(__file__), "golden")
G = json.load(open(os.path.join(GOLD, "reference_goldens.json")))


@pytest.mark.parametrize("case", G["kernel_region"], ids=lambda c: c["source"].split(" ")[-1])
def test_kernel_region_goldens(case):
    D = len(case["kernel_size"])
    regions = O.region_coordinates(case["coordinates"], O.HYPER_CUBE, case["kernel_size"],
                                   [1] * D, [1] * D)
    assert len(regions) == case["count"]
    assert regions[:len(case["first_regions"])] == case["first_regions"]


@pytest.mark.parametrize("case", G["stride_map_size"], ids=lambda c: c["source"].split(":")[-1])
def test_stride_map_size_goldens(case):
    D = len(case["stride"])
    out, ts = O.stride_map_coords(np.array(case["coordinates"], np.int32), [1] * D, case["stride"])
    assert len(out) == case["size"] and ts == case["tensor_stride"]


def test_batch_find_golden():
    c = G["batch_find"]
    ui, _ = O.insert_and_map(np.array(c["coordinates"], np.int32))
    uniq = np.array(c["coordinates"], np.int32)[ui]
    valid, val = O.map_find(uniq, np.array(c["queries"], np.int32))
    assert valid.tolist() == c["valid_query_index"] and val.tolist() == c["query_value"]


def test_negative_stride_golden():
    c = G["negative_stride"]
    out, _ = O.stride_map_coords(np.array(c["coordinates"], np.int32), [1], c["stride"])
    assert len(out) == c["size"]
    have = {tuple(r) for r in out.tolist()}
    for m in c["must_contain"]:
        assert tuple(m) in have


def test_insert_unique_golden():
    c = G["insert_unique"]
    ui, inv = O.insert_and_map(np.array(c["coordinates"], np.int32))
    assert ui.tolist() == c["unique_index"] and inv.tolist() == c["inverse_map"]
    coords = np.array(c["coordinates"], np.int32)
    assert (coords[ui][inv] == coords).all()


def test_hyper_cross_offsets():
    offs = O.region_offsets(O.HYPER_CROSS, [3, 3, 3], [1, 1, 1], [2, 2, 2]).tolist()
    assert offs[0] == [0, 0, 0] and len(offs) == 7
    assert offs[1:3] == [[2, 0, 0], [-2, 0, 0]] and offs[5:7] == [[0, 0, 2], [0, 0, -2]]


# ---- fixtures produced by the compiled reference -------------------------------------------
CONV_FIX = sorted(glob.glob(os.path.join(GOLD, "ref_conv_*.npz")))
CONV_FIX = [f for f in CONV_FIX if "transpose" not in f]


@pytest.mark.parametrize("path", CONV_FIX, ids=lambda p: os.path.basename(p)[9:-4])
def test_oracle_matches_reference_conv_fixture(path):
    f = np.load(path)
    D, cin, cout, ks, stride = f["meta"].tolist()
    # dedup semantics: first occurrence wins, numbered by rank of first occurrence
    ui, inv = O.insert_and_map(f["raw_coords"])
    assert (f["raw_coords"][ui] == f["in_coords"]).all()
    assert np.array_equal(f["raw_feats"][ui], f["in_feats"])
    out_c, ts = O.stride_map_coords(f["in_coords"], [1] * D, [stride] * D)
    assert out_c.shape == f["out_coords"].shape and (out_c == f["out_coords"]).all()
    offs = O.region_offsets(O.HYPER_CUBE, [ks] * D, [1] * D, [1] * D)
    im, om = O.kernel_map(f["in_coords"], out_c, offs)
    tri = O.kernel_map_triples(f["in_coords"], out_c, im, om)
    assert tri.shape == f["kmap"].shape and (tri == f["kmap"]).all()      # bit-exact index pairs
    out = O.conv_forward(f["in_feats"], f["weight"], im, om, len(out_c))
    assert np.abs(out - f["out_feats"]).max() / np.abs(f["out_feats"]).max() < 1e-5
    gi, gw = O.conv_backward(f["in_feats"], f["grad_out"], f["weight"], im, om)
    assert np.abs(gi - f["grad_in"]).max() / np.abs(f["grad_in"]).max() < 1e-5
    assert np.abs(gw - f["grad_weight"]).max() / np.abs(f["grad_weight"]).max() < 1e-5


@pytest.mark.parametrize("path", sorted(glob.glob(os.path.join(GOLD, "ref_pool_*.npz"))),
                         ids=lambda p: os.path.basename(p)[9:-4])
def test_oracle_matches_reference_pool_fixture(path):
    f = np.load(path)
    ks, stride, mode = f["meta"].tolist()
    D = 3
    out_c, _ = O.stride_map_coords(f["in_coords"], [1] * D, [stride] * D)
    assert (out_c == f["out_coords"]).all()
    if ks == stride:
        im, om = O.stride_map(f["in_coords"], out_c, [stride] * D)
    else:
        im, om = O.kernel_map(f["in_coords"], out_c, O.region_offsets(O.HYPER_CUBE, [ks] * D, [1] * D, [1] * D))
    out, aux = O.pool_forward(f["in_feats"], im, om, len(out_c), mode)
    assert np.abs(out - f["out_feats"]).max() < 1e-5
    gi = O.pool_backward(f["grad_out"], len(f["in_coords"]), im, om, mode, aux)
    assert np.abs(gi - f["grad_in"]).max() < 1e-5


def test_oracle_matches_reference_transpose_fixture():
    f = np.load(os.path.join(GOLD, "ref_conv_transpose_pair.npz"))
    D = 3
    in_c = f["in_coords"]
    mid_c, _ = O.stride_map_coords(in_c, [1] * D, [2] * D)
    offs = O.region_offsets(O.HYPER_CUBE, [2] * D, [1] * D, [1] * D)
    im, om = O.kernel_map(in_c, mid_c, offs)
    mid = O.conv_forward(f["in_feats"], f["w_down"], im, om, len(mid_c))
    imt, omt = O.transposed_kernel_map(mid_c, in_c, offs)
    out = O.conv_forward(mid, f["w_up"], imt, omt, len(in_c))
    assert np.abs(out - f["out_feats"]).max() / np.abs(f["out_feats"]).max() < 1e-5
    gmid, gw_up = O.conv_backward(mid, f["grad_out"], f["w_up"], imt, omt)
    gin, gw_dn = O.conv_backward(f["in_feats"], gmid, f["w_down"], im, om)
    for a, b in ((gw_up, f["grad_w_up"]), (gw_dn, f["grad_w_down"]), (gin, f["grad_in"])):
        assert np.abs(a - b).max() / np.abs(b).max() < 1e-5


def test_oracle_live_against_compiled_reference():
    """One strided convolution of the compiled reference on seeded inputs (stored in
    tests/golden/ref_live_conv.npz by tests/golden/make_reference_runs.py)."""
    f = np.load(os.path.join(GOLD, "ref_live_conv.npz"))
    oc, _ = O.stride_map_coords(f["in_coords"], [1, 1, 1], [2, 2, 2])
    assert (O.unique_rows(f["out_coords"]) == oc).all()
    im, om = O.kernel_map(f["in_coords"], f["out_coords"], O.region_offsets(O.HYPER_CUBE, [3] * 3, [1] * 3, [1] * 3))
    ref_out = O.conv_forward(f["in_feats"], f["kernel"], im, om, len(f["out_coords"]))
    assert np.abs(ref_out - f["out_feats"]).max() < 1e-5
