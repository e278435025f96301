"""Pins the numpy restatement of global pooling (tests/global_oracle.py), which
tests/test_gpu_field_global.py checks the GPU against, to the compiled reference's pooling of
TensorField points (tests/golden/ref_field_global_*, written by
tests/golden/make_field_global_fixtures.py).  No GPU needed."""
import os

import numpy as np
import pytest

import global_oracle as GO
from helpers import rel_err

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
MODES = {"sum": GO.POOL_SUM, "avg": GO.POOL_AVG, "max": GO.POOL_MAX}


@pytest.mark.parametrize("mode", ["sum", "avg", "max"])
def test_oracle_matches_reference_field_pooling(mode):
    G = np.load(os.path.join(GOLDEN, f"ref_field_global_{mode}.npz"))
    pts, feats = G["pts"], G["feats"]
    assert (pts[:, 0] == np.round(pts[:, 0])).all()        # integer batch values
    coords = np.zeros((len(pts), 4), np.int32)
    coords[:, 0] = pts[:, 0]
    origin, seg = GO.origin_segments(coords)
    assert len(pts) > len(origin) >= 3
    assert (origin == G["out_coords"]).all()
    out, aux = GO.global_pool_forward(feats, seg, len(origin), MODES[mode])
    assert rel_err(out, G["out_feats"]) < 1e-6
    grad = GO.global_pool_backward(G["grad_out"], seg, len(pts), MODES[mode], aux)
    assert rel_err(grad, G["grad_in"]) < 1e-6
