"""The stride pyramid enqueued ahead of time (backend._Prediction: device-side row counts,
meb200_insert_and_map_enqueue + meb200_map_build_table) must produce exactly the maps the
blocking path produces — same rows in the same order, same parent links, same kernel maps —
and a wrong prediction must fall back to the blocking path."""
import pytest
import torch

from minkowskiengine_b200 import backend as B

pytestmark = pytest.mark.gpu


def _coords(n, seed, extent=64, dup=True):
    g = torch.Generator().manual_seed(seed)
    c = torch.randint(-extent, extent, (n, 3), generator=g, dtype=torch.int32)
    c = torch.cat([torch.randint(0, 3, (n, 1), generator=g, dtype=torch.int32), c], 1)
    if dup and n > 10:
        c[n // 2:n // 2 + n // 10] = c[:n // 10]          # duplicates: unique count < n
    return c


def _pyramid(ME, coords, strides):
    """-> (manager, [key per level]) after asking for the chain of strided maps."""
    x = ME.SparseTensor(torch.ones(len(coords), 1), coords, device="cuda")
    cm = x.coordinate_manager
    keys = [x.coordinate_map_key]
    for s in strides:
        assert cm.stride(keys[-1], [1] * len(s)) == keys[-1]      # stride-1 layers in between
        keys.append(cm.stride(keys[-1], s))
    return x, cm, keys


def _state(cm, keys):
    m = cm._manager
    out = []
    for a, b in zip(keys[:-1], keys[1:]):
        kb = m._k(b)
        par = m._parents[kb]
        km = m._kernel_map(a, b, [3, 3, 3], [2, 2, 2], [1, 1, 1], ME_HYPER, None, False, False)
        out.append((m._maps[kb].coords.clone(), par[0], par[1].clone(), km.out_nbr.clone(),
                    km.in_nbr.clone()))
    return out


ME_HYPER = None


def _forget_pyramids():
    """Drops every learnt stride pyramid; the kernel-map hints stay, as they do between managers."""
    for h in B._HINTS.values():
        h.pyramid = ()


@pytest.mark.parametrize("n", [1, 37, 5000, 200000])
def test_predicted_pyramid_equals_blocking_path(ME, cuda, n, monkeypatch):
    global ME_HYPER
    ME_HYPER = ME.RegionType.HYPER_CUBE
    coords = _coords(n, seed=n)
    strides = [[2, 2, 2]] * 4
    monkeypatch.setattr(B, "_PREFETCH", False)
    _forget_pyramids()
    _, cm0, k0 = _pyramid(ME, coords, strides)
    assert not cm0._manager._prediction.pending
    want = _state(cm0, k0)
    monkeypatch.setattr(B, "_PREFETCH", True)
    assert B._HINTS[4].pyramid == ((2, 2, 2),) * 4         # learnt from the first manager
    x1, cm1, k1 = _pyramid(ME, coords, strides)
    assert not cm1._manager._prediction.pending            # every level was taken
    got = _state(cm1, k1)
    for lvl, (w, g) in enumerate(zip(want, got)):
        assert torch.equal(w[0], g[0]), f"coordinates differ at level {lvl}"
        assert w[1] == g[1] and torch.equal(w[2], g[2]), f"parent link differs at level {lvl}"
        assert torch.equal(w[3], g[3]) and torch.equal(w[4], g[4]), f"kernel map differs at level {lvl}"


def test_wrong_prediction_falls_back_to_blocking_path(ME, cuda, monkeypatch):
    monkeypatch.setattr(B, "_PREFETCH", True)
    _forget_pyramids()
    B._hint(4).pyramid = ((2, 2, 2), (2, 2, 2))
    coords = _coords(3000, seed=5)
    _, cm, keys = _pyramid(ME, coords, [[3, 3, 3], [2, 2, 2]])      # first request mispredicted
    m = cm._manager
    monkeypatch.setattr(B, "_PREFETCH", False)
    _forget_pyramids()
    _, cm_ref, keys_ref = _pyramid(ME, coords, [[3, 3, 3], [2, 2, 2]])
    for a, b in zip(keys[1:], keys_ref[1:]):
        assert torch.equal(m._maps[m._k(a)].coords, cm_ref._manager._maps[m._k(b)].coords)
    # a 2-D manager is not confused by a 3-D hint
    B._hint(4).pyramid = ((2, 2, 2),)
    monkeypatch.setattr(B, "_PREFETCH", True)
    c2 = _coords(500, seed=1)[:, :3].contiguous()
    x = ME.SparseTensor(torch.ones(500, 1), c2, device="cuda")
    assert cm.stride is not None and x.coordinate_manager.stride(x.coordinate_map_key, [2, 2]) is not None
