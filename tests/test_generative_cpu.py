"""Host side of pruning, union and non-matching arithmetic without a GPU: map bookkeeping (row
order, union sources, cache), argument validation and the plumbing of the native calls, with the
native library replaced by a recorder and the insert by a restatement of its semantics (first
occurrence wins, rows numbered by first occurrence, invalid rows dropped)."""
import pytest
import torch


def _fake_build(B):
    def build(cand, tensor_stride, valid=None):
        seen, uidx, inv = {}, [], []
        for i, row in enumerate(cand.tolist()):
            if valid is not None and not int(valid[i]):
                inv.append(-1)
                continue
            t = tuple(row)
            if t not in seen:
                seen[t] = len(uidx)
                uidx.append(i)
            inv.append(seen[t])
        uidx = torch.tensor(uidx, dtype=torch.int64)
        coords = cand[uidx] if len(uidx) else cand[:0]
        table = torch.zeros(1024, dtype=torch.int32)
        return (B._CoordinateMap(coords, table, 1024, tensor_stride), uidx,
                torch.tensor(inv, dtype=torch.int64))
    return build


@pytest.fixture
def stub(monkeypatch):
    from minkowskiengine_b200 import _lib, backend as B
    calls = []

    class Stub:
        def __getattr__(self, name):
            def fn(*args):
                calls.append((name, args))
                return 0
            return fn

    monkeypatch.setattr(_lib, "load", lambda: Stub())
    monkeypatch.setattr(_lib, "current_stream", lambda: None)
    monkeypatch.setattr(B._CoordinateMap, "build", staticmethod(_fake_build(B)))
    mgr = B.CoordinateMapManagerGPU_c10()

    def add(name, rows, ts=(1, 1, 1)):
        key = (tuple(ts), name)
        mgr._maps[key] = B._CoordinateMap(torch.tensor(rows, dtype=torch.int32).reshape(-1, 4),
                                          torch.zeros(1024, dtype=torch.int32), 1024, ts)
        return B.CoordinateMapKey(list(ts), name)
    return B, mgr, add, calls


def test_union_map_order_sources_and_cache(stub):
    B, mgr, add, calls = stub
    a = add("a", [[0, 0, 0, 0], [0, 1, 0, 0], [1, 2, 2, 2]])
    b = add("b", [[0, 5, 5, 5], [0, 1, 0, 0]])
    e = add("e", [])
    out = B.CoordinateMapKey(4)
    pairs = mgr.union_map([a, b], out)
    assert out.is_key_set() and out.get_tensor_stride() == [1, 1, 1]
    assert mgr.get_coordinates(out).tolist() == [[0, 0, 0, 0], [0, 1, 0, 0], [1, 2, 2, 2],
                                                 [0, 5, 5, 5]]
    assert [p.tolist() for p in pairs] == [[[0, 1, 2], [0, 1, 2]], [[0, 1], [3, 1]]]
    um = mgr._union([a, b])
    assert um.src.dtype == torch.int32 and um.src.tolist() == [[0, 1, 2, -1], [-1, 1, -1, 0]]
    out2 = B.CoordinateMapKey(4)
    mgr.union_map([a, b], out2)
    assert out2 == out                                     # cached per ordered tuple of keys
    out3 = B.CoordinateMapKey(4)
    mgr.union_map([b, a], out3)
    assert out3 != out
    # a 0-row input contributes nothing
    ue = mgr._union([a, e, b])
    assert ue.M == 4 and ue.sizes == [3, 0, 2] and ue.src[1].tolist() == [-1, -1, -1, -1]


def test_union_rejects_mixed_strides(stub):
    B, mgr, add, calls = stub
    a = add("a", [[0, 0, 0, 0]])
    s = add("s", [[0, 0, 0, 0]], ts=(2, 2, 2))
    with pytest.raises(RuntimeError, match="tensor stride"):
        mgr.union_map([a, s], B.CoordinateMapKey(4))
    with pytest.raises(RuntimeError, match="not found"):
        mgr.union_map([a, B.CoordinateMapKey([1, 1, 1], "missing")], B.CoordinateMapKey(4))


def test_union_fold_plumbing(stub, monkeypatch):
    B, mgr, add, calls = stub
    a = add("a", [[0, 0, 0, 0], [0, 1, 0, 0]])
    b = add("b", [[0, 1, 0, 0], [0, 2, 0, 0], [0, 3, 0, 0]])
    um = mgr._union([a, b])
    fa, fb = torch.randn(2, 8), torch.randn(3, 8)
    with pytest.raises(RuntimeError, match="CUDA"):
        B.union_fold_forward([fa, fb], um, 2)
    monkeypatch.setattr(B, "_check_union_devices", lambda feats: None)
    out = B.union_fold_forward([fa, fb], um, 2)
    assert out.shape == (4, 8)
    name, args = calls[-1]
    assert name == "meb200_union_fold_forward"
    assert args[1:3] == (2, 16) and args[4:8] == (4, 8, 0, 2)        # N, align, M, C, F32, MUL
    calls.clear()
    ga, gb = B.union_fold_backward(torch.randn(4, 8), [fa, fb], um, 3, needs=(True, True))
    assert ga.shape == fa.shape and gb.shape == fb.shape
    assert [c[0] for c in calls] == ["meb200_union_fold_backward"] * 2
    assert [c[1][9] for c in calls] == [0, 1] and [c[1][11] for c in calls] == [2, 3]
    calls.clear()
    ga, gb = B.union_fold_backward(torch.randn(4, 8), [fa, fb], um, 0, needs=(False, True))
    assert ga is None and len(calls) == 1
    with pytest.raises(RuntimeError, match="do not match"):
        B.union_fold_forward([fa, torch.randn(2, 8)], um, 0)
    with pytest.raises(RuntimeError, match="channels"):
        B.union_fold_forward([fa, torch.randn(3, 4)], um, 0)
    with pytest.raises(RuntimeError, match="dtype"):
        B.union_fold_forward([fa, fb.double()], um, 0)


def test_pruned_map_and_validation(stub):
    B, mgr, add, calls = stub
    a = add("a", [[0, 0, 0, 0], [0, 1, 0, 0], [1, 2, 2, 2], [0, 3, 0, 0]])
    keep = torch.tensor([True, False, True, True])
    ok = mgr._prune(a, keep)
    assert ok[0] == (1, 1, 1) and ok != mgr._k(a)
    assert mgr._maps[ok].coords.tolist() == [[0, 0, 0, 0], [1, 2, 2, 2], [0, 3, 0, 0]]
    uidx, inv = mgr._prunes[(mgr._k(a), ok)]
    assert uidx.tolist() == [0, 2, 3] and inv.tolist() == [0, -1, 1, 2]
    assert mgr._prune(a, keep) != ok                      # not cached: a new key every call
    fwd = B.PruningForwardGPU
    f = torch.randn(4, 3)
    key = B.CoordinateMapKey(4)
    with pytest.raises(RuntimeError, match="boolean"):
        fwd(f, keep.float(), a, key, mgr)
    with pytest.raises(RuntimeError, match="keep.dim"):
        fwd(f, keep.view(2, 2), a, key, mgr)
    with pytest.raises(RuntimeError, match="in_feat.dim"):
        fwd(f[:, 0].contiguous(), keep, a, key, mgr)
    with pytest.raises(RuntimeError, match="keep size mismatch"):
        fwd(f, keep[:3], a, key, mgr)
    with pytest.raises(RuntimeError, match="Invalid in_feat size"):
        fwd(f[:3], keep[:3], a, key, mgr)
    with pytest.raises(RuntimeError, match="not found"):
        fwd(f, keep, B.CoordinateMapKey([1, 1, 1], "missing"), key, mgr)
    with pytest.raises(RuntimeError, match="must be CUDA"):
        fwd(f, keep, a, key, mgr)
    assert not key.is_key_set()


def test_modules_are_exported_with_reference_names():
    import minkowskiengine_b200 as ME
    for name in ("MinkowskiPruning", "MinkowskiPruningFunction", "MinkowskiUnion",
                 "MinkowskiUnionFunction"):
        assert hasattr(ME, name), name
    assert callable(ME.backend.PruningForwardGPU) and callable(ME.backend.PruningBackwardGPU)
    assert hasattr(ME.CoordinateManager, "union_map")


def test_completion_net_parameter_count_matches_reference_widths():
    import minkowskiengine_b200 as ME
    from examples.completion import completion_net
    net = completion_net(ME, (8, 16, 32, 64), (8, 16, 32, 64))
    names = [n for n, _ in net.named_parameters()]
    assert "dec_cls.2.bias" in names and "dec_blocks.0.0.kernel" in names
    # the deepest decoder level up-samples with a 4^3 kernel, the others with 2^3
    assert net.dec_blocks[0][0].kernel.shape == (64, 64, 32)
    assert net.dec_blocks[1][0].kernel.shape == (8, 32, 16)
