"""CPU tests of the host side: the C-ABI library exports what include/meb200.h declares, the
key / kernel-generator logic mirrors the reference, and the product path refuses CPU tensors
loudly (there is no fallback)."""
import ctypes
import os
import re
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    import minkowskiengine_b200 as ME
    header = open(os.path.join(ROOT, "include", "meb200.h")).read()
    declared = set(re.findall(r"\b(meb200_[a-z0-9_]+)\s*\(", header))
    assert declared, "no declarations parsed"
    assert os.path.isfile(ME._lib.LIB_PATH), "libmeb200.so missing: run __graft_entry__.build()"
    lib = ctypes.CDLL(ME._lib.LIB_PATH)
    for name in sorted(declared):
        assert hasattr(lib, name), f"{name} declared in include/meb200.h but not exported"
    assert declared == set(ME._lib.PROTOTYPES), "ctypes prototypes out of sync with the header"
    assert ME._lib.load().meb200_build_arch() == b"sm_90a"


def test_library_pure_helpers_without_gpu():
    import minkowskiengine_b200 as ME
    lib = ME._lib.load()
    cap = lib.meb200_hash_capacity(100000)
    assert cap >= 200000 and cap & (cap - 1) == 0
    assert lib.meb200_insert_scratch_bytes(1000) >= 8000
    assert lib.meb200_launch_count() == 0 or lib.meb200_launch_count() > 0
    assert lib.meb200_conv_workspace_bytes(10, 10, 64, 128, 27, ME._lib.F32) == 0
    assert lib.meb200_conv_workspace_bytes(10, 10, 64, 128, 27, ME._lib.BF16) >= 27 * 64 * 128 * 2
    # the SIMT weight gradients keep their row splits' partial sums in the workspace, in any
    # dtype: the MinkUNet head (96 -> 20, K = 1) and a stem (3 -> 20, K = 125) at 200k rows
    for dt in (ME._lib.F32, ME._lib.BF16, ME._lib.F16):
        assert lib.meb200_conv_workspace_bytes(0, 200000, 96, 20, 1, dt) >= 2 * 96 * 20 * 4
        assert lib.meb200_conv_workspace_bytes(0, 200000, 3, 20, 125, dt) >= 2 * 125 * 3 * 20 * 4


def test_coordinate_map_key_semantics():
    import minkowskiengine_b200 as ME
    k = ME.CoordinateMapKey(4)
    assert not k.is_key_set() and k.get_coordinate_size() == 4
    with pytest.raises(RuntimeError):
        k.get_key()
    k.set_key([2, 2, 2], "")
    assert k.is_key_set() and k.get_tensor_stride() == [2, 2, 2] and k.get_key() == ([2, 2, 2], "")
    assert k == ME.CoordinateMapKey([2, 2, 2], "") and k != ME.CoordinateMapKey([2, 2, 2], "a")
    assert hash(k) == hash(ME.CoordinateMapKey([2, 2, 2], ""))
    assert "coordinate map key:[2, 2, 2]" in repr(k)
    with pytest.raises(RuntimeError):
        ME.CoordinateMapKey(3).set_key([1, 1, 1], "")     # wrong dimension


def test_kernel_generator_matches_reference_enumeration():
    import json
    import minkowskiengine_b200 as ME
    from minkowskiengine_b200.kernel_generator import region_offsets
    gold = json.load(open(os.path.join(ROOT, "tests", "golden", "reference_goldens.json")))
    for case in gold["kernel_region"]:
        D = len(case["kernel_size"])
        offs = region_offsets(ME.RegionType.HYPER_CUBE, case["kernel_size"], [1] * D, [1] * D)
        regions = [[c[0]] + [a + b for a, b in zip(c[1:], d)] for c in case["coordinates"] for d in offs]
        assert regions[:len(case["first_regions"])] == case["first_regions"], case["source"]
    kg = ME.KernelGenerator(kernel_size=3, stride=2, dimension=3)
    assert kg.kernel_volume == 27 and kg.kernel_stride == [2, 2, 2]
    assert not kg.requires_strided_coordinates            # (sic) True iff stride == 1
    assert ME.KernelGenerator(kernel_size=1, stride=1, dimension=3).requires_strided_coordinates
    cross = ME.KernelGenerator(kernel_size=3, region_type=ME.RegionType.HYPER_CROSS, dimension=3)
    assert cross.kernel_volume == 7
    # dilation and tensor stride scale the offsets
    assert region_offsets(ME.RegionType.HYPER_CUBE, [3], [2], [4]) == [[-8], [0], [8]]
    assert region_offsets(ME.RegionType.HYPER_CUBE, [2], [1], [4]) == [[0], [4]]


def test_layer_parameter_shapes_match_reference():
    import minkowskiengine_b200 as ME
    c = ME.MinkowskiConvolution(3, 8, kernel_size=5, dimension=3)
    assert tuple(c.kernel.shape) == (125, 3, 8) and c.bias is None
    c1 = ME.MinkowskiConvolution(8, 4, kernel_size=1, bias=True, dimension=3)
    assert c1.use_mm and tuple(c1.kernel.shape) == (8, 4) and tuple(c1.bias.shape) == (1, 4)
    c2 = ME.MinkowskiConvolution(8, 4, kernel_size=1, stride=2, dimension=3)
    assert not c2.use_mm and tuple(c2.kernel.shape) == (1, 8, 4)
    t = ME.MinkowskiConvolutionTranspose(8, 4, kernel_size=2, stride=2, dimension=3)
    assert t.is_transpose and tuple(t.kernel.shape) == (8, 8, 4)
    assert set(dict(c.named_parameters())) == {"kernel"}


def test_cpu_tensors_are_rejected_loudly():
    """No CPU backend and no silent fallback: the product path must raise."""
    import minkowskiengine_b200 as ME
    coords = torch.zeros((4, 4), dtype=torch.int32)
    feats = torch.rand(4, 3)
    with pytest.raises(RuntimeError, match="CUDA"):
        ME.SparseTensor(feats, coords)
    with pytest.raises(RuntimeError, match="CUDA"):
        ME.CoordinateManager(D=3, coordinate_map_type=ME.CoordinateMapType.CPU)
    if not torch.cuda.is_available():
        mgr = ME.CoordinateManager(D=3)
        with pytest.raises(RuntimeError):
            mgr.insert_and_map(coords)


def test_product_package_never_imports_the_oracle():
    """The oracle is test infrastructure: no source file of the product package may import,
    open or execute anything under oracle/ (doc comments stating exactly that are fine)."""
    pkg = os.path.join(ROOT, "minkowskiengine_b200")
    pat = re.compile(r"^\s*(from\s+oracle|import\s+oracle)|oracle[/.](oracle_np|ref|build_ref|_ref)")
    for dirpath, _, files in os.walk(pkg):
        for fn in files:
            if fn.endswith((".py", ".cu", ".cuh", ".h")):
                for ln in open(os.path.join(dirpath, fn)).read().splitlines():
                    assert not pat.search(ln), (fn, ln)


def test_minkunet_definition_parameter_count():
    import minkowskiengine_b200 as ME
    from examples.minkunet import minkunet
    net = minkunet("MinkUNet34C", ME, 3, 20, 3)
    assert sum(p.numel() for p in net.parameters()) == 37_856_052   # SURVEY.md §2 probe count
    assert sum(1 for m in net.modules() if isinstance(m, ME.MinkowskiBatchNorm)) == 62


def test_convert_sync_batchnorm_keeps_sync_holder():
    """reference MinkowskiNormalization.py:123-192: every MinkowskiBatchNorm becomes a
    MinkowskiSyncBatchNorm whose parameter holder is a torch SyncBatchNorm sharing the
    original affine parameters and running statistics."""
    import torch
    import minkowskiengine_b200 as ME
    net = torch.nn.Sequential(ME.MinkowskiBatchNorm(8), torch.nn.Sequential(ME.MinkowskiBatchNorm(16)))
    w0 = net[0].bn.weight
    out = ME.MinkowskiSyncBatchNorm.convert_sync_batchnorm(net)
    bns = [m for m in out.modules() if isinstance(m, ME.MinkowskiBatchNorm)]
    assert len(bns) == 2 and all(isinstance(m, ME.MinkowskiSyncBatchNorm) for m in bns)
    assert all(isinstance(m.bn, torch.nn.SyncBatchNorm) for m in bns)
    assert out[0].bn.weight is w0 and out[1][0].bn.num_features == 16


def test_bench_nvml_clock_sampler_with_a_stub(monkeypatch):
    """bench.py's NVML sampler: median SM clock of the samples taken inside the region, the
    union of the clock-event reason bits, and a clean `False` when NVML is missing."""
    import importlib.util
    import time
    import types
    spec = importlib.util.spec_from_file_location("bench_mod", os.path.join(ROOT, "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    fake = types.ModuleType("pynvml")
    fake.NVML_CLOCK_SM = 1
    fake.nvmlInit = lambda: None
    fake.nvmlDeviceGetHandleByIndex = lambda i: ("h", i)
    fake.nvmlDeviceGetMaxClockInfo = lambda h, c: 1965
    clocks = iter([1000] + [1950] * 1000)
    fake.nvmlDeviceGetClockInfo = lambda h, c: next(clocks)
    fake.nvmlDeviceGetCurrentClocksEventReasons = lambda h: 0x4 | 0x1     # power cap + idle bit
    monkeypatch.setitem(sys.modules, "pynvml", fake)
    s = bench.NvmlClockSampler(0, period_s=0.005)
    assert s.start() is True
    time.sleep(0.1)
    out = s.stop()
    assert out["sm_mhz"] == 1950.0 and out["sm_max_mhz"] == 1965.0 and out["samples"] >= 3
    assert out["reasons"] == ["sw_power_cap"] and out["source"] == "nvml"
    broken = types.ModuleType("pynvml")
    monkeypatch.setitem(sys.modules, "pynvml", broken)       # no nvmlInit -> AttributeError
    assert bench.NvmlClockSampler(0).start() is False


def test_argument_errors_carry_location_condition_and_values():
    """Argument checks run before any CUDA call, so they can be exercised without a GPU: the
    message names the source location, the failed condition and the offending value."""
    from minkowskiengine_b200 import _lib
    lib = _lib.load()
    ts = (ctypes.c_int32 * 3)(2, 2, 2)
    rc = lib.meb200_stride_coords(None, 5, 1, ts, None, None)       # ncols = 1 is invalid
    assert rc != 0
    msg = lib.meb200_last_error().decode()
    assert "coords.cu" in msg and "ncols >= 2" in msg and msg.rstrip().endswith("ncols=1"), msg
    rc = lib.meb200_bn_backward_reduce_peer(None, None, None, 1, 4, 32, None, None, None, None,
                                            1024, 1, 0, 2, None, None, None, None)
    assert rc != 0 and "null buffer" in lib.meb200_last_error().decode()
    with pytest.raises(_lib.BackendError):
        _lib.check(rc)


def test_batchnorm_host_path_runs_against_a_stub_library(monkeypatch):
    """Drives `_BatchNormFunction` forward + backward (the single-GPU path and the NCCL-style
    synchronised path with a fake process group) with the native library replaced by a recorder:
    checks the call sequence and argument plumbing of the Python host, not the kernels."""
    import minkowskiengine_b200 as ME
    from minkowskiengine_b200 import _lib, normalization as N

    calls = []

    class Stub:
        def __getattr__(self, name):
            def fn(*args):
                calls.append((name, args))
                return 0
            return fn

    monkeypatch.setattr(_lib, "load", lambda: Stub())
    monkeypatch.setattr(_lib, "current_stream", lambda: None)
    monkeypatch.setattr(N, "_USE_PEER", False)
    N._WORKSPACES.clear()
    x = torch.randn(10, 16, requires_grad=True)
    w, b = torch.ones(16, requires_grad=True), torch.zeros(16, requires_grad=True)
    rm, rv = torch.zeros(16), torch.ones(16)
    y = N._BatchNormFunction.apply(x, w, b, rm, rv, 0.1, 1e-5, None, False, None, False)
    y.sum().backward()
    names = [c[0] for c in calls]
    # one workspace query, then two launches-worth of calls per pass
    assert names == ["meb200_bn_workspace_bytes", "meb200_bn_forward_train",
                     "meb200_bn_backward_reduce_to", "meb200_bn_backward_apply_fused"]
    assert calls[3][1][11] is None                                   # no device-side count
    assert calls[1][1][6] is None and calls[1][1][7] == 0            # no residual, no ReLU
    assert calls[2][1][2] is None and calls[3][1][13] is None        # no ReLU mask, no d_residual
    assert calls[2][1][10] is not None and calls[2][1][11] is not None   # fp32 parameter gradients
    assert x.grad.shape == x.shape and w.grad.shape == (16,) and b.grad.shape == (16,)
    # fused tail of a residual block: relu(bn(x) + residual), gradient of the residual returned
    calls.clear()
    x3 = torch.randn(10, 16, requires_grad=True)
    res = torch.randn(10, 16, requires_grad=True)
    y3 = N._BatchNormFunction.apply(x3, w, b, rm, rv, 0.1, 1e-5, None, True, res, False)
    y3.sum().backward()
    assert [c[0] for c in calls] == ["meb200_bn_forward_train", "meb200_bn_backward_reduce_to",
                                     "meb200_bn_backward_apply_fused"]
    assert calls[0][1][6] is not None and calls[0][1][7] == 1
    assert calls[1][1][2] is not None and calls[2][1][2] is not None and calls[2][1][13] is not None
    assert res.grad is not None and res.grad.shape == res.shape
    # inference under autograd: running statistics, no statistics pass, gradients still flow
    calls.clear()
    x4 = torch.randn(10, 16, requires_grad=True)
    y4 = N._BatchNormFunction.apply(x4, w, b, rm, rv, 0.1, 1e-5, None, False, None, True)
    y4.sum().backward()
    assert [c[0] for c in calls] == ["meb200_bn_apply_fused", "meb200_bn_backward_reduce_to",
                                     "meb200_bn_backward_apply_fused"]
    assert x4.grad is not None
    # synchronised: the count travels with the sums and is read on the device
    calls.clear()
    reduced = []
    monkeypatch.setattr(torch.distributed, "all_reduce", lambda t, group=None: reduced.append(t.numel()))
    x2 = torch.randn(10, 16, requires_grad=True)
    y2 = N._BatchNormFunction.apply(x2, w, b, rm, rv, 0.1, 1e-5, object(), False, None, False)
    y2.sum().backward()
    assert reduced == [2 * 16 + 1, 2 * 16]
    assert [c[0] for c in calls] == ["meb200_bn_stats_to", "meb200_bn_finalize", "meb200_bn_apply_fused",
                                     "meb200_bn_backward_reduce_to", "meb200_bn_backward_apply_fused"]
    assert calls[1][1][2] is not None and calls[4][1][11] is not None
    assert isinstance(ME.MinkowskiSyncBatchNorm(16).bn, torch.nn.SyncBatchNorm)


def test_pack_table_bookkeeping_against_a_stub_library(monkeypatch):
    """backend._PackTable (one batched re-pack launch for every registered kernel) driven with CPU
    tensors and the native library replaced by a recorder: first sight packs a kernel alone and
    registers it; a stale registered kernel triggers ONE batched call that refreshes every entry;
    dead and re-allocated tensors leave the job table."""
    import ctypes
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
    monkeypatch.setattr(B, "_PACK_BATCHED", True)
    B._PACKED.clear()
    B._PACK_TABLES.clear()
    dtype = torch.bfloat16
    ks = [torch.nn.Parameter(torch.randn(27, 32, 64)), torch.nn.Parameter(torch.randn(8, 5, 7)),
          torch.nn.Parameter(torch.randn(1, 96, 96))]
    for k in ks:
        p = B._packed_weights(k, dtype)
        assert p[0].shape == k.shape and p[1].shape == (k.shape[0], k.shape[2], k.shape[1])
    assert [c[0] for c in calls] == ["meb200_conv_pack_weights"] * 3
    assert all(len(B._packed_weights(k, dtype)) == 2 for k in ks)         # no permuted copies built
    assert all(c[1][7] is None and c[1][8] is None for c in calls)
    tbl = B._PACK_TABLES[(None, dtype)]
    assert len(tbl.entries) == 3 and tbl.jobs_dev is None                  # table built lazily
    calls.clear()
    for k in ks:                                                           # all fresh: no calls at all
        B._packed_weights(k, dtype)
    assert calls == []
    with torch.no_grad():
        for k in ks:
            k.add_(1.0)                                                    # the optimizer stepped
    B._packed_weights(ks[2], dtype)
    assert [c[0] for c in calls] == ["meb200_conv_pack_weights_batched"]
    _, n_jobs, total_tiles = calls[0][1][0], calls[0][1][1], calls[0][1][2]
    assert n_jobs == 3 and total_tiles == 27 * 1 * 2 + 8 * 1 * 1 + 1 * 3 * 3
    jobs = (B._PackJob * 3).from_buffer_copy(bytes(tbl.jobs_dev.numpy().tobytes()))
    assert [j.tile_begin for j in jobs] == [0, 54, 62] and [j.K for j in jobs] == [27, 8, 1]
    assert all(j.w_cp is None and j.w_tp is None for j in jobs) and jobs[0].w == ks[0].data_ptr()
    assert ctypes.sizeof(B._PackJob) == 56
    calls.clear()
    for k in ks:                                                           # every entry was refreshed
        B._packed_weights(k, dtype)
    assert calls == []
    # one tensor dies, one moves: the next batched call sees a rebuilt table without them
    moved = ks[1]
    dead_id = id(ks[0])
    del ks[0]
    import gc
    gc.collect()
    with torch.no_grad():
        moved.data = moved.data.clone()
        ks[1].add_(1.0)
    B._packed_weights(moved, dtype)                # re-allocated: first sight again (packed alone)
    B._packed_weights(ks[1], dtype)                # stale registered kernel: batched
    names = [c[0] for c in calls]
    assert names == ["meb200_conv_pack_weights", "meb200_conv_pack_weights_batched"]
    assert calls[1][1][1] == 2 and dead_id not in tbl.entries


def test_lazy_reverse_table_does_not_keep_the_manager_alive(monkeypatch):
    """A kernel map of a large kernel (K >= 64) defers its reverse neighbour table; the deferred
    build must work and must not tie the manager into a reference cycle (its tables would then
    outlive the tensors until a cyclic garbage collection)."""
    import gc
    import weakref
    from minkowskiengine_b200 import _lib, backend as B

    class Stub:
        def __getattr__(self, name):
            return lambda *a: 0

    monkeypatch.setattr(_lib, "load", lambda: Stub())
    monkeypatch.setattr(_lib, "current_stream", lambda: None)
    mgr = B.CoordinateMapManagerGPU_c10()
    coords = torch.zeros((10, 4), dtype=torch.int32)
    cmap = B._CoordinateMap(coords, torch.zeros(64, dtype=torch.int32), 64, (1, 1, 1))
    mgr._maps[((1, 1, 1), "")] = cmap
    key = B.CoordinateMapKey([1, 1, 1], "")
    km = mgr._kernel_map(key, key, [5, 5, 5], [1, 1, 1], [1, 1, 1], B.RegionType.HYPER_CUBE, None,
                         False, False)
    assert km.K == 125 and km._in_nbr is None and km.n_in == 10          # reverse table deferred
    rev = km.in_nbr                                                        # built on demand
    assert rev.shape == (125, 10) and int((rev == -1).sum()) == 1250 and km._in_thunk is None
    km2 = mgr._kernel_map(key, key, [5, 5, 5], [1, 1, 1], [1, 1, 1], B.RegionType.HYPER_CUBE, None,
                          False, False)
    assert km2 is km
    small = mgr._kernel_map(key, key, [3, 3, 3], [1, 1, 1], [1, 1, 1], B.RegionType.HYPER_CUBE,
                            None, False, False)
    assert small._in_nbr is not None                                       # K = 27: built eagerly
    # a fresh manager with an UNBUILT deferred table dies by reference counting alone
    gc.disable()
    try:
        mgr2 = B.CoordinateMapManagerGPU_c10()
        mgr2._maps[((1, 1, 1), "")] = cmap
        mgr2._kernel_map(key, key, [5, 5, 5], [1, 1, 1], [1, 1, 1], B.RegionType.HYPER_CUBE, None,
                         False, False)
        ref = weakref.ref(mgr2)
        del mgr2
        assert ref() is None, "the manager is kept alive by a reference cycle"
    finally:
        gc.enable()


def test_no_floating_point_atomic_adds_in_the_kernels():
    """Every floating-point reduction runs in a fixed order (results are bit-identical run to
    run), so no atomic add may target a floating-point value.  The integer counters and tickets
    that remain are listed here by file and destination."""
    allowed = {
        ("global.cu", "cnt + s"),             # per-cloud row counts of the counting sort
        ("coords.cu", "ticket"),              # last-CTA ticket
        ("batchnorm.cu", "tail.ticket"),      # last-CTA ticket
        ("kernel_map.cu", "num_pairs"),       # pair count of the compacted lists
    }
    csrc = os.path.join(ROOT, "minkowskiengine_b200", "csrc")
    call = re.compile(r"\b(?:unsafeAtomicAdd|atomicAdd(?:_block|_system)?)\s*\(\s*([^,]+?)\s*,")
    ptx = re.compile(r"\b(?:red|atom)(?:\.[a-z]+)*\.add\.(?:f|bf|noftz)")
    found = set()
    for name in sorted(os.listdir(csrc)):
        if not name.endswith((".cu", ".cuh", ".h")):
            continue
        text = open(os.path.join(csrc, name)).read()
        text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
        text = re.sub(r"//[^\n]*", "", text)
        assert not ptx.search(text), f"{name}: floating-point atomic add in inline PTX"
        found |= {(name, m.group(1)) for m in call.finditer(text)}
    assert found, "no atomic add found at all: the pattern no longer matches the sources"
    assert found <= allowed, f"atomic adds outside the integer allowlist: {sorted(found - allowed)}"
