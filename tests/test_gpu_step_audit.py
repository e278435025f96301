"""MinkUNet training steps (and an eval forward) audited layer by layer against float64 on the
inputs each layer received (tests/step_audit.py): convolutions forward, dgrad and wgrad within
their kernels' one-rounding bounds on kernel maps rebuilt from the coordinates, batch norm within
the bounds of tests/test_gpu_batchnorm_fp64.py, `cat` and the K = 1 matrix products bit for bit.

Two steps with `opt.step()` in between: the second runs on the maps the first step's requests
predicted, on weights re-packed in one batched launch after the update, and on the workspaces the
first step left.  `cfg3` is bench.py's flagship step at full size."""
import time
from collections import Counter

import pytest
import torch

from examples.minkunet import minkunet
from examples.synthetic import surface_cloud
from step_audit import RecordingHandle, StepAudit

pytestmark = pytest.mark.gpu

# model, dtype, torch fp32 matmul precision, clouds, voxels per cloud, training steps (0: eval)
CASES = {
    "fp16": ("MinkUNet14", torch.float16, "ieee", 1, 50_000, 2),
    "fp32": ("MinkUNet34C", torch.float32, "ieee", 2, 20_000, 2),
    "tf32": ("MinkUNet34C", torch.float32, "tf32", 2, 20_000, 2),
    "eval": ("MinkUNet34C", torch.bfloat16, "ieee", 2, 50_000, 0),
    "cfg3": ("MinkUNet34C", torch.bfloat16, "ieee", 8, 100_000, 2),
}


@pytest.fixture
def precision():
    saved = torch.backends.cuda.matmul.fp32_precision
    yield
    torch.backends.cuda.matmul.fp32_precision = saved


def _batch(clouds, voxels, device, dtype):
    """bench.make_batch(clouds, voxels, 0): one surface cloud per batch index."""
    coords = torch.cat([surface_cloud(voxels, j, batch=j) for j in range(clouds)], 0)
    feats = torch.rand(len(coords), 3, generator=torch.Generator().manual_seed(0))
    labels = torch.zeros(len(coords), dtype=torch.int64)
    return coords.to(device), feats.to(device).to(dtype), labels.to(device)


def _network(ME, model, audit, device):
    from minkowskiengine_b200.convolution import MinkowskiConvolutionBase
    torch.manual_seed(0)
    net = minkunet(model, RecordingHandle(ME, audit), 3, 20, 3)
    audit.names(net)
    convs = [n for n, m in net.named_modules() if isinstance(m, MinkowskiConvolutionBase)]
    norms = [n for n, m in net.named_modules() if isinstance(m, ME.MinkowskiBatchNorm)]
    return net.to(device), convs, norms


def _count_predictions(monkeypatch, audit):
    """Per step, how many pyramid levels the manager took from the prediction."""
    from minkowskiengine_b200 import backend
    takes = Counter()
    real = backend._Prediction.take

    def take(self, mgr, in_key, out_key):
        hit = real(self, mgr, in_key, out_key)
        takes[audit.step] += int(hit)
        return hit
    monkeypatch.setattr(backend._Prediction, "take", take)
    return takes


def _train(ME, net, audit, batch, steps, lr=1e-2):
    """bench.py's step: zero_grad, forward, cross entropy, backward, SGD.  Returns the backend
    manager of every step's input."""
    coords, feats, labels = batch
    opt = torch.optim.SGD(net.parameters(), lr=lr)
    crit = torch.nn.CrossEntropyLoss()
    managers = []
    with audit.backward_routes():
        for s in range(1, steps + 1):
            audit.begin_step(s)
            opt.zero_grad(set_to_none=True)
            x = ME.SparseTensor(feats, coords)
            managers.append(x._manager._manager)
            out = net(x)
            crit(out.F.float(), labels).backward()
            opt.step()
            torch.cuda.synchronize()
    return managers


def _report(case, audit, record_property, seconds):
    print(f"\n[step audit] {case}: {len(audit.rows)} audited calls in {seconds:.1f} s, peak memory "
          f"{torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB")
    for r in audit.rows:
        print("[step audit]", r.line(), " ".join(r.notes))
    kinds = {}
    for r in audit.rows:
        k = (r.kind, r.route)
        kinds[k] = max(kinds.get(k, 0.0), r.worst)
    for (kind, route), w in sorted(kinds.items()):
        print(f"[step audit] {case} worst {kind} {route}: {w:.3g}")
    worst = max(r.worst for r in audit.rows)
    record_property("worst_ratio_to_bound", worst)
    record_property("seconds", round(seconds, 1))
    record_property("peak_gib", round(torch.cuda.max_memory_allocated() / 2 ** 30, 2))
    bad = [f"step {r.step} {r.name} ({r.kind}): " + "; ".join(r.failures or
                                                              [f"ratio {r.worst:.3g}"])
           for r in audit.rows if r.failures or r.worst > 1]
    assert not bad, "\n".join(bad)


def _assert_coverage(audit, convs, norms, steps):
    for s in steps:
        for n in convs + norms:
            assert audit.calls[(s, n)] == 1, f"step {s}: {n} audited {audit.calls[(s, n)]} times"
        assert audit.cats[s] == 4, f"step {s}: {audit.cats[s]} cats"
        assert sum(c for (st, _), c in audit.calls.items() if st == s) == len(convs) + len(norms)


@pytest.mark.parametrize("case", list(CASES))
def test_step_layers_match_float64(ME, cuda, case, precision, monkeypatch, record_property):
    model, dtype, prec, clouds, voxels, steps = CASES[case]
    torch.backends.cuda.matmul.fp32_precision = prec
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    audit = StepAudit(ME)
    takes = _count_predictions(monkeypatch, audit)
    net, convs, norms = _network(ME, model, audit, cuda)
    batch = _batch(clouds, voxels, cuda, dtype)
    if steps:
        managers = _train(ME, net, audit, batch, steps)
        _assert_coverage(audit, convs, norms, range(1, steps + 1))
        assert takes[2] > 0, "the second step built its maps without the prediction"
        if case == "cfg3":
            chunks = [km._pairs[3] for km in managers[1]._kernel_maps.values()
                      if km._pairs is not None]
            assert max(chunks) > 1, "no pair list of the step spans two row chunks"
    else:
        audit.enabled = False
        with torch.no_grad():          # running statistics of one batch
            net(ME.SparseTensor(batch[1], batch[0]))
        audit.enabled = True
        net.eval()
        audit.begin_step(1)
        with torch.no_grad():
            net(ME.SparseTensor(batch[1], batch[0]))
        _assert_coverage(audit, convs, norms, [1])
        fused = [r for r in audit.rows if r.kind == "conv+bn"]
        assert len(fused) == len(norms) - sum("downsample" in n for n in norms)
        assert all("one_launch" in r.ratios for r in fused)
    torch.cuda.synchronize()
    missing = audit.missing()
    assert not missing, "checks that did not run:\n" + "\n".join(missing)
    if dtype == torch.float32 and prec == "ieee":
        # the default switch keeps fp32 on the exact CUDA cores, forward and backward
        moved = [f"step {r.step} {r.name}: {r.route}" for r in audit.rows
                 if r.kind in ("conv", "convtr") and r.route not in ("cuda", "cuda/cuda")]
        assert not moved, "fp32 layers on the tensor cores:\n" + "\n".join(moved)
    _report(case, audit, record_property, time.perf_counter() - t0)


def test_stale_packed_weights_are_caught(ME, cuda, monkeypatch):
    """The audit's own sensitivity: with the packed-weight lookup returning step 1's packs on
    step 2, every step-2 convolution must be reported out of bound.  fp16 (its rounding resolves
    the update) and lr 0.1, so that every kernel moves by more than one fp16 rounding."""
    from minkowskiengine_b200 import backend
    audit = StepAudit(ME)
    net, _, _ = _network(ME, "MinkUNet14", audit, cuda)
    stash = {}
    real_packed, real_stem = backend._packed_weights, backend._stem_weights

    def packed(kernel, dtype):
        out = real_packed(kernel, dtype)
        key = (id(kernel), str(dtype))
        if audit.step == 1:
            stash.setdefault(key, tuple(t.clone() for t in out))
        return stash.get(key, out) if audit.step == 2 else out

    def stem(kernel, dtype):
        out = real_stem(kernel, dtype)
        key = (id(kernel), str(dtype), "stem")
        if audit.step == 1:
            stash.setdefault(key, out.clone())
        return stash.get(key, out) if audit.step == 2 else out
    monkeypatch.setattr(backend, "_packed_weights", packed)
    monkeypatch.setattr(backend, "_stem_weights", stem)
    _train(ME, net, audit, _batch(1, 20_000, cuda, torch.float16), 2, lr=0.1)
    convs = [r for r in audit.rows if r.kind in ("conv", "convtr")]
    step1 = [r for r in convs if r.step == 1]
    step2 = [r for r in convs if r.step == 2]
    assert step1 and all(r.worst <= 1 for r in step1), "step 1 must pass"
    caught = [r for r in step2 if r.ratios["fwd"] > 1]
    print(f"[step audit] stale packs: {len(caught)} of {len(step2)} step-2 convolutions out of "
          f"bound; worst {max(r.ratios['fwd'] for r in step2):.3g}")
    assert step2 and len(caught) == len(step2), \
        f"only {len(caught)} of {len(step2)} step-2 convolutions caught the stale packs"
