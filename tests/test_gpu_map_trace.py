"""Every call into the native library during six seeded training steps, each run twice on one
network (so that the second step runs on the map prediction the first one taught), must match the
trace recorded in tests/golden/map_trace.json: the same entry points in the same order, with the
same integer and tensor-stride arguments, return codes and unique counts.  Device pointers and
streams are left out.  The size queries `meb200_hash_capacity` and `meb200_insert_scratch_bytes`
are pure functions of their argument and are compared through the calls that use their results
(every table capacity is an argument of the insert, the table build, the find and the kernel map),
so where they are asked does not matter.

The steps run in a fresh interpreter, so that no hint learnt by an earlier manager is left.
Record the fixture with `python tests/test_gpu_map_trace.py --write tests/golden/map_trace.json`.
"""
import ctypes
import json
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
FIXTURE = os.path.join(HERE, "golden", "map_trace.json")
SIZE_QUERIES = {"meb200_hash_capacity", "meb200_insert_scratch_bytes"}

pytestmark = pytest.mark.gpu


class _Tracer:
    """Stands in for the loaded library and appends [name, args..., result] per call."""

    def __init__(self, lib, log):
        self._lib, self._log = lib, log

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        if not name.startswith("meb200_"):
            return fn
        from minkowskiengine_b200 import _lib
        argtypes = _lib.PROTOTYPES[name][1]

        def call(*args):
            rc = fn(*args)
            rec = [name]
            for t, a in zip(argtypes, args):
                if t is ctypes.c_void_p:
                    continue                                 # device pointer or stream
                if isinstance(a, ctypes.Array):
                    rec.append(list(a))                      # tensor stride
                elif hasattr(a, "_obj"):
                    rec.append(a._obj.value)                 # count written back (byref)
                else:
                    rec.append(a)
            rec.append(rc.decode() if isinstance(rc, bytes) else rc)
            self._log.append(rec)
            return rc
        return call


def record():
    """Runs the six workloads twice each -> the list of calls."""
    for p in (ROOT, HERE):
        if p not in sys.path:
            sys.path.insert(0, p)
    import torch
    from minkowskiengine_b200 import _lib
    log = []
    _lib._lib = _Tracer(_lib.load(), log)
    import minkowskiengine_b200 as ME
    import test_gpu_field as TF
    import test_gpu_generative as TG
    import test_gpu_global as TGL
    import test_gpu_unpool_splat as TU
    from examples.completion import completion_net
    from examples.minkunet import minkunet
    from examples.resnet import resnet
    from oracle import oracle_np as O
    dev = torch.device("cuda:0")

    def minkunet14():
        torch.manual_seed(0)
        return minkunet("MinkUNet14", ME, 3, 20, 3).to(dev).train()

    def minkunet14_step(ME, net, dev):
        coords = O.surface_cloud(50_000, seed=5)
        feats = torch.rand(50_000, 3, generator=torch.Generator().manual_seed(2)).bfloat16()
        net.zero_grad(set_to_none=True)
        out = net(ME.SparseTensor(feats.to(dev), coords.to(dev)))
        out.F.float().pow(2).mean().backward()

    def completion():
        torch.manual_seed(TG.COMPLETION_SEED)
        return completion_net(ME, TG.COMPLETION_CHANNELS, TG.COMPLETION_CHANNELS)

    def resnet14():
        torch.manual_seed(0)
        return resnet("ResNet14", ME, 3, 40, 3, dropout=0.0)

    workloads = [("minkunet14_bf16", minkunet14, minkunet14_step),
                 ("completion", completion, TG._completion_step),
                 ("resnet14", resnet14, TGL._resnet_step),
                 ("fcnn", lambda: TF.fcnn_net(ME), TF.fcnn_step),
                 ("stack_unet", lambda: TU.stack_unet_net(ME), TU.stack_unet_step),
                 ("splat_fcnn", lambda: TU.splat_fcnn_net(ME), TU.splat_fcnn_step)]
    for name, make, step in workloads:
        net = make()
        for i in range(2):
            log.append(["#", name, i])
            step(ME, net, dev)
            torch.cuda.synchronize()
    return log


def _compared(trace):
    return [c for c in trace if c[0] not in SIZE_QUERIES]


def test_native_calls_match_the_recorded_trace(cuda, tmp_path):
    out = tmp_path / "trace.json"
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + \
        [os.path.abspath(__file__), "--write", str(out)]
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    with open(out) as f:
        got = _compared(json.load(f))
    with open(FIXTURE) as f:
        want = _compared(json.load(f))
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, f"call {i} differs: {g} != {w} (recorded)"
    assert len(got) == len(want)


if __name__ == "__main__":
    path = sys.argv[sys.argv.index("--write") + 1]
    trace = record()
    with open(path, "w") as f:
        f.write("[\n" + ",\n".join(json.dumps(c) for c in trace) + "\n]\n")
    print(f"{len(trace)} calls -> {path}")
