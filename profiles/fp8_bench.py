"""Times the eval-mode forward of MinkUNet34C (examples/minkunet.py) on 8 clouds x 100k voxels of
examples.synthetic.surface_cloud, made as bench.py makes them, on bf16 features: the fused bf16
path (ME.fused_conv_bn_relu) against the same network inside ME.fp8_inference(), where every conv
on the e4m3 grid runs on e4m3 operands.

    python profiles/fp8_bench.py [--reps 20] [--warmup 3]

One network, one input tensor (its maps are built by the warm-up); the two modes alternate within
one loop, each forward timed with CUDA events under torch.no_grad().  Then one forward per mode
with CUDA events around every native convolution call and every activation quantisation, which
gives the per-layer table (device time of the call's kernels; the events add no work to them).
Prints the card's name and power limit, one JSON line with the end-to-end times, the logits'
distance to the exact fp32 network, and one JSON line per layer."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import minkowskiengine_b200 as ME  # noqa: E402
from minkowskiengine_b200 import _lib  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return {"gpu": torch.cuda.get_device_name(), "nvidia_smi": q[0] if q else "unavailable"}


def make_batch(n_clouds, n_voxels, seed0=0):
    """bench.py's make_batch: one surface cloud per batch index, uniform [0, 1) RGB features."""
    from examples.synthetic import surface_cloud
    coords = torch.cat([surface_cloud(n_voxels, seed0 + j, batch=j) for j in range(n_clouds)], 0)
    feats = torch.rand(len(coords), 3, generator=torch.Generator().manual_seed(seed0))
    return coords.contiguous(), feats


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), out


class _Recorder:
    """CUDA events around the library's convolution and quantisation calls, in call order."""
    NAMES = ("meb200_conv_forward", "meb200_conv_stem_forward", "meb200_conv_forward_fp8",
             "meb200_quantize_e4m3")

    def __init__(self):
        self.lib = _lib.load()
        self.real = {n: getattr(self.lib, n) for n in self.NAMES}
        self.recs = []

    def __enter__(self):
        for n, fn in self.real.items():
            setattr(self.lib, n, self._wrap(n, fn))
        return self

    def __exit__(self, *exc):
        for n, fn in self.real.items():
            setattr(self.lib, n, fn)

    def _wrap(self, name, fn):
        def call(*args):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            rc = fn(*args)
            e1.record()
            self.recs.append((name, args, e0, e1))
            return rc
        return call

    def layers(self):
        """[(c_in, c_out, K, n_out, route, conv ms, quantise ms)]: a quantisation belongs to the
        e4m3 forward that follows it."""
        torch.cuda.synchronize()
        out, q_ms = [], 0.0
        for name, a, e0, e1 in self.recs:
            ms = e0.elapsed_time(e1)
            if name == "meb200_quantize_e4m3":
                q_ms = ms
                continue
            if name == "meb200_conv_forward_fp8":
                out.append((a[3], a[6], a[5], a[8], "e4m3", ms, q_ms))
            elif name == "meb200_conv_forward":
                out.append((a[3], a[7], a[6], a[9], "bf16", ms, 0.0))
            else:
                out.append((4, a[4], a[2], a[6], "bf16 stem", ms, 0.0))
            q_ms = 0.0
        return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clouds", type=int, default=8)
    ap.add_argument("--voxels", type=int, default=100_000)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("fp8_bench: no CUDA device")
    dev = torch.device("cuda:0")
    print(json.dumps(card()), flush=True)
    torch.backends.cuda.matmul.fp32_precision = "ieee"
    from examples.minkunet import minkunet
    coords, feats = make_batch(a.clouds, a.voxels)
    torch.manual_seed(0)
    net = minkunet("MinkUNet34C", ME, 3, 20, 3).to(dev)
    x32 = ME.SparseTensor(feats.to(dev), coords.to(dev))
    with torch.no_grad():
        for _ in range(3):                 # running statistics of a few batches
            net.train()(x32)
    net.eval()
    x = ME.SparseTensor(feats.bfloat16().to(dev), coords.to(dev))

    def fp8():
        with ME.fp8_inference():
            return net(x)
    modes = {"bf16_fused": lambda: net(x), "fp8_fused": fp8}
    ms = {k: [] for k in modes}
    with torch.no_grad():
        for fn in modes.values():
            for _ in range(a.warmup):
                fn()
        torch.cuda.synchronize()
        for _ in range(a.reps):
            for k, fn in modes.items():
                ms[k].append(timed(fn)[0])
        want = net(x32).F.double()
        res = {"rows": int(len(coords)), "reps": a.reps}
        for k, fn in modes.items():
            y = fn().F.double()
            res[k] = {"median_ms": statistics.median(ms[k]), "min_ms": min(ms[k]),
                      "max_ms": max(ms[k]),
                      "logits_rms_rel_vs_fp32": float((y - want).pow(2).mean().sqrt()
                                                      / want.pow(2).mean().sqrt()),
                      "argmax_agreement_vs_fp32": float((y.argmax(1) == want.argmax(1))
                                                        .double().mean())}
        res["speedup"] = res["bf16_fused"]["median_ms"] / res["fp8_fused"]["median_ms"]
        print(json.dumps(res), flush=True)
        tables = {}
        for k, fn in modes.items():
            with _Recorder() as rec:
                fn()
            tables[k] = rec.layers()
    tot = {k: [sum(r[5] for r in t), sum(r[6] for r in t)] for k, t in tables.items()}
    print(json.dumps({"conv_ms_total": {k: v[0] for k, v in tot.items()},
                      "quantise_ms_total": {k: v[1] for k, v in tot.items()}}), flush=True)
    for i, (b, f) in enumerate(zip(tables["bf16_fused"], tables["fp8_fused"])):
        print(json.dumps({"layer": i, "c_in": b[0], "c_out": b[1], "K": b[2], "n_out": b[3],
                          "bf16_ms": round(b[5], 4), "route": f[4], "fp8_conv_ms": round(f[5], 4),
                          "quantise_ms": round(f[6], 4)}), flush=True)


if __name__ == "__main__":
    main()
