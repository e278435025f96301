"""Times bench.py's cfg3 training step (MinkUNet34C, examples/minkunet.py, on 8 clouds x 100k voxels
of examples.synthetic.surface_cloud, bf16 features, maps rebuilt every step, SGD) in bf16 against the
same step inside ME.fp8_training().

    python profiles/fp8_train_bench.py [--steps 20] [--warmup 3]

One network per mode, both from the same initial state; the two modes alternate within one loop,
each step timed with CUDA events from before its SparseTensor is built to after the optimizer step.
Then, in a separate run of one step per mode, backend.profile_conv_kernels splits every backward
into its dgrad and its wgrad call, and CUDA events around every library call of the convolutions,
the fp8 quantisations and the weight packs give the per-family and per-layer breakdown.  Prints the
card's name and power limit, one JSON line with the step times and the step-0 losses, one with the
per-family totals and one JSON line per convolution layer."""
import argparse
import contextlib
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import minkowskiengine_b200 as ME  # noqa: E402
from minkowskiengine_b200 import _lib, backend  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return {"gpu": torch.cuda.get_device_name(), "nvidia_smi": q[0] if q else "unavailable"}


def make_batch(n_clouds, n_voxels, seed0=0):
    """bench.py's make_batch: one surface cloud per batch index, uniform [0, 1) RGB, labels 0."""
    from examples.synthetic import surface_cloud
    coords = torch.cat([surface_cloud(n_voxels, seed0 + j, batch=j) for j in range(n_clouds)], 0)
    feats = torch.rand(len(coords), 3, generator=torch.Generator().manual_seed(seed0))
    return coords.contiguous(), feats, torch.zeros(len(coords), dtype=torch.int64)


class _Recorder:
    """CUDA events around the library calls of the convolutions, quantisations and packs."""
    NAMES = ("meb200_conv_forward", "meb200_conv_stem_forward", "meb200_conv_forward_fp8",
             "meb200_conv_backward", "meb200_conv_stem_wgrad", "meb200_conv_dgrad_fp8",
             "meb200_quantize_e4m3", "meb200_quantize_e5m2", "meb200_conv_pack_weights",
             "meb200_conv_pack_weights_batched", "meb200_conv_pack_weights_e4m3",
             "meb200_conv_pack_weights_e4m3_dgrad")

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

    def families(self):
        """[(family, K, c_in, c_out, ms)] in call order."""
        torch.cuda.synchronize()
        out = []
        for name, a, e0, e1 in self.recs:
            ms = e0.elapsed_time(e1)
            if name == "meb200_conv_backward":      # profile_conv_kernels splits dgrad and wgrad
                fam = "dgrad" if a[11] is not None else "wgrad"
                out.append((fam, a[6], a[4], a[7], ms))
            elif name == "meb200_conv_forward":
                out.append(("forward", a[6], a[3], a[7], ms))
            elif name == "meb200_conv_forward_fp8":
                out.append(("forward", a[5], a[3], a[6], ms))
            elif name == "meb200_conv_dgrad_fp8":
                out.append(("dgrad", a[6], a[7], a[3], ms))
            elif name == "meb200_conv_stem_forward":
                out.append(("forward", a[2], 4, a[4], ms))
            elif name == "meb200_conv_stem_wgrad":
                out.append(("wgrad", a[3], 4, a[4], ms))
            elif name.startswith("meb200_quantize"):
                out.append(("quantise " + name[-4:], 0, a[3], 0, ms))
            else:
                out.append(("pack " + name[len("meb200_conv_pack_weights"):].strip("_"), 0, 0, 0, ms))
        return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clouds", type=int, default=8)
    ap.add_argument("--voxels", type=int, default=100_000)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("fp8_train_bench: no CUDA device")
    dev = torch.device("cuda:0")
    print(json.dumps(card()), flush=True)
    from examples.minkunet import minkunet
    coords_h, feats_h, labels_h = make_batch(a.clouds, a.voxels)
    coords, labels = coords_h.to(dev), labels_h.to(dev)
    feats = feats_h.to(dev).bfloat16()
    crit = torch.nn.CrossEntropyLoss()
    nets, opts = {}, {}
    for mode in ("bf16", "fp8"):
        torch.manual_seed(0)
        nets[mode] = minkunet("MinkUNet34C", ME, 3, 20, 3).to(dev)
        opts[mode] = torch.optim.SGD(nets[mode].parameters(), lr=1e-2)

    def step(mode):
        net, opt = nets[mode], opts[mode]
        opt.zero_grad(set_to_none=True)
        with ME.fp8_training() if mode == "fp8" else contextlib.nullcontext():
            out = net(ME.SparseTensor(feats, coords))
            loss = crit(out.F.float(), labels)
            loss.backward()
        opt.step()
        return loss

    loss0 = {m: float(step(m)) for m in nets}          # step 0 from the same state
    for _ in range(a.warmup):
        for m in nets:
            step(m)
    torch.cuda.synchronize()
    ms = {m: [] for m in nets}
    for _ in range(a.steps):
        for m in nets:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            step(m)
            e1.record()
            torch.cuda.synchronize()
            ms[m].append(e0.elapsed_time(e1))
    res = {"rows": int(len(coords)), "steps": a.steps, "step0_loss": loss0}
    for m, v in ms.items():
        res[m] = {"median_ms": statistics.median(v), "min_ms": min(v), "max_ms": max(v)}
    res["fp8_over_bf16"] = res["fp8"]["median_ms"] / res["bf16"]["median_ms"]
    print(json.dumps(res), flush=True)

    tables = {}
    for m in nets:
        with _Recorder() as rec:
            backend.profile_conv_kernels(lambda: step(m), steps=1)
        tables[m] = rec.families()
    fam = {}
    for m, t in tables.items():
        for f, K, ci, co, v in t:
            key = f if f.startswith(("quantise", "pack")) else f"{f} K={K}"
            d = fam.setdefault(key, {})
            d[m] = round(d.get(m, 0.0) + v, 4)
    print(json.dumps({"ms_per_family": fam}), flush=True)
    for f in ("forward", "dgrad", "wgrad"):
        rows = {m: [r for r in t if r[0] == f] for m, t in tables.items()}
        for i, (b, q) in enumerate(zip(rows["bf16"], rows["fp8"])):
            print(json.dumps({"pass": f, "layer": i, "K": b[1], "c_in": b[2], "c_out": b[3],
                              "bf16_ms": round(b[4], 4), "fp8_mode_ms": round(q[4], 4)}),
                  flush=True)


if __name__ == "__main__":
    main()
