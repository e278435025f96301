"""fp32 convolutions in exact fp32 against TF32 (torch.backends.cuda.matmul.fp32_precision), with
bf16 alongside for context: one MinkUNet34C training step (fwd + bwd + SGD) on 8 synthetic surface
clouds x 100k voxels, every coordinate and kernel map rebuilt each step as in bench.py cfg3.

    python profiles/tf32_bench.py [--out DIR] [--rounds 3] [--steps 5] [--warmup 3]

Step times come from CUDA events around `steps` consecutive steps; the three modes are timed in
alternating rounds after every mode has been warmed up.  A second pass times every convolution
call (forward, dgrad and wgrad separately, as backend.profile_conv_kernels splits them) with CUDA
events and sums them per layer shape; achieved TFLOP/s are algorithmic (2 P c_in c_out per call,
P the pairs of the kernel map) over that time.  Data-sheet dense rates of the H100 SXM, for
scale only: 495 TFLOP/s TF32, 67 TFLOP/s FP32, 989 TFLOP/s BF16.  The card's name and power limit
are read in the same run and printed with the results."""
import argparse
import json
import os
import subprocess
import sys
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import minkowskiengine_b200 as ME  # noqa: E402
from bench import make_batch  # noqa: E402
from examples.minkunet import minkunet  # noqa: E402
from minkowskiengine_b200 import backend  # noqa: E402

MODES = ("fp32", "tf32", "bf16")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else \
        torch.cuda.get_device_name(0)


def set_mode(mode):
    torch.backends.cuda.matmul.fp32_precision = "tf32" if mode == "tf32" else "ieee"


def make_step(net, opt, crit, c, f, lab, mode):
    feats = f.to(torch.bfloat16) if mode == "bf16" else f

    def step():
        set_mode(mode)
        opt.zero_grad(set_to_none=True)
        out = net(ME.SparseTensor(feats, c))
        loss = crit(out.F.float(), lab)
        loss.backward()
        opt.step()
        return loss
    return step


def time_steps(step, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        step()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def per_layer(step):
    """{(kind, K, c_in, c_out): [ms, flops, calls]} over one step; kind fwd / dgrad / wgrad."""
    recs = []
    f_impl, b_impl = backend._conv_forward_impl, backend._conv_backward_impl

    def timed(kind, fn, kernel, km):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        K, ci, co = kernel.shape
        recs.append((kind, int(K), int(ci), int(co), e0, e1, 2.0 * km.n_pairs * ci * co))
        return out

    def fwd(in_feat, kernel, km, out_dtype=None):
        return timed("fwd", lambda: f_impl(in_feat, kernel, km, out_dtype), kernel, km)

    def bwd(in_feat, grad_out, kernel, km, need_in=True, need_w=True):
        kind = "dgrad" if need_in and not need_w else ("wgrad" if need_w and not need_in else "bwd")
        return timed(kind, lambda: b_impl(in_feat, grad_out, kernel, km, need_in, need_w), kernel, km)

    backend._conv_forward_impl, backend._conv_backward_impl = fwd, bwd
    try:
        families = backend.profile_conv_kernels(step, steps=1)   # splits dgrad and wgrad calls
    finally:
        backend._conv_forward_impl, backend._conv_backward_impl = f_impl, b_impl
    torch.cuda.synchronize()
    table = defaultdict(lambda: [0.0, 0.0, 0])
    for kind, K, ci, co, e0, e1, fl in recs:
        t = table[(kind, K, ci, co)]
        t[0] += e0.elapsed_time(e1)
        t[1] += fl
        t[2] += 1
    return table, families


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--clouds", type=int, default=8)
    ap.add_argument("--voxels", type=int, default=100_000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("tf32_bench.py needs a CUDA device")
    dev = torch.device("cuda:0")
    saved = torch.backends.cuda.matmul.fp32_precision
    torch.manual_seed(0)
    net = minkunet("MinkUNet34C", ME, 3, 20, 3).to(dev)
    opt = torch.optim.SGD(net.parameters(), lr=1e-4)
    crit = torch.nn.CrossEntropyLoss()
    c, f, lab = make_batch(a.clouds, a.voxels, 0)
    c, f, lab = c.to(dev), f.to(dev), lab.to(dev)
    steps = {m: make_step(net, opt, crit, c, f, lab, m) for m in MODES}
    res = {"card": card(), "workload": f"MinkUNet34C fwd+bwd+SGD, {a.clouds} x {a.voxels} "
           "surface voxels, maps rebuilt every step", "step_ms": {m: [] for m in MODES}}
    try:
        for m in MODES:
            for _ in range(a.warmup):
                steps[m]()
        torch.cuda.synchronize()
        for _ in range(a.rounds):
            for m in MODES:
                res["step_ms"][m].append(time_steps(steps[m], a.steps))
        layers = {}
        for m in MODES:
            table, fam = per_layer(steps[m])
            layers[m] = table
            res.setdefault("tc_families", {})[m] = fam
    finally:
        torch.backends.cuda.matmul.fp32_precision = saved

    lines = [f"card: {res['card']}", f"workload: {res['workload']}", "",
             "step time, ms (CUDA events, alternating rounds):"]
    for m in MODES:
        v = res["step_ms"][m]
        lines.append(f"  {m:5s} " + " ".join(f"{x:8.2f}" for x in v) + f"   min {min(v):.2f}")
    lines += ["", "per layer shape, one step (ms summed over calls; TFLOP/s algorithmic):",
              f"  {'kind':5s} {'K':>4s} {'c_in':>5s} {'c_out':>5s} {'calls':>5s} | "
              + " | ".join(f"{m:>5s} ms  TF/s" for m in MODES) + " | tf32/fp32"]
    keys = sorted(set().union(*[set(t) for t in layers.values()]),
                  key=lambda k: ("fwd", "dgrad", "wgrad", "bwd").index(k[0]) * 10 ** 7
                  + k[1] * 10 ** 4 + k[2] * 10 + k[3] / 1000)
    rows = []
    for k in keys:
        cells, ms = [], {}
        for m in MODES:
            t = layers[m].get(k)
            if t is None:
                cells.append(f"{'-':>14s}")
                continue
            ms[m] = t[0]
            cells.append(f"{t[0]:8.3f} {t[1] / t[0] / 1e9 if t[0] > 0 else 0:5.1f}")
        ratio = ms["tf32"] / ms["fp32"] if "tf32" in ms and ms.get("fp32") else float("nan")
        calls = max(layers[m].get(k, [0, 0, 0])[2] for m in MODES)
        lines.append(f"  {k[0]:5s} {k[1]:4d} {k[2]:5d} {k[3]:5d} {calls:5d} | " + " | ".join(cells)
                     + f" | {ratio:5.2f}")
        rows.append({"kind": k[0], "K": k[1], "c_in": k[2], "c_out": k[3], "calls": calls,
                     **{m: layers[m].get(k) for m in MODES}})
    for m in MODES:
        tot = defaultdict(float)
        for (kind, *_), t in layers[m].items():
            tot[kind] += t[0]
        lines.append(f"  total {m:5s}: " + ", ".join(f"{kd} {v:.2f} ms" for kd, v in tot.items()))
    text = "\n".join(lines)
    print(text)
    res["layers"] = rows
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "tf32_bench.txt"), "w") as fh:
            fh.write(text + "\n")
        with open(os.path.join(a.out, "tf32_bench.json"), "w") as fh:
            json.dump(res, fh, indent=1, default=str)


if __name__ == "__main__":
    main()
