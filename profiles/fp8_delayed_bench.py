"""Times bench.py's cfg3 training step (MinkUNet34C, bf16, 8 clouds x 100k voxels, maps rebuilt
every step, SGD) in bf16, inside ME.fp8_training(weight_gradient=True) with dynamic scales, and the
same with delayed scaling (ME.Fp8DelayedScaling, history 16, margin 0).

    python profiles/fp8_delayed_bench.py [--steps 20] [--warmup 3]

The modes alternate within one loop as in profiles/fp8_train_bench.py, each step timed with CUDA
events from before its SparseTensor is built to after the optimizer step.  Then one profiled step
per mode gives the per-family table (CUDA events around every library call of the convolutions,
quantisations, weight packs and batch-norm passes) and one more step per mode its peak memory.
Prints the card's name and power limit, then one JSON line each for the step times, the families
and the peak memory."""
import argparse
import contextlib
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import minkowskiengine_b200 as ME  # noqa: E402
from minkowskiengine_b200 import backend  # noqa: E402
from fp8_train_bench import _Recorder, card, make_batch  # noqa: E402

MODES = ("bf16", "fp8_wgrad", "fp8_wgrad_delayed")


class _DelayedRecorder(_Recorder):
    """_Recorder, with the delayed-scaling conversions, the roll and the batch-norm passes."""
    EXTRA = {"meb200_quantize_fp8_record": "quantise record", "meb200_fp8_roll": "roll",
             "meb200_amax_accumulate": "quantise amax"}
    BN = ("meb200_bn_forward_train", "meb200_bn_forward_train_q", "meb200_bn_backward_reduce_to",
          "meb200_bn_backward_apply_fused", "meb200_bn_backward_apply_fused_q")
    NAMES = _Recorder.NAMES + tuple(EXTRA) + BN

    def families(self):
        torch.cuda.synchronize()
        out, rest = [], []
        for r in self.recs:
            name, ms = r[0], r[2].elapsed_time(r[3])
            if name in self.EXTRA:
                out.append((self.EXTRA[name], 0, 0, 0, ms))
            elif name in self.BN:
                kind = "bn forward (stats + apply)" if "forward" in name else \
                    "bn backward reduce" if "reduce" in name else "bn backward apply"
                out.append((kind, 0, 0, 0, ms))
            else:
                rest.append(r)
        self.recs = rest
        return out + super().families()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clouds", type=int, default=8)
    ap.add_argument("--voxels", type=int, default=100_000)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("fp8_delayed_bench: no CUDA device")
    dev = torch.device("cuda:0")
    print(json.dumps(card()), flush=True)
    from examples.minkunet import minkunet
    coords_h, feats_h, labels_h = make_batch(a.clouds, a.voxels)
    coords, labels = coords_h.to(dev), labels_h.to(dev)
    feats = feats_h.to(dev).bfloat16()
    crit = torch.nn.CrossEntropyLoss()
    nets, opts, scaling = {}, {}, {}
    for mode in MODES:
        torch.manual_seed(0)
        nets[mode] = minkunet("MinkUNet34C", ME, 3, 20, 3).to(dev)
        opts[mode] = torch.optim.SGD(nets[mode].parameters(), lr=1e-2)
    scaling["fp8_wgrad_delayed"] = ME.Fp8DelayedScaling(nets["fp8_wgrad_delayed"], history=16)

    def step(mode):
        net, opt = nets[mode], opts[mode]
        opt.zero_grad(set_to_none=True)
        ctx = contextlib.nullcontext() if mode == "bf16" else \
            ME.fp8_training(weight_gradient=True, scaling=scaling.get(mode))
        with ctx:
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
    losses = {m: [] for m in nets}
    for _ in range(a.steps):
        for m in nets:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            loss = step(m)
            e1.record()
            torch.cuda.synchronize()
            ms[m].append(e0.elapsed_time(e1))
            losses[m].append(float(loss))
    res = {"rows": int(len(coords)), "steps": a.steps, "step0_loss": loss0,
           "last_loss": {m: v[-1] for m, v in losses.items()}}
    for m, v in ms.items():
        res[m] = {"median_ms": statistics.median(v), "min_ms": min(v), "max_ms": max(v)}
    res["delayed_over_dynamic"] = res["fp8_wgrad_delayed"]["median_ms"] / res["fp8_wgrad"]["median_ms"]
    print(json.dumps(res), flush=True)

    fam = {}
    for m in nets:
        with _DelayedRecorder() as rec:
            backend.profile_conv_kernels(lambda: step(m), steps=1)
        for f, K, ci, co, v in rec.families():
            key = f if K == 0 else f"{f} K={K}"
            d = fam.setdefault(key, {})
            d[m] = round(d.get(m, 0.0) + v, 4)
    print(json.dumps({"ms_per_family": fam}), flush=True)
    peak = {}
    for m in nets:
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        step(m)
        torch.cuda.synchronize()
        peak[m] = round(torch.cuda.max_memory_allocated() / 2 ** 30, 3)
    print(json.dumps({"peak_memory_gib": peak}), flush=True)


if __name__ == "__main__":
    main()
