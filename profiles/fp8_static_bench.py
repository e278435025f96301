"""Times the eval-mode forward of MinkUNet34C (examples/minkunet.py) on 8 clouds x 100k voxels of
examples.synthetic.surface_cloud, made as bench.py makes them, on bf16 features, three ways: the
fused bf16 path, ME.fp8_inference() (dynamic scales: an amax pass and a conversion before every
e4m3 layer) and ME.fp8_inference(calibration) (static scales: layers fed directly by a convolution
read the e4m3 shadow it wrote in its epilogue; the others convert once).  The calibration observes
two batches of clouds with seeds other than the timed ones.

    python profiles/fp8_static_bench.py [--reps 20] [--warmup 3]

The three modes alternate within one loop, each forward timed with CUDA events under
torch.no_grad().  Then one forward per mode with CUDA events around every native convolution and
quantisation call, which gives the per-layer table: the convolution's device time, the quantisation
time charged to it (zero where it reads a shadow), and for the static mode the difference to the
same layer's dynamic-mode convolution, which is what the shadow store costs the epilogue (the two
launches differ only in that store).  Prints the card's name and power limit, one JSON line with
the end-to-end times and the logits' distance to the exact fp32 network, one with the totals, and
one JSON line per layer."""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import minkowskiengine_b200 as ME  # noqa: E402
from fp8_bench import _Recorder, card, make_batch, timed  # noqa: E402

QUANT = ("meb200_quantize_e4m3", "meb200_quantize_e4m3_static")


class _StaticRecorder(_Recorder):
    NAMES = ("meb200_conv_forward", "meb200_conv_stem_forward", "meb200_conv_forward_fp8",
             "meb200_conv_forward_q", "meb200_conv_stem_forward_q", "meb200_conv_forward_fp8_q",
             "meb200_quantize_e4m3", "meb200_quantize_e4m3_static")

    def layers(self):
        """[(c_in, c_out, K, n_out, route, conv ms, quantise ms)]: a quantisation belongs to the
        convolution that follows it."""
        torch.cuda.synchronize()
        out, q_ms = [], 0.0
        for name, a, e0, e1 in self.recs:
            ms = e0.elapsed_time(e1)
            if name in QUANT:
                q_ms += ms
                continue
            shadow = " +shadow" if name.endswith("_q") else ""
            if name.startswith("meb200_conv_forward_fp8"):
                route = "e4m3" + shadow + (" (reads a shadow)" if q_ms == 0 else "")
                out.append((a[3], a[6], a[5], a[8], route, ms, q_ms))
            elif name.startswith("meb200_conv_forward"):
                out.append((a[3], a[7], a[6], a[9], "bf16" + shadow, ms, q_ms))
            else:
                out.append((4, a[4], a[2], a[6], "bf16 stem" + shadow, ms, q_ms))
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
        sys.exit("fp8_static_bench: no CUDA device")
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
    calib = ME.Fp8Calibration(net)
    with torch.no_grad(), calib.observe():
        for seed0 in (1000, 2000):         # other clouds than the timed ones
            c, f = make_batch(a.clouds, a.voxels, seed0=seed0)
            net(ME.SparseTensor(f.bfloat16().to(dev), c.to(dev)))
    sd = calib.state_dict()

    def dynamic():
        with ME.fp8_inference():
            return net(x)

    def static():
        with ME.fp8_inference(calib):
            return net(x)
    modes = {"bf16_fused": lambda: net(x), "fp8_dynamic": dynamic, "fp8_static": static}
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
        res = {"rows": int(len(coords)), "reps": a.reps,
               "calibrated_layers": sum(1 for v in sd.values() if v["amax"] is not None),
               "links": sum(len(v["feeds"]) for v in sd.values())}
        for k, fn in modes.items():
            y = fn().F.double()
            res[k] = {"median_ms": statistics.median(ms[k]), "min_ms": min(ms[k]),
                      "max_ms": max(ms[k]),
                      "logits_rms_rel_vs_fp32": float((y - want).pow(2).mean().sqrt()
                                                      / want.pow(2).mean().sqrt()),
                      "argmax_agreement_vs_fp32": float((y.argmax(1) == want.argmax(1))
                                                        .double().mean())}
        res["static_vs_dynamic_speedup"] = (res["fp8_dynamic"]["median_ms"]
                                            / res["fp8_static"]["median_ms"])
        res["static_vs_bf16_speedup"] = res["bf16_fused"]["median_ms"] / res["fp8_static"]["median_ms"]
        print(json.dumps(res), flush=True)
        tables = {}
        for k, fn in modes.items():
            with _StaticRecorder() as rec:
                fn()
            tables[k] = rec.layers()
    tot = {k: {"conv_ms": sum(r[5] for r in t), "quantise_ms": sum(r[6] for r in t),
               "quantise_calls": sum(1 for r in t if r[6] > 0)} for k, t in tables.items()}
    shadow_cost = sum(s[5] - d[5] for s, d in zip(tables["fp8_static"], tables["fp8_dynamic"])
                      if "shadow" in s[4] and "e4m3" in d[4] and "e4m3" in s[4])
    tot["shadow_store_ms_e4m3_producers"] = shadow_cost
    print(json.dumps(tot), flush=True)
    for i, (b, d, s) in enumerate(zip(tables["bf16_fused"], tables["fp8_dynamic"],
                                      tables["fp8_static"])):
        print(json.dumps({"layer": i, "c_in": b[0], "c_out": b[1], "K": b[2], "n_out": b[3],
                          "bf16_ms": round(b[5], 4), "dyn_route": d[4],
                          "dyn_conv_ms": round(d[5], 4), "dyn_quantise_ms": round(d[6], 4),
                          "static_route": s[4], "static_conv_ms": round(s[5], 4),
                          "static_quantise_ms": round(s[6], 4),
                          "shadow_epilogue_ms": round(s[5] - d[5], 4) if "shadow" in s[4] else 0.0}),
              flush=True)


if __name__ == "__main__":
    main()
