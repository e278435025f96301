"""Times the eval-mode forward of MinkUNet34C (examples/minkunet.py) on 8 clouds x 100k voxels of
examples.synthetic.surface_cloud, made as bench.py makes them, with every conv -> batch norm
[-> + residual] -> ReLU run as one convolution with an epilogue (ME.fused_conv_bn_relu) against the
two-pass composition (the convolution, then fused_bn_relu), in bf16 and in fp32 (exact fp32, torch's
default matmul precision).

    python profiles/inference_bench.py [--reps 20] [--warmup 3]

Both nets hold the same weights and running statistics (a few training-mode forwards set the
latter).  The input tensor is built once per dtype, so its coordinate and kernel maps are built by
the warm-up and every timed forward reuses them: the times are the network's device work, under
torch.no_grad().  The two nets alternate within one loop, each forward timed with CUDA events;
prints the card's name and power limit, then one JSON line per dtype with the median and spread of
both, the native launches per forward and how far the two outputs are apart."""
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


class _Unfused:
    """The package as a module handle without fused_conv_bn_relu: the examples then build the
    two-pass composition."""

    def __init__(self, me):
        self._me = me

    def __getattr__(self, name):
        if name == "fused_conv_bn_relu":
            raise AttributeError(name)
        return getattr(self._me, name)


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


def nets(dev, x):
    from examples.minkunet import minkunet
    torch.manual_seed(0)
    fused = minkunet("MinkUNet34C", ME, 3, 20, 3).to(dev)
    plain = minkunet("MinkUNet34C", _Unfused(ME), 3, 20, 3).to(dev)
    with torch.no_grad():
        for _ in range(3):
            fused.train()(x)
    plain.load_state_dict(fused.state_dict())
    return fused.eval(), plain.eval()


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clouds", type=int, default=8)
    ap.add_argument("--voxels", type=int, default=100_000)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("inference_bench: no CUDA device")
    dev = torch.device("cuda:0")
    print(json.dumps(card()), flush=True)
    torch.backends.cuda.matmul.fp32_precision = "ieee"
    coords, feats = make_batch(a.clouds, a.voxels)
    for dtype in (torch.bfloat16, torch.float32):
        x = ME.SparseTensor(feats.to(dtype).to(dev), coords.to(dev))
        fused, plain = nets(dev, x)
        runs = {"fused": (fused, []), "composition": (plain, [])}
        launches = {}
        with torch.no_grad():
            for name, (net, _) in runs.items():
                for _ in range(a.warmup):
                    net(x)
                torch.cuda.synchronize()
                n0 = _lib.launch_count()
                net(x)
                launches[name] = _lib.launch_count() - n0
            for _ in range(a.reps):
                for name, (net, ms) in runs.items():
                    ms.append(timed(lambda: net(x))[0])
            y, want = fused(x).F.double(), plain(x).F.double()
        res = {"dtype": str(dtype).replace("torch.", ""), "rows": int(len(coords)), "reps": a.reps}
        for name, (_, ms) in runs.items():
            res[name] = {"median_ms": statistics.median(ms), "min_ms": min(ms), "max_ms": max(ms),
                         "native_launches": launches[name]}
        res["speedup"] = res["composition"]["median_ms"] / res["fused"]["median_ms"]
        res["logits_rms_rel"] = float((y - want).pow(2).mean().sqrt() / want.pow(2).mean().sqrt())
        res["argmax_agreement"] = float((y.argmax(1) == want.argmax(1)).double().mean())
        print(json.dumps(res), flush=True)
        del fused, plain, x, runs
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
