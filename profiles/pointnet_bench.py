"""Device time of global pooling over TensorField points against pooling a coordinate map of the
same rows, and of a MinkowskiPointNet training step, with CUDA events, in one call:

    python profiles/pointnet_bench.py [--iters 20] [--json out.json]

Timed after warm-up:
  * the first grouping of a field (meb200_field_origin_group; its one host read included), at
    8 clouds x 125k points;
  * cached max / avg pooling forward and backward of that field, and of the stride-1 map of the
    same points (no two points share a voxel, so its rows are the points), C = 1024, fp32 and bf16;
  * one examples/pointnet.py training step (default widths) on 32 clouds x 2048 points, fp32 and
    bf16.
The card name and power limit are recorded with the numbers."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import minkowskiengine_b200 as ME  # noqa: E402
from examples.pointnet import pointnet  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=20).stdout.strip().splitlines()
        name, power = [v.strip() for v in q[0].split(",")]
    except Exception:                      # noqa: BLE001
        name, power = torch.cuda.get_device_name(), "unknown"
    return {"name": name, "power_limit": power}


def timed(fn, iters):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def points(B, n_per, dev):
    """B clouds of n_per points, each point in its own stride-1 voxel, in shuffled order."""
    i = torch.arange(n_per, device=dev)
    xyz = torch.stack([i % 64, (i // 64) % 64, i // 4096], 1).float() + 0.5
    pts = torch.cat([torch.arange(B, device=dev).repeat_interleave(n_per)[:, None].float(),
                     xyz.repeat(B, 1)], 1)
    return pts[torch.randperm(B * n_per, device=dev)].contiguous()


def pooling(B, n_per, C, dtype, iters):
    dev = torch.device("cuda")
    pts = points(B, n_per, dev)
    feats = torch.randn(B * n_per, C, device=dev).to(dtype)
    res = {"clouds": B, "points": B * n_per, "C": C, "dtype": str(dtype)}
    # the first grouping, over fresh fields of the same points (the origin exists already)
    mgr = ME.TensorField(feats, pts).coordinate_manager
    ME.MinkowskiGlobalMaxPooling()(ME.TensorField(feats, pts, coordinate_manager=mgr))
    times = []
    for _ in range(5):
        x = ME.TensorField(feats, pts, coordinate_manager=mgr)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        mgr._manager._field_grouping(x.coordinate_field_map_key)
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t0) * 1e3)
    res["first_grouping_ms"] = min(times)
    x = ME.TensorField(feats.clone().requires_grad_(True), pts)
    s = x.sparse()
    assert len(s) == len(pts)
    for name, mode in (("max", ME.PoolingMode.GLOBAL_MAX_POOLING_KERNEL),
                       ("avg", ME.PoolingMode.GLOBAL_AVG_POOLING_KERNEL)):
        pool = ME.MinkowskiGlobalPooling(mode)
        for kind, inp in (("field", x), ("map", s)):
            with torch.no_grad():
                res[f"{name}_fwd_{kind}_ms"] = timed(lambda: pool(inp), iters)
            y = pool(inp)
            g = torch.randn_like(y.F)
            res[f"{name}_fwd_bwd_{kind}_ms"] = timed(
                lambda: torch.autograd.grad(pool(inp).F, inp.F, g), iters)
    return res


def pointnet_step(B, n_per, dtype, iters):
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(0)
    pts = torch.cat([torch.arange(B, device=dev).repeat_interleave(n_per)[:, None].float(),
                     torch.rand(B * n_per, 3, device=dev, generator=g) * 2 - 1], 1)
    feats = pts[:, 1:].clone().to(dtype)
    labels = torch.randint(0, 40, (B,), device=dev, generator=g)
    net = pointnet(ME, 3, 40).to(dev).to(dtype).train()
    opt = torch.optim.SGD(net.parameters(), lr=1e-3)

    def step():
        opt.zero_grad(set_to_none=True)
        out = net(ME.TensorField(feats, pts))
        loss = torch.nn.functional.cross_entropy(out.F.float(), labels[out.C[:, 0].long()])
        loss.backward()
        opt.step()
    return {"clouds": B, "points": B * n_per, "dtype": str(dtype), "step_ms": timed(step, iters)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    out = {"card": card(), "pooling": [], "pointnet": []}
    print(out["card"], flush=True)
    for dtype in (torch.float32, torch.bfloat16):
        r = pooling(8, 125_000, 1024, dtype, a.iters)
        print(r, flush=True)
        out["pooling"].append(r)
    for dtype in (torch.float32, torch.bfloat16):
        r = pointnet_step(32, 2048, dtype, a.iters)
        print(r, flush=True)
        out["pointnet"].append(r)
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
