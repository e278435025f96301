"""Device time of the per-cloud ops (csrc/global.cu) against a torch index_add_ / scatter_reduce
composition of the same result, with CUDA events, in one call:

    python profiles/global_bench.py [--iters 20] [--json out.json]

Shapes: 8 clouds x 100k rows at C in {32, 64, 128, 256} and 64 clouds x 2k rows at C = 512, bf16;
plus one ResNet14 bf16 forward+backward step at 8 x 100k.  Bytes are ALGORITHMIC (every [n, C]
operand read or written once, [B, C] terms ignored); GB/s is against the H100 SXM's 3.35 TB/s.
The card name and power limit are recorded with the numbers."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import minkowskiengine_b200 as ME  # noqa: E402
from minkowskiengine_b200 import backend as _C  # noqa: E402

PEAK_GBS = 3350.0


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


def shape_rows(B, n_per, C, iters):
    dev = torch.device("cuda")
    n = B * n_per
    b = torch.arange(B, device=dev, dtype=torch.int32).repeat_interleave(n_per)
    i = torch.arange(n_per, device=dev, dtype=torch.int32).repeat(B)
    coords = torch.stack([b, i % 64, (i // 64) % 64, i // 4096], 1).int().contiguous()
    x = ME.SparseTensor(torch.randn(n, C, device=dev).bfloat16(), coords)
    mgr, key = x.coordinate_manager._manager, x.coordinate_map_key
    F = x.F
    dy = torch.randn_like(F)
    grp = mgr._origin_grouping(key)
    okey = ME.CoordinateMapKey(4)
    seg = grp.row_seg.long()
    g = torch.randn(B, C, device=dev).bfloat16()
    esz = 2
    nc = n * C * esz
    rows = []

    def add(op, ms, nbytes, torch_ms):
        rows.append({"B": B, "rows_per_cloud": n_per, "C": C, "op": op, "ms": ms,
                     "GBs": nbytes / ms / 1e6, "of_peak": nbytes / ms / 1e6 / PEAK_GBS,
                     "torch_ms": torch_ms})

    for name, mode in (("sum", ME.PoolingMode.GLOBAL_SUM_POOLING_KERNEL),
                       ("avg", ME.PoolingMode.GLOBAL_AVG_POOLING_KERNEL),
                       ("max", ME.PoolingMode.GLOBAL_MAX_POOLING_KERNEL)):
        out, aux = _C.GlobalPoolingForwardGPU(F, mode, key, okey, mgr)
        ms = timed(lambda: _C.GlobalPoolingForwardGPU(F, mode, key, okey, mgr), iters)
        if name == "max":
            t = timed(lambda: torch.full((B, C), float("-inf"), device=dev, dtype=F.dtype)
                      .scatter_reduce_(0, seg[:, None].expand(-1, C), F, "amax"), iters)
        else:
            t = timed(lambda: torch.zeros(B, C, device=dev, dtype=F.dtype).index_add_(0, seg, F),
                      iters)
        add(f"global_{name}_fwd", ms, nc, t)
        gb = out.contiguous()
        ms = timed(lambda: _C.GlobalPoolingBackwardGPU(F, gb, aux, mode, key, okey, mgr), iters)
        t = timed(lambda: gb.index_select(0, seg), iters)
        add(f"global_{name}_bwd", ms, nc, t)
    for name, mode in (("add", ME.BroadcastMode.ELEMENTWISE_ADDITON),
                       ("mul", ME.BroadcastMode.ELEMENTWISE_MULTIPLICATION)):
        ms = timed(lambda: _C.BroadcastForwardGPU(F, g, mode, key, okey, mgr), iters)
        t = timed((lambda: F + g.index_select(0, seg)) if name == "add"
                  else (lambda: F * g.index_select(0, seg)), iters)
        add(f"broadcast_{name}_fwd", ms, 2 * nc, t)
        ms = timed(lambda: _C.BroadcastBackwardGPU(F, g, dy, mode, key, okey, mgr), iters)
        if name == "add":
            t = timed(lambda: torch.zeros(B, C, device=dev, dtype=F.dtype).index_add_(0, seg, dy),
                      iters)
            nbytes = nc
        else:
            t = timed(lambda: (dy * g.index_select(0, seg),
                               torch.zeros(B, C, device=dev, dtype=F.dtype)
                               .index_add_(0, seg, dy * F)), iters)
            nbytes = 4 * nc          # dy, g-broadcast product out; dy, x for the reduction
        add(f"broadcast_{name}_bwd", ms, nbytes, t)
    norm = ME.MinkowskiInstanceNormFunction
    xf = F.detach().requires_grad_(True)

    def inorm_fwd():
        return norm.apply(xf, key, None, x.coordinate_manager)

    def torch_inorm(v):
        cnt = torch.zeros(B, device=dev).index_add_(0, seg, torch.ones(n, device=dev))[:, None]
        mean = torch.zeros(B, C, device=dev).index_add_(0, seg, v.float()) / cnt
        c = v.float() - mean.index_select(0, seg)
        var = torch.zeros(B, C, device=dev).index_add_(0, seg, c * c) / cnt
        return (c * torch.rsqrt(var + 1e-8).index_select(0, seg)).to(v.dtype)

    ms = timed(inorm_fwd, iters)
    t = timed(lambda: torch_inorm(F), iters)
    add("instnorm_fwd", ms, 4 * nc, t)      # read x twice, centred fp32 write + read (2x), write y
    y = inorm_fwd()
    ms = timed(lambda: torch.autograd.grad(y, xf, dy, retain_graph=True), iters)
    xt = F.detach().requires_grad_(True)
    yt = torch_inorm(xt)
    t = timed(lambda: torch.autograd.grad(yt, xt, dy, retain_graph=True), iters)
    add("instnorm_bwd", ms, 5 * nc, t)      # dy twice, y twice, write dx
    return rows


def resnet_step(iters):
    from examples.resnet import resnet
    from examples.synthetic import surface_cloud
    dev = torch.device("cuda")
    coords = torch.cat([surface_cloud(100_000, seed=b, batch=b) for b in range(8)]).to(dev)
    feats = torch.rand(len(coords), 3, device=dev).bfloat16()
    labels = torch.randint(0, 40, (8,), device=dev)
    torch.manual_seed(0)
    net = resnet("ResNet14", ME, 3, 40, 3).to(dev).train()

    def step():
        with torch.autocast("cuda", dtype=torch.bfloat16):     # the linear head in bf16
            out = net(ME.SparseTensor(feats, coords))
        loss = torch.nn.functional.cross_entropy(out.F.float(), labels[out.C[:, 0].long()])
        loss.backward()

    for _ in range(2):
        step()
    return {"resnet14_bf16_8x100k_fwd_bwd_ms": timed(step, max(3, iters // 4))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    res = {"card": card(), "rows": []}
    for C in (32, 64, 128, 256):
        res["rows"] += shape_rows(8, 100_000, C, a.iters)
    res["rows"] += shape_rows(64, 2_000, 512, a.iters)
    res.update(resnet_step(a.iters))
    print(f"# {res['card']['name']}, power limit {res['card']['power_limit']}")
    print("| B x rows | C | op | ms | GB/s | of 3.35 TB/s | torch ms | torch / native |")
    print("|---|---|---|---|---|---|---|---|")
    for r in res["rows"]:
        print(f"| {r['B']} x {r['rows_per_cloud']} | {r['C']} | {r['op']} | {r['ms']:.3f} | "
              f"{r['GBs']:.0f} | {100 * r['of_peak']:.0f} % | {r['torch_ms']:.3f} | "
              f"{r['torch_ms'] / r['ms']:.2f} |")
    print(f"ResNet14 bf16 8 x 100k forward+backward: {res['resnet14_bf16_8x100k_fwd_bwd_ms']:.2f} ms")
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
