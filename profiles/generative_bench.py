"""Device time of pruning, union and arithmetic on different coordinate maps (csrc/union.cu) against
the torch composition the reference itself uses for the same result, with CUDA events, in one call:

    python profiles/generative_bench.py [--iters 20] [--json out.json]

Shapes: 8 clouds x 100k rows, bf16, C in {32, 64, 128, 256}; pruning keeps half the rows, the two
union / mul inputs share half their rows.  Bytes are ALGORITHMIC (every feature row read or written
once, int64 / int32 row indices counted); the share is of the H100 SXM's 3.35 TB/s.  The kernel
rows use maps built beforehand; the "+ map" rows also build the map, as the first call on new
coordinates does (the insert and its host read of the row count).  Also one bf16
forward + backward step of examples/completion.py at the reference widths on 8 synthetic clouds,
and the share of the prune / union kernels in it from torch.profiler.  The card name and power
limit are recorded with the numbers."""
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
from minkowskiengine_b200 import _lib, backend as _C  # noqa: E402

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


def shape_rows(C, iters, B=8, n_per=100_000):
    dev = torch.device("cuda")
    n = B * n_per
    b = torch.arange(B, device=dev, dtype=torch.int32).repeat_interleave(n_per)
    i = torch.arange(n_per, device=dev, dtype=torch.int32).repeat(B)
    ca = torch.stack([b, i % 64, (i // 64) % 64, i // 4096], 1).int().contiguous()
    cb = ca.clone()
    cb[:, 1] += 32                                   # half the rows of b are rows of a
    g = torch.Generator(device=dev).manual_seed(0)
    x = ME.SparseTensor(torch.randn(n, C, device=dev, generator=g).bfloat16(), ca)
    y = ME.SparseTensor((torch.rand(n, C, device=dev, generator=g) + 0.5).bfloat16(), cb,
                        coordinate_manager=x.coordinate_manager)
    mgr = x.coordinate_manager._manager
    keep = torch.rand(n, device=dev, generator=g) < 0.5
    ok = mgr._prune(x.coordinate_map_key, keep)
    uidx, inv = mgr._prunes[(mgr._k(x.coordinate_map_key), ok)]
    m = uidx.numel()
    um = mgr._union([x.coordinate_map_key, y.coordinate_map_key])
    M = um.M
    u0, u1 = um.u
    ar = torch.arange(n, device=dev)
    F, G = x.F, y.F
    dy_p = torch.randn(m, C, device=dev).bfloat16()
    dy_u = torch.randn(M, C, device=dev).bfloat16()
    esz = 2
    shared = 2 * n - M

    def zeros_assign_union():
        out = torch.zeros(M, C, dtype=F.dtype, device=dev)
        out[u0] += F[ar]
        out[u1] += G[ar]
        return out

    def torch_union_bwd():
        g0 = torch.zeros_like(F)
        g0[ar] = dy_u[u0]
        g1 = torch.zeros_like(G)
        g1[ar] = dy_u[u1]
        return g0, g1

    def torch_mul():
        out = torch.zeros(M, C, dtype=F.dtype, device=dev)
        out[u0] = F[ar]
        out[u1] = out[u1] * G[ar]
        return out

    fa = F.detach().clone().requires_grad_(True)
    fb = G.detach().clone().requires_grad_(True)

    def torch_mul_bwd():
        out = torch.zeros(M, C, dtype=F.dtype, device=dev)
        out[u0] = fa[ar]
        out[u1] = out[u1] * fb[ar]
        return torch.autograd.grad(out, [fa, fb], dy_u)

    xk, yk = x.coordinate_map_key, y.coordinate_map_key
    ik = mgr._k(xk)

    def prune_with_map():
        # what MinkowskiPruning.forward runs: the insert with the mask (one host read of the row
        # count), then the gather; the new map is dropped again so that the loop does not grow
        key = ME.CoordinateMapKey(4)
        out = _C.PruningForwardGPU(F, keep, xk, key, mgr)
        k = mgr._k(key)
        del mgr._maps[k], mgr._prunes[(ik, k)]
        return out

    def union_with_map():
        # a union map built afresh (the first `a + b` of two keys), then the fold
        mgr._unions.pop((ik, mgr._k(yk)))
        u = mgr._union([xk, yk])
        out = _C.union_fold_forward([F, G], u, _lib.UNION_ADD)
        del mgr._maps[u.key]
        return out

    rows = []
    ops = [
        ("prune fwd", lambda: _C._gather_rows(F, uidx, m), lambda: F[keep],
         2 * m * C * esz + 8 * m),
        ("prune fwd + map", prune_with_map, lambda: F[keep], 2 * m * C * esz + 8 * m),
        ("prune bwd", lambda: _C._gather_rows(dy_p, inv, n),
         lambda: torch.zeros_like(F).index_put_((keep,), dy_p), (m + n) * C * esz + 8 * n),
        ("union fwd", lambda: _C.union_fold_forward([F, G], um, _lib.UNION_ADD), zeros_assign_union,
         (2 * n + M) * C * esz + 8 * M),
        ("union fwd + map", union_with_map, zeros_assign_union, (2 * n + M) * C * esz + 8 * M),
        ("union bwd", lambda: _C.union_fold_backward(dy_u, [F, G], um, _lib.UNION_ADD), torch_union_bwd,
         4 * n * C * esz + 16 * n),
        ("mul fwd", lambda: _C.union_fold_forward([F, G], um, _lib.UNION_MUL), torch_mul,
         (2 * n + M) * C * esz + 8 * M),
        ("mul bwd", lambda: _C.union_fold_backward(dy_u, [F, G], um, _lib.UNION_MUL), torch_mul_bwd,
         (4 * n + 2 * shared) * C * esz + 16 * n + 16 * M),
    ]
    for name, native, ref, nbytes in ops:
        t_n = timed(native, iters)
        if name == "union fwd + map":
            mgr._unions[(ik, mgr._k(yk))] = um       # the map the other rows use
        t_r = timed(ref, iters)
        rows.append({"op": name, "C": C, "rows": n, "ms": t_n, "torch_ms": t_r, "bytes": nbytes,
                     "GBs": nbytes / t_n / 1e6, "share": nbytes / t_n / 1e6 / PEAK_GBS})
    return rows


def completion_step(iters):
    from examples.completion import completion_loss, completion_net, shell_pair
    dev = torch.device("cuda")
    torch.manual_seed(0)
    net = completion_net(ME).to(dev).train()
    pairs = [shell_pair(40.0, seed=100 + b, batch=b) for b in range(8)]
    partial = torch.cat([p for p, _ in pairs]).to(dev)
    full = torch.cat([f for _, f in pairs]).to(dev)

    def step():
        x = ME.SparseTensor(torch.ones(len(partial), 1, dtype=torch.bfloat16, device=dev), partial)
        tkey, _ = x.coordinate_manager.insert_and_map(full, string_id="target")
        out_cls, targets, final = net(x, tkey)
        completion_loss(out_cls, targets).backward()
        net.zero_grad(set_to_none=True)
        return out_cls

    out_cls = step()
    sizes = [len(o) for o in out_cls]
    for _ in range(2):
        step()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(iters):
        step()
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3 / iters
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    total = prune = union = 0.0
    for ev in prof.key_averages():
        t = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
        if t <= 0:
            continue
        total += t
        if "k_gather_rows" in ev.key:
            prune += t
        elif "k_union_fold" in ev.key:
            union += t
    return {"ms": ms, "input_voxels": int(len(partial)), "level_voxels": sizes,
            "kernel_ms": total / 1e3, "prune_ms": prune / 1e3, "union_ms": union / 1e3,
            "prune_share": prune / total if total else 0.0,
            "union_share": union / total if total else 0.0}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark measures the GPU; there is no CPU fallback"
    res = {"card": card(), "rows": []}
    print(json.dumps(res["card"]), flush=True)
    for C in (32, 64, 128, 256):
        for r in shape_rows(C, a.iters):
            res["rows"].append(r)
            print(f"{r['op']:15s} C={C:4d}  {r['ms']:.4f} ms  torch {r['torch_ms']:.4f} ms  "
                  f"{r['GBs']:.0f} GB/s  {100 * r['share']:.1f}% of 3.35 TB/s", flush=True)
    res["completion"] = completion_step(max(3, a.iters // 4))
    print("completion bf16 step:", json.dumps(res["completion"]), flush=True)
    res["card_after"] = card()
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
