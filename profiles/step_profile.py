"""Kernel-time breakdown of one bench step using torch.profiler (CUPTI activity records, no
kernel replay — cheap).  python profiles/step_profile.py [--clouds 8] [--dtype bf16] [--top 25]"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

import minkowskiengine_b200 as ME  # noqa: E402
from bench import make_batch  # noqa: E402
from examples.minkunet import minkunet  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clouds", type=int, default=8)
    ap.add_argument("--voxels", type=int, default=100000)
    ap.add_argument("--dtype", default="bf16")
    ap.add_argument("--model", default="MinkUNet34C")
    ap.add_argument("--top", type=int, default=25)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    dt = {"bf16": torch.bfloat16, "fp16": torch.float16, "fp32": torch.float32}[a.dtype]
    torch.manual_seed(0)
    net = minkunet(a.model, ME, 3, 20, 3).to(dev)
    opt = torch.optim.SGD(net.parameters(), lr=1e-2)
    crit = torch.nn.CrossEntropyLoss()
    c, f, l = make_batch(a.clouds, a.voxels, 0)
    c, f, l = c.to(dev), f.to(dev).to(dt), l.to(dev)

    def step():
        opt.zero_grad(set_to_none=True)
        out = net(ME.SparseTensor(f, c))
        loss = crit(out.F.float(), l)
        loss.backward()
        opt.step()

    for _ in range(3):
        step()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(3):
        step()
    e1.record()
    torch.cuda.synchronize()
    print(f"step time (no profiler): {e0.elapsed_time(e1) / 3:.2f} ms")
    print(f"peak memory allocated in a step: {torch.cuda.max_memory_allocated() / 2**20:.0f} MiB")
    with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
        step()
        torch.cuda.synchronize()
    rows = []
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = getattr(ev, "cuda_time_total", 0)
        if t and ev.device_type.name == "CUDA":
            rows.append((ev.key, ev.count, t / 1e3))
    tot = sum(r[2] for r in rows)
    print(f"total device kernel time in one step: {tot:.2f} ms over {sum(r[1] for r in rows)} launches")
    for k, n, ms in sorted(rows, key=lambda r: -r[2])[:a.top]:
        print(f"{ms:9.3f} ms {100 * ms / tot:5.1f}% x{n:5d}  {k[:110]}")


if __name__ == "__main__":
    main()
