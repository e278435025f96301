"""Times the dense-tensor interop, native kernels against the torch compositions they replace, with
CUDA events after a warm-up of every timed shape, alternating the two in the same run.

    python profiles/dense_bench.py [--reps 30] [--rounds 3]

A 100k-voxel surface cloud (examples/synthetic.py), the grid sized to the cloud, C = 16 / 128 in
bf16 and fp32:
  rows_to_dense   SparseTensor.dense forward   vs  zeros + index-put through a permuted view
  dense_to_rows   its backward                 vs  an index-get through the permuted view
  to_sparse       non-zero cells + features    vs  abs().sum() + where + stack + index-get
Prints the card's name and power limit, then one JSON line per case and path: milliseconds per call
(the median of the rounds), the bytes the operation must move (computed here from the shapes: the
volume written or read once, the rows read or written once, the int32 coordinates), that over the
time, and its share of the H100 SXM data sheet's 3.35 TB/s."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import minkowskiengine_b200 as ME  # noqa: E402
from examples.synthetic import surface_cloud  # noqa: E402
from minkowskiengine_b200 import dense as MD  # noqa: E402

PEAK = 3.35e12


def timed(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def compare(case, native, torch_path, nbytes, reps, rounds, **tag):
    for fn in (native, torch_path):
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    ms = {"native": [], "torch": []}
    for _ in range(rounds):
        ms["native"].append(timed(native, reps))
        ms["torch"].append(timed(torch_path, reps))
    for path, v in ms.items():
        t = statistics.median(v)
        bps = nbytes / (t * 1e-3)
        print(json.dumps(dict(case=case, path=path, ms=round(t, 4), ms_rounds=[round(x, 4) for x in v],
                              bytes=int(nbytes), gbps=round(bps / 1e9, 1),
                              share_of_3350_gbps=round(bps / PEAK, 3), **tag)), flush=True)


def run(C, dtype, reps, rounds):
    coords = surface_cloud(100_000, seed=0).cuda()
    n, es = len(coords), torch.empty(0, dtype=dtype).element_size()
    f = torch.randn(n, C, device="cuda").to(dtype)
    f[f == 0] = 1
    x = ME.SparseTensor(f, coords)
    lo = coords[:, 1:].min(0).values
    origin = lo.tolist()
    idx = (coords[:, 0].long(),) + tuple((coords[:, 1 + i] - lo[i]).long() for i in range(3))
    d0 = x.dense()[0]
    shape = list(d0.shape)
    cells = d0.numel() // C
    cmap = x.coordinate_manager._manager._get(x.coordinate_map_key)
    tag = dict(C=C, dtype=str(dtype).replace("torch.", ""), rows=n, grid=shape[2:], cells=cells)
    volume = es * C * cells

    def old_coords():   # the int64 coordinate copies the old dense() made on every call
        c = coords.long()
        return (c[:, 0],) + tuple(c[:, 1 + i] - lo[i] for i in range(3))

    def old_dense_full():
        i = old_coords()
        d = torch.zeros(shape, dtype=dtype, device="cuda")
        d.permute(0, 2, 3, 4, 1)[i] = f
        return d

    out = torch.empty(shape, dtype=dtype, device="cuda")
    assert torch.equal(MD.rows_to_dense(f, cmap, out, 1, origin), old_dense_full())
    # volume written once, rows read once, one table probe (4 B) per cell
    compare("rows_to_dense", lambda: MD.rows_to_dense(f, cmap, out, 1, origin), old_dense_full,
            volume + es * C * n + 4 * cells, reps, rounds, **tag)
    g = torch.randn(shape, device="cuda").to(dtype)
    assert torch.equal(MD.dense_to_rows(g, coords, 1, origin), g.permute(0, 2, 3, 4, 1)[idx])
    # the rows' cells read (a 32-byte sector per element in a channel-first volume is the
    # hardware's cost, not counted), rows written once, coordinates read once
    compare("dense_to_rows", lambda: MD.dense_to_rows(g, coords, 1, origin),
            lambda: g.permute(0, 2, 3, 4, 1)[old_coords()], 2 * es * C * n + 16 * n, reps, rounds,
            **tag)

    def old_to_sparse():
        b = torch.where(torch.abs(d0).sum(1) != 0)
        c = torch.stack(b, dim=1).int()
        return c, d0.permute(0, 2, 3, 4, 1)[b]

    def new_to_sparse():
        c = MD.nonzero_coordinates(d0, 1)
        return c, MD.dense_to_rows(d0, c, 1)

    (c0, f0), (c1, f1) = new_to_sparse(), old_to_sparse()
    assert torch.equal(c0, c1) and torch.equal(f0, f1) and len(c0) == n
    # volume read once, coordinates written once, rows read and written once
    compare("to_sparse", new_to_sparse, old_to_sparse, volume + 16 * n + 2 * es * C * n, reps,
            rounds, **tag)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "dense_bench.py measures on the GPU only"
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                          "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": torch.cuda.get_device_name(), "nvidia_smi": smi}), flush=True)
    for dtype in (torch.bfloat16, torch.float32):
        for C in (16, 128):
            run(C, dtype, a.reps, a.rounds)


if __name__ == "__main__":
    main()
