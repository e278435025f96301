"""Times MinkowskiPoolingTranspose (k2s2) and TensorField.splat, forward and backward, with CUDA
events after a warm-up of every timed shape.

    python profiles/unpool_splat_bench.py [--reps 50]

Unpooling runs at a MinkUNet decoder size (SURVEY.md 8a: 39 234 -> 100 000 rows; the synthetic
surface cloud used here gives row counts near those, printed with each line) for C = 32 / 64 / 96 in
bf16 and fp32.  Splatting runs on a 200k-point D = 3 cloud at C = 32.  Prints the card's name and
power limit, then one JSON line per case: milliseconds per call and the bytes each kernel must move
(computed here from the shapes: neighbour tables, every input row read once, every output row
written once) over that time."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import minkowskiengine_b200 as ME  # noqa: E402
from minkowskiengine_b200 import backend  # noqa: E402


def timed(fn, reps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def surface_cloud(n_target=100_000, seed=0):
    """Unique stride-1 voxels on the surfaces of spheres in 4 clouds, about n_target rows."""
    g = torch.Generator().manual_seed(seed)
    pts = []
    per = n_target // 4
    for b in range(4):
        d = torch.randn(per * 3, 3, generator=g)
        d = d / d.norm(dim=1, keepdim=True) * 45.0
        c = torch.cat([torch.full((len(d), 1), b), torch.floor(d)], 1).int()
        pts.append(torch.unique(c, dim=0)[:per])
    return torch.cat(pts)


def report(case, ms, nbytes, **kw):
    out = dict(case=case, ms=round(ms, 4), bytes=int(nbytes), gbps=round(nbytes / (ms * 1e-3) / 1e9, 1))
    out.update(kw)
    print(json.dumps(out), flush=True)


def unpool(C, dtype, reps):
    coords = surface_cloud()
    x = ME.SparseTensor(torch.ones(len(coords), 1), coords, device="cuda")
    y = ME.MinkowskiSumPooling(kernel_size=2, stride=2, dimension=3)(x)
    mgr = x.coordinate_manager._manager
    kg = ME.KernelGenerator(kernel_size=2, stride=2, dimension=3)
    args = (kg.kernel_size, kg.kernel_stride, kg.kernel_dilation, kg.region_type, kg.region_offsets)
    feats = torch.randn(len(y), C, device="cuda").to(dtype)
    fwd = lambda: backend.LocalPoolingTransposeForwardGPU(  # noqa: E731
        feats, *args, False, ME.PoolingMode.LOCAL_SUM_POOLING, y.coordinate_map_key,
        x.coordinate_map_key, mgr)
    out, nnz = fwd()
    g = torch.randn_like(out)
    bwd = lambda: backend.LocalPoolingTransposeBackwardGPU(  # noqa: E731
        feats, g, nnz, *args, ME.PoolingMode.LOCAL_SUM_POOLING, y.coordinate_map_key,
        x.coordinate_map_key, mgr)
    bwd()
    km = mgr._kernel_map(y.coordinate_map_key, x.coordinate_map_key, *args[:4], None, True, True)
    es = feats.element_size()
    n_in, n_out, K = len(y), len(x), km.K
    tag = dict(C=C, dtype=str(dtype).replace("torch.", ""), rows_in=n_in, rows_out=n_out)
    report("unpool_fwd", timed(fwd, reps), 4 * K * n_out + es * C * (n_in + n_out), **tag)
    report("unpool_bwd", timed(bwd, reps), 4 * K * n_in + es * C * (n_in + n_out), **tag)


def splat(C, dtype, reps, n=200_000):
    g = torch.Generator().manual_seed(1)
    pts = torch.cat([torch.randint(0, 4, (n, 1), generator=g).float(),
                     torch.rand(n, 3, generator=g) * 60], 1).cuda()
    x = torch.randn(n, C, generator=g).cuda().to(dtype)
    tf = ME.TensorField(x, pts)
    st = tf.splat()
    M = len(st)
    rows, w, group = tf._splat[st.coordinate_map_key]
    K = rows.size(1)
    es = x.element_size()
    tag = dict(C=C, dtype=str(dtype).replace("torch.", ""), points=n, voxels=M)

    def build():
        t = ME.TensorField(x, pts)
        t.splat()
    report("splat_map_and_fwd", timed(build, reps), 4 * n * 4 + 4 * n * K * 4 * 3 + es * C * (n + M),
           **tag)
    fwd = lambda: ME.interpolation.interp_adjoint(x, rows, w, M, group)  # noqa: E731
    gv = torch.randn(M, C, device="cuda").to(dtype)
    bwd = lambda: backend.interp_forward(gv, rows, w)  # noqa: E731
    # forward: perm + start + weights, every point row read once, every voxel row written once
    report("splat_fwd", timed(fwd, reps), 4 * n * K * 2 + 4 * (M + 1) + es * C * (n + M), **tag)
    report("splat_bwd", timed(bwd, reps), 4 * n * K * 2 + es * C * (n + M), **tag)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "unpool_splat_bench.py measures on the GPU only"
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                          "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": torch.cuda.get_device_name(), "nvidia_smi": smi}), flush=True)
    for dtype in (torch.bfloat16, torch.float32):
        for C in (32, 64, 96):
            unpool(C, dtype, a.reps)
    splat(32, torch.bfloat16, a.reps)
    splat(32, torch.float32, a.reps)


if __name__ == "__main__":
    main()
