"""Times the channel-wise convolution kernels (forward, input gradient, weight gradient) in bf16 on
8 clouds x 100k voxels of examples.synthetic.surface_cloud, the generator bench.py uses, for
C in {32, 64, 128, 256} and k in {3, 5, 7}, next to the reference's torch composition (one
`out[o] += x[i] * W[k]` per offset, backward by autograd) on the same kernel maps; then one bf16
forward + backward step of examples/convnext.py on the same clouds.

    python profiles/chwise_bench.py [--reps 20] [--torch-reps 5]

Kernel maps (both tables, and the pair lists of the torch composition) are built before any timing
and excluded from the times.  Every shape is warmed up first; each time is CUDA events around
`reps` launches.  Prints one JSON line per row: milliseconds per call, the compulsory bytes
(computed here from the shapes: features in and out, fp32 weights, the int32 table) and their share
of the 3.35 TB/s HBM3 bound of an H100 SXM.  The card's name and power limit are read in the same
run."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import minkowskiengine_b200 as ME  # noqa: E402
from minkowskiengine_b200 import _lib  # noqa: E402

HBM = 3.35e12


def timed(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return {"gpu": torch.cuda.get_device_name(), "nvidia_smi": q[0] if q else "unavailable"}


def clouds(n_clouds, n_voxels):
    from examples.synthetic import surface_cloud
    return torch.cat([surface_cloud(n_voxels, seed=j, batch=j) for j in range(n_clouds)], 0)


def gather(x, W, nbr, y):
    lib = _lib.load()
    K, n_rows = nbr.shape
    _lib.check(lib.meb200_chwise_gather(
        _lib.ptr(x), _lib.dtype_code(x.dtype), x.shape[0], x.shape[1], _lib.ptr(W), _lib.ptr(nbr),
        K, n_rows, _lib.ptr(y), _lib.current_stream()))


def wgrad(x, g, nbr, dW, ws):
    lib = _lib.load()
    K, n_out = nbr.shape
    _lib.check(lib.meb200_chwise_wgrad(
        _lib.ptr(x), _lib.ptr(g), _lib.dtype_code(x.dtype), x.shape[0], x.shape[1], _lib.ptr(nbr),
        K, n_out, _lib.ptr(dW), _lib.ptr(ws), 0 if ws is None else ws.numel(),
        _lib.current_stream()))


def torch_forward(x, W, pairs, n_out):
    """The reference's composition (MinkowskiChannelwiseConvolution.py:178-183)."""
    out = x.new_zeros(n_out, x.shape[1])
    for k, (i, o) in pairs:
        out[o] += x[i] * W[k]
    return out


def layer_rows(coords, C, k, reps, torch_reps):
    dtype = torch.bfloat16
    g = torch.Generator().manual_seed(k * 1000 + C)
    x = (torch.rand(len(coords), C, generator=g) - 0.5).to(dtype).cuda()
    st = ME.SparseTensor(x, coords.cuda())
    layer = ME.MinkowskiChannelwiseConvolution(C, kernel_size=k, dimension=3).cuda()
    kg = layer.kernel_generator
    out_key = ME.CoordinateMapKey(4)
    mgr = st.coordinate_manager._manager
    ok, _ = mgr._stride(st.coordinate_map_key, kg.kernel_stride)
    out_key.set_key(list(ok[0]), ok[1])
    km = mgr._kernel_map(st.coordinate_map_key, out_key, kg.kernel_size, kg.kernel_stride,
                         kg.kernel_dilation, kg.region_type, kg.region_offsets, False, False)
    K, n_out, n_in = km.K, km.n_out, km.n_in
    out_nbr, in_nbr = km.out_nbr, km.in_nbr
    W = layer.kernel.detach().float().contiguous()
    go = (torch.rand(n_out, C, generator=g) - 0.5).to(dtype).cuda()
    y = torch.empty((n_out, C), dtype=dtype, device="cuda")
    gi = torch.empty_like(x)
    dW = torch.empty((K, C), dtype=torch.float32, device="cuda")
    nb = int(_lib.load().meb200_chwise_wgrad_workspace_bytes(n_out, C, K, _lib.BF16))
    ws = torch.empty(nb, dtype=torch.uint8, device="cuda") if nb else None
    pairs = [(kk, (io[0].long(), io[1].long())) for kk, io in km.to_dict().items()]
    n_pairs = sum(len(io[0]) for _, io in pairs)
    fns = {"forward": lambda: gather(x, W, out_nbr, y),
           "input_grad": lambda: gather(go, W, in_nbr, gi),
           "weight_grad": lambda: wgrad(x, go, out_nbr, dW, ws)}
    s = 2
    nbytes = {"forward": n_in * C * s + n_out * C * s + 4 * K * C + 4 * K * n_out,
              "input_grad": n_out * C * s + n_in * C * s + 4 * K * C + 4 * K * n_in,
              "weight_grad": n_in * C * s + n_out * C * s + 4 * K * C + 4 * K * n_out}
    for fn in fns.values():       # warm-up of every timed shape
        fn()
    torch.cuda.synchronize()
    base = {"k": k, "K": K, "C": C, "dtype": "bf16", "n_in": n_in, "n_out": n_out,
            "pairs": n_pairs}
    for name, fn in fns.items():
        ms = timed(fn, reps)
        print(json.dumps({**base, "case": name, "ms": round(ms, 4), "bytes": nbytes[name],
                          "hbm_share": round(nbytes[name] / HBM / (ms * 1e-3), 3)}), flush=True)

    # the torch composition: forward, and its autograd backward (input and kernel gradients)
    Wb = W.to(dtype)
    try:
        with torch.no_grad():
            torch_forward(x, Wb, pairs, n_out)
            torch.cuda.synchronize()
            t_fwd = timed(lambda: torch_forward(x, Wb, pairs, n_out), torch_reps)
        xr, Wr = x.clone().requires_grad_(True), Wb.clone().requires_grad_(True)
        t_bwd = 0.0
        for rep in range(torch_reps + 1):
            out = torch_forward(xr, Wr, pairs, n_out)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out.backward(go)
            e1.record()
            torch.cuda.synchronize()
            if rep:                 # the first one is the warm-up
                t_bwd += e0.elapsed_time(e1) / torch_reps
            del out
            xr.grad = Wr.grad = None
        print(json.dumps({**base, "case": "torch_forward", "ms": round(t_fwd, 4)}), flush=True)
        print(json.dumps({**base, "case": "torch_backward", "ms": round(t_bwd, 4)}), flush=True)
    except torch.cuda.OutOfMemoryError:
        print(json.dumps({**base, "case": "torch", "ms": None, "note": "out of memory"}),
              flush=True)
    torch.cuda.empty_cache()


def convnext_step(coords, reps):
    from examples.convnext import convnext
    torch.manual_seed(0)
    net = convnext(ME, 3, 10, 3).cuda().train()
    feats = torch.rand(len(coords), 3, generator=torch.Generator().manual_seed(0))
    feats = feats.to(torch.bfloat16).cuda()
    labels = torch.arange(8, device="cuda") % 10
    c = coords.cuda()

    def step():
        net.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            out = net(ME.SparseTensor(feats, c))
            loss = torch.nn.functional.cross_entropy(out.F.float(), labels[out.C[:, 0].long()])
        loss.backward()

    for _ in range(3):
        step()
    torch.cuda.synchronize()
    ms = timed(step, reps)
    print(json.dumps({"case": "convnext_step", "dtype": "bf16 (autocast)", "voxels": len(coords),
                      "ms": round(ms, 3), "note": "forward + backward, coordinate maps included"}),
          flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--torch-reps", type=int, default=5)
    ap.add_argument("--clouds", type=int, default=8)
    ap.add_argument("--voxels", type=int, default=100_000)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "chwise_bench.py measures on the GPU only"
    print(json.dumps(card()), flush=True)
    coords = clouds(a.clouds, a.voxels)
    for k in (3, 5, 7):
        for C in (32, 64, 128, 256):
            layer_rows(coords, C, k, a.reps, a.torch_reps)
    convnext_step(coords, 10)
    print(json.dumps(card()), flush=True)


if __name__ == "__main__":
    main()
