"""Worker for tests/test_gpu_zz_syncbn_fp8.py: run under torch.distributed.run (or alone with
WORLD_SIZE unset = one rank), with MEB200_SYNCBN_PEER choosing the exchange (1: NVLink peer memory
where symmetric memory is available, 0: NCCL all-reduce).  Every rank builds the same [n, C]
matrix and keeps its slice of the rows (the last rank none in one case), and runs the synchronised
batch norm forward + backward on the slice twice: without and with the fp8 copies of delayed
scaling (the e4m3 copy of y, the e5m2 copy of dx).  Every output must be the same bits, and the
copies the torch expression of y and dx at their scales, with their amaxes recorded."""
import os
import sys
import types

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from minkowskiengine_b200 import normalization as N  # noqa: E402
from minkowskiengine_b200.fp8_delayed import _BnStep  # noqa: E402


def _bytes(t):
    return t.contiguous().view(torch.uint8)


def _expect(v, inv, dt, M):
    return (v.float() * inv).clamp(-M, M).to(dt).view(torch.uint8)


def _amax(v):
    return float(v.float().abs().max()) if v.numel() else 0.0


def _run(x, g, res, bn, group, fp8):
    xs = x.clone().requires_grad_(True)
    rs = res.clone().requires_grad_(True)
    for p in (bn.weight, bn.bias):
        p.grad = None
    y = N._batch_norm(bn, xs, group, relu=True, residual=rs, fp8=fp8)
    y.backward(g)
    return [y.detach(), xs.grad, rs.grad, bn.weight.grad.clone(), bn.bias.grad.clone(),
            bn.running_mean.clone(), bn.running_var.clone()]


def main():
    rank = int(os.environ.get("RANK", 0))
    world = int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", 0))
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "29533")
    dev = torch.device("cuda", local)
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    group = dist.group.WORLD
    try:
        for dtype in (torch.float32, torch.bfloat16):
            for n, C, empty_last in ((6001, 32, False), (20000, 96, False), (5000, 64, True)):
                torch.manual_seed(n + C)
                x = (torch.randn(n, C) * 2.0 + torch.linspace(-3, 3, C)).to(dev).to(dtype)
                g = torch.randn(n, C).to(dev).to(dtype)
                r = torch.randn(n, C).to(dev).to(dtype)
                parts = world - 1 if empty_last and world > 1 else world
                lo, hi = (rank * n // parts, (rank + 1) * n // parts) if rank < parts else (n, n)
                if empty_last and world == 1:
                    lo = hi = n                           # the one rank has no rows
                runs = []
                for with_fp8 in (False, True):
                    bn = torch.nn.SyncBatchNorm(C).to(dev)
                    with torch.no_grad():
                        bn.weight.copy_(torch.linspace(0.5, 1.5, C))
                        bn.bias.copy_(torch.linspace(-1, 1, C))
                    step = None
                    if with_fp8:
                        q = torch.empty(hi - lo, C, dtype=torch.uint8, device=dev)
                        ys = torch.tensor([1 / 64.0, 64.0], device=dev)
                        gs = torch.tensor([1 / 8192.0, 8192.0], device=dev)
                        grad = types.SimpleNamespace(scale=gs, slot=torch.zeros(1, device=dev),
                                                     shadow=None)
                        step = _BnStep(None, None, (q, ys, torch.zeros(1, device=dev)), grad)
                    runs.append((_run(x[lo:hi], g[lo:hi], r[lo:hi], bn, group, step), step))
                (plain, _), (got, step) = runs
                same = all(torch.equal(_bytes(a), _bytes(b)) for a, b in zip(plain, got))
                q, ys, yslot = step.y_out
                y, dx = got[0], got[1]
                ok_y = torch.equal(q, _expect(y, ys[1], torch.float8_e4m3fn, 448.0)) and \
                    float(yslot) == _amax(y)
                ok_dx = hi == lo or (
                    torch.equal(step.grad.shadow[0],
                                _expect(dx, step.grad.scale[1], torch.float8_e5m2, 57344.0))
                    and float(step.grad.slot) == _amax(dx))
                peer = any(v is not None for v in N._PeerExchange._cache.values())
                ok = same and step.written and ok_y and ok_dx
                print(f"rank {rank} {dtype} n={n} C={C} rows={hi - lo} peer={peer}: same {same} "
                      f"y copy {ok_y} dx copy {ok_dx} {'ok' if ok else 'FAIL'}", flush=True)
                if not ok:
                    sys.exit(1)
        print(f"rank {rank}: SYNCBN_FP8_OK", flush=True)
    finally:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
