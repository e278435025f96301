#!/usr/bin/env python
"""Benchmark of the sparse-convolution hot path.  Default workload = BASELINE.json configs[3]:
MinkUNet34C forward+backward(+SGD) over synthetic 100k-voxel clouds, batch 8 per rank,
reporting active-voxels/s.  Contract: see the one JSON line printed by rank 0.

    python bench.py [--gpus N] [--steps K] [--warmup W] [--impl ours|reference] [--config cfgN]
                    [--dump-outputs DIR]
    python -m torch.distributed.run --nproc-per-node N ... bench.py --gpus N ...

--config selects the BASELINE.json configuration the line is measured on:
  cfg3 (default)  MinkUNet34C, 8 clouds x 100k voxels per rank, DDP over the ranks
  cfg2            MinkUNet14 on one 50k-voxel cloud, fwd+bwd(+SGD)
  cfg1            single MinkowskiConvolution k=3 s=2, 100k coords, 64 -> 128, bf16
  cfg4            4-D MinkowskiConvolution k=3 (K=81), 200k coordinate draws, C = 32

A "step" = fresh SparseTensor (all coordinate maps and kernel maps rebuilt, as in the
reference's examples/multigpu_ddp.py:103-106) -> forward -> loss -> backward (DDP gradient
all-reduce when N>1) -> SGD step.  For cfg1 the maps are built once and the step is the layer's
forward + backward alone (the gather-GEMM-scatter north_star asks a roofline for); `e2e` always
starts from host buffers and rebuilds every map.
  value : inputs already resident in HBM when the timed region starts
  e2e   : the same step driven through the public API from PINNED HOST buffers — H2D copy of
          coordinates/features/labels and a D2H read of the loss inside the timed region
--dump-outputs DIR writes what the last timed step computed (rank 0) as DIR/<name>.npy, float32 or
float64, at most 64 MB in all (seeded row / element samples of the large arrays).  The inputs and
the seeded weights depend only on the arguments, so two builds can be compared output for output.
--impl reference times the reference's own CPU implementation (oracle/_ref, compiled from
the reference sources by oracle/build_ref.py) on the host cores, on a bounded sample.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

UNIT = "voxels/s"
# algorithmic conv FLOPs per voxel, fwd+bwd (SURVEY.md §8d: 601.6 GFLOP / 100k voxels)
FLOP_PER_VOXEL_FWD_BWD = 601.6e9 / 100_000

CONFIGS = {
    "cfg3": dict(kind="net", model="MinkUNet34C", clouds=8, voxels=100_000,
                 metric="active-voxels/sec MinkUNet34C fwd+bwd @100k pts, 1/2/4/8 H100 vs CPU ref",
                 what="BASELINE configs[3]"),
    "cfg2": dict(kind="net", model="MinkUNet14", clouds=1, voxels=50_000,
                 metric="active-voxels/sec MinkUNet14 fwd+bwd @50k pts, 1xH100 vs CPU ref",
                 what="BASELINE configs[2]"),
    "cfg1": dict(kind="conv", D=3, voxels=100_000, c_in=64, c_out=128, ks=3, stride=2,
                 metric="active-voxels/sec single MinkowskiConvolution k3 s2 64->128 bf16 "
                        "fwd+bwd @100k coords, 1xH100 vs CPU ref",
                 what="BASELINE configs[1]"),
    "cfg4": dict(kind="conv", D=4, voxels=200_000, c_in=32, c_out=32, ks=3, stride=1,
                 metric="active-voxels/sec 4-D (D=4) MinkowskiConvolution k3 C=32: hashing + "
                        "kernel map (K=81) + fwd+bwd @200k coordinate draws, 1xH100 vs CPU ref",
                 what="BASELINE configs[4]"),
}
# bf16 network on bf16-rounded inputs vs the reference's fp32 loss (tests/golden/bench_step0_loss.json):
# the loss is a mean over >= 50k voxels of per-voxel errors of ~1e-2 relative (see
# tests/test_gpu_network.py for the derivation), observed ~1e-3
LOSS_TOL = 2e-2


def parse_args():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--config", default="cfg3", choices=sorted(CONFIGS))
    ap.add_argument("--dtype", default=os.environ.get("MEB200_BENCH_DTYPE", "bf16"),
                    choices=["bf16", "fp16", "fp32"])
    ap.add_argument("--clouds", type=int, default=None)
    ap.add_argument("--voxels", type=int, default=None)
    ap.add_argument("--model", default=None)
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None)
    a = ap.parse_args()
    cfg = dict(CONFIGS[a.config])
    if cfg["kind"] == "net":
        a.clouds = a.clouds or cfg["clouds"]
        a.model = a.model or cfg["model"]
    else:
        a.clouds = 1
    a.voxels = a.voxels or cfg["voxels"]
    a.cfg = cfg
    return a


# --------------------------------------------------------------------------------------
def make_batch(n_clouds, n_voxels, seed0):
    """Synthetic 'surface' clouds (SURVEY.md §8d generator), one batch index per cloud."""
    import torch
    from examples.synthetic import surface_cloud
    coords = torch.cat([surface_cloud(n_voxels, seed0 + j, batch=j) for j in range(n_clouds)], 0)
    g = torch.Generator().manual_seed(seed0)
    feats = torch.rand(len(coords), 3, generator=g)
    labels = torch.zeros(len(coords), dtype=torch.int64)
    return coords.contiguous(), feats, labels


def make_conv_inputs(cfg, n_draws, seed):
    """cfg1 / cfg4 inputs (SURVEY.md §8d): coordinates, features [n, c_in]."""
    import torch
    from examples.synthetic import surface_cloud
    g = torch.Generator().manual_seed(seed)
    if cfg["D"] == 3:
        coords = surface_cloud(n_draws, seed)
    else:   # 4-D: c = floor(45 v + 0.5 t), columns (b, x, y, z, t); duplicates are part of the load
        v = torch.randn(n_draws, 3, generator=g)
        v = v / v.norm(dim=1, keepdim=True)
        t = torch.randint(0, 8, (n_draws, 1), generator=g)
        r = 45.0 * (n_draws / 200_000) ** 0.5
        c = torch.floor(r * v + 0.5 * t).int()
        coords = torch.cat([torch.zeros(n_draws, 1, dtype=torch.int32), c, t.int()], 1)
    feats = torch.rand(len(coords), cfg["c_in"], generator=g)
    return coords.contiguous(), feats


def weights_digest(net):
    """Order-independent fingerprint of a network's parameters (seeded-init check)."""
    return float(sum(p.detach().double().abs().sum() for p in net.parameters()))


def load_peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.isfile(p):
        d = json.load(open(p))
        return {"hbm_gbs": d["hbm_gbs"], "bf16_tflops": d["bf16_tflops"],
                "bf16_tflops_sustained": d.get("bf16_tflops_sustained", d["bf16_tflops"]),
                "source": "measured"}
    # NVIDIA H100 SXM data sheet (700 W): 3.35 TB/s HBM3, 989 dense BF16 TFLOP/s
    return {"hbm_gbs": 3350.0, "bf16_tflops": 989.0, "bf16_tflops_sustained": 989.0,
            "source": "fallback (H100 SXM data sheet)"}


DUMP_LIMIT_BYTES = 64 << 20


def dump_outputs(out_dir, arrays, seed=0):
    """Writes {name: tensor} as out_dir/<name>.npy (float64 stays float64, everything else
    float32).  Arrays whose rows do not fit the remaining share of DUMP_LIMIT_BYTES are replaced
    by a fixed, seeded sample of rows (2-D) or elements (1-D), saved with the indices taken."""
    import numpy as np
    import torch
    os.makedirs(out_dir, exist_ok=True)
    share = DUMP_LIMIT_BYTES // max(1, len(arrays))
    for name, t in sorted(arrays.items()):
        a = t.detach().cpu()
        a = np.atleast_1d(a.double().numpy() if a.dtype == torch.float64 else a.float().numpy())
        row_bytes = a.itemsize * (a.size // max(1, a.shape[0]))
        keep = max(1, share // (row_bytes + 8))          # + 8: the float64 index of a kept row
        if a.nbytes > share and keep < a.shape[0]:
            idx = np.sort(np.random.default_rng(seed).choice(a.shape[0], keep, replace=False))
            np.save(os.path.join(out_dir, f"{name}.sample_index.npy"), idx.astype(np.float64))
            a = a[idx]
        np.save(os.path.join(out_dir, f"{name}.npy"), a)


class NvmlClockSampler:
    """SM clock + clock-event reasons read through NVML (nvidia_ml_py) every 20 ms from a
    thread, so that even a half-second timed region gets tens of samples.  `start()` returns
    False when NVML is not usable; the caller then falls back to the nvidia-smi sampler."""
    # nvmlClocksEventReason* bit masks (nvml.h)
    REASONS = {0x8: "hw_slowdown", 0x40: "hw_thermal_slowdown", 0x20: "sw_thermal_slowdown",
               0x4: "sw_power_cap", 0x80: "hw_power_brake_slowdown"}

    def __init__(self, index=0, period_s=0.02):
        self.index, self.period, self.sm, self.mask, self.mx = index, period_s, [], 0, None
        self._stop = threading.Event()

    def start(self):
        try:
            import pynvml
            pynvml.nvmlInit()
            self.nv = pynvml
            self.h = None
            try:   # CUDA_VISIBLE_DEVICES may renumber devices: match on the PCI address
                import torch
                pr = torch.cuda.get_device_properties(self.index)
                bus = f"{pr.pci_domain_id:08x}:{pr.pci_bus_id:02x}:{pr.pci_device_id:02x}.0"
                self.h = pynvml.nvmlDeviceGetHandleByPciBusId(bus.encode())
            except Exception:
                self.h = None
            if self.h is None:
                self.h = pynvml.nvmlDeviceGetHandleByIndex(self.index)
            self.mx = float(pynvml.nvmlDeviceGetMaxClockInfo(self.h, pynvml.NVML_CLOCK_SM))
            self._sample()
        except Exception:
            return False
        self.th = threading.Thread(target=self._loop, daemon=True)
        self.th.start()
        return True

    def _sample(self):
        self.sm.append(float(self.nv.nvmlDeviceGetClockInfo(self.h, self.nv.NVML_CLOCK_SM)))
        get = getattr(self.nv, "nvmlDeviceGetCurrentClocksEventReasons", None) or \
            self.nv.nvmlDeviceGetCurrentClocksThrottleReasons
        self.mask |= int(get(self.h))

    def _loop(self):
        while not self._stop.wait(self.period):
            try:
                self._sample()
            except Exception:
                return

    def stop(self):
        self._stop.set()
        self.th.join(timeout=2)
        sm = sorted(self.sm[1:] or self.sm)      # the first sample predates the timed region
        reasons = sorted(nm for bit, nm in self.REASONS.items() if self.mask & bit)
        return {"sm_mhz": sm[len(sm) // 2], "sm_max_mhz": self.mx, "reasons": reasons,
                "samples": len(sm), "source": "nvml"}


class ClockSampler:
    """nvidia-smi clocks/throttle reasons sampled every 200 ms during the timed region."""
    Q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")

    def __init__(self, index=0):
        self.lines, self.proc, self.index = [], None, index

    def start(self):
        try:
            self.proc = subprocess.Popen(
                ["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits",
                 "-i", str(self.index), "-lms", "200"], stdout=subprocess.PIPE,
                stderr=subprocess.DEVNULL, text=True)
            self.th = threading.Thread(target=self._pump, daemon=True)
            self.th.start()
        except Exception:
            self.proc = None

    def _pump(self):
        for ln in self.proc.stdout:
            self.lines.append(ln.strip())

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        try:
            self.proc.wait(timeout=5)
        except Exception:
            self.proc.kill()
        sm, mx, reasons = [], None, set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for ln in self.lines:
            f = [x.strip() for x in ln.split(",")]
            if len(f) < 7:
                continue
            try:
                sm.append(float(f[0])); mx = float(f[1])
            except ValueError:
                continue
            for nm, v in zip(names, f[3:7]):
                if v.lower().startswith("active"):
                    reasons.add(nm)
        sm.sort()
        med = sm[len(sm) // 2] if sm else None
        return {"sm_mhz": med, "sm_max_mhz": mx, "reasons": sorted(reasons), "samples": len(sm)}


# --------------------------------------------------------------------------------------
# The reference's own CPU implementation (oracle/_ref) on the host cores
# --------------------------------------------------------------------------------------
def _ref_threads():
    cores = os.cpu_count() or 1
    return cores, min(cores, 16)  # the reference caps itself at 16 (MinkowskiEngine/__init__.py:35-46)


def _ref_step_factory(args, REF):
    """-> (step() -> loss, voxels per step, sample description) for args.config on module REF."""
    import torch
    from examples.minkunet import minkunet
    cfg = args.cfg
    torch.manual_seed(0)
    if cfg["kind"] == "net":
        net = minkunet(args.model, REF, 3, 20, 3)
        opt = torch.optim.SGD(net.parameters(), lr=1e-2)
        crit = torch.nn.CrossEntropyLoss()
        # bounded sample: ONE cloud of the configured size (the repo arm runs `clouds` of them
        # per step; the metric is per voxel)
        coords, feats, labels = make_batch(1, args.voxels, seed0=0)

        def step():
            opt.zero_grad()
            out = net(REF.SparseTensor(feats, coords))
            loss = crit(out.F, labels)
            loss.backward()
            opt.step()
            return float(loss)
        return step, coords.shape[0], f"1 cloud x {coords.shape[0]} voxels per step ({args.model}, fp32)"
    D = cfg["D"]
    conv = REF.MinkowskiConvolution(cfg["c_in"], cfg["c_out"], kernel_size=cfg["ks"],
                                    stride=cfg["stride"], dimension=D)
    coords, feats = make_conv_inputs(cfg, args.voxels, seed=0)

    def step():
        conv.kernel.grad = None
        x = REF.SparseTensor(feats, coords)    # duplicates (4-D draws): first occurrence kept
        y = conv(x)
        loss = y.F.square().mean()
        loss.backward()
        return float(loss)
    return step, coords.shape[0], (f"{coords.shape[0]} coordinate draws per step, D={D} conv "
                                   f"{cfg['c_in']}->{cfg['c_out']} k{cfg['ks']} s{cfg['stride']}, "
                                   "maps rebuilt, fwd+bwd, fp32")


def run_reference(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    cores, threads = _ref_threads()
    import torch
    from oracle import ref
    torch.set_num_threads(threads)
    REF = ref.import_reference()
    step, n_vox, sample = _ref_step_factory(args, REF)
    for _ in range(args.warmup):
        step()
    t0 = time.perf_counter()
    for _ in range(args.steps):
        step()
    dt = time.perf_counter() - t0
    value = n_vox * args.steps / dt
    sample += f", {args.steps} steps after {args.warmup} warm-up"
    world = int(os.environ.get("WORLD_SIZE", "1"))
    line = {
        "impl": "reference", "metric": args.cfg["metric"], "value": value, "unit": UNIT,
        "n_gpus": args.gpus, "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": 1e3 * dt / args.steps, "higher_is_better": True, "scaling": "weak",
        "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": {"workload": f"{args.cfg['what']}; reference CPU path (oracle/_ref), maps rebuilt "
                               "every step",
                   "voxels_per_step": n_vox,
                   "note": ("ONE CPU process regardless of --gpus: at N>1 the driver's ratio "
                            "compares N GPUs with this single 16-thread process") if world > 1 else
                           "one CPU process, reference thread cap 16"},
        "cpu_baseline": {"value": value, "unit": UNIT, "cores": threads, "kind": "reference",
                         "sample": sample, "host_cores": cores,
                         "omp_num_threads": os.environ.get("OMP_NUM_THREADS")},
        "e2e": {"value": value, "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "gpu_launches": 0,
    }
    print(json.dumps(line), flush=True)


def cpu_baseline(args):
    """Bounded CPU sample of the same workload through the compiled reference."""
    import torch
    from oracle import ref
    cores, threads = _ref_threads()
    torch.set_num_threads(threads)
    try:
        REF = ref.import_reference()
    except Exception as e:
        return {"value": None, "unit": UNIT, "cores": threads, "kind": "reference",
                "sample": f"unavailable: {e}"}
    step, n_vox, sample = _ref_step_factory(args, REF)
    times = []
    for it in range(3):
        t0 = time.perf_counter()
        step()
        times.append(time.perf_counter() - t0)
    best = min(times[1:])
    return {"value": n_vox / best, "unit": UNIT, "cores": threads, "kind": "reference",
            "host_cores": cores,
            "sample": f"{sample}; min of 2 after 1 warm-up ({best:.3f} s/step)"}


# --------------------------------------------------------------------------------------
def _golden_loss(args):
    try:
        d = json.load(open(os.path.join(ROOT, "tests", "golden", "bench_step0_loss.json")))
    except (OSError, ValueError):
        return None
    for case in d["cases"].values():
        if (case["model"], case["clouds"], case["voxels"]) == (args.model, args.clouds, args.voxels):
            return case
    return None


def bind_to_gpu_numa_node(index):
    """Pins this rank's threads to the CPUs NVML reports as local to its GPU (the step is launch
    bound in places: a rank whose interpreter runs on the other socket pays for it on every
    launch, and a multi-rank step waits for the slowest rank).  Returns the number of CPUs in the
    mask, or None when NVML / the mask is unavailable (nothing changes then).
    MEB200_BENCH_AFFINITY=0 disables it."""
    if os.environ.get("MEB200_BENCH_AFFINITY", "1") in ("", "0"):
        return None
    try:
        import pynvml
        import torch
        pynvml.nvmlInit()
        try:
            bus = torch.cuda.get_device_properties(index).pci_bus_id
            dom = torch.cuda.get_device_properties(index).pci_domain_id
            dv = torch.cuda.get_device_properties(index).pci_device_id
            h = pynvml.nvmlDeviceGetHandleByPciBusId(f"{dom:08x}:{bus:02x}:{dv:02x}.0".encode())
        except Exception:                           # noqa: BLE001
            h = pynvml.nvmlDeviceGetHandleByIndex(index)
        words = (os.cpu_count() + 63) // 64
        mask = pynvml.nvmlDeviceGetCpuAffinity(h, words)
        cpus = {64 * w + b for w, m in enumerate(mask) for b in range(64) if (int(m) >> b) & 1}
        cpus &= set(os.sched_getaffinity(0))
        if len(cpus) >= 4:                          # never squeeze a rank onto a handful of cores
            os.sched_setaffinity(0, cpus)
            return len(cpus)
    except Exception:                               # noqa: BLE001
        pass
    return None


def run_ours(args):
    import torch
    import torch.distributed as dist
    import minkowskiengine_b200 as ME
    from examples.minkunet import minkunet

    cfg = args.cfg
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    numa_cpus = bind_to_gpu_numa_node(local_rank)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    dtype = {"bf16": torch.bfloat16, "fp16": torch.float16, "fp32": torch.float32}[args.dtype]
    is_net = cfg["kind"] == "net"
    loss_check = None
    flush_l2 = False
    ablate = []
    last = {}          # --dump-outputs: the arrays the last step computed

    torch.manual_seed(0)
    if is_net:
        net = minkunet(args.model, ME, 3, 20, 3)
        digest = weights_digest(net)
        net = net.to(dev)
        raw_net = net
        # MEB200_BENCH_ABLATE=nosyncbn,noddp,samedata: DIAGNOSIS ONLY (which part of the N>1 step
        # costs what); recorded in config.ablate, never a bench value.
        ablate = sorted(x for x in os.environ.get("MEB200_BENCH_ABLATE", "").split(",") if x)
        if world > 1 and "nosyncbn" not in ablate:
            net = ME.MinkowskiSyncBatchNorm.convert_sync_batchnorm(net)
        if world > 1 and "noddp" not in ablate:
            # SyncBN keeps the running statistics identical on every rank, so DDP's per-step
            # buffer broadcast is redundant; gradients live in the all-reduce buckets.
            # MEB200_DDP_PLAIN=1 restores the reference example's plain DDP
            # (examples/multigpu_ddp.py).
            ddp_kw = dict(broadcast_buffers=False, gradient_as_bucket_view=True)
            if os.environ.get("MEB200_DDP_BUCKET_MB"):      # A/B: all-reduce bucket size
                ddp_kw["bucket_cap_mb"] = int(os.environ["MEB200_DDP_BUCKET_MB"])
            if os.environ.get("MEB200_DDP_PLAIN", "0") not in ("", "0"):
                ddp_kw = {}
            net = torch.nn.parallel.DistributedDataParallel(net, device_ids=[local_rank], **ddp_kw)
        opt = torch.optim.SGD(net.parameters(), lr=1e-2)
        crit = torch.nn.CrossEntropyLoss()
        seed0 = 0 if "samedata" in ablate else rank * args.clouds
        coords_h, feats_h, labels_h = make_batch(args.clouds, args.voxels, seed0=seed0)
        host = [coords_h.pin_memory(), feats_h.pin_memory(), labels_h.pin_memory()]
        coords_d, labels_d = host[0].to(dev), host[2].to(dev)
        feats_d = host[1].to(dev).to(dtype)
        n_vox = coords_h.shape[0]

        def run(c, f, l):
            opt.zero_grad(set_to_none=True)
            out = net(ME.SparseTensor(f, c))
            loss = crit(out.F.float(), l)
            loss.backward()
            if args.dump_outputs:
                last.update(logits=out.F, loss=loss, **{
                    "grad." + n: p.grad for n, p in raw_net.named_parameters() if p.grad is not None})
            opt.step()
            return loss

        def step_resident():
            return run(coords_d, feats_d, labels_d)

        def step_e2e():
            c = host[0].to(dev, non_blocking=True)
            f = host[1].to(dev, non_blocking=True).to(dtype)
            l = host[2].to(dev, non_blocking=True)
            return float(run(c, f, l).item())           # D2H read of the step's result

        # ---- step-0 loss against the reference's (tests/golden/bench_step0_loss.json) -------
        if world == 1 and rank == 0 and dtype == torch.bfloat16:
            gold = _golden_loss(args)
            if gold is not None and abs(gold["weights_digest"] - digest) <= 1e-6 * abs(digest):
                with torch.no_grad():
                    l0 = float(crit(raw_net(ME.SparseTensor(feats_d, coords_d)).F.float(), labels_d))
                err = abs(l0 - gold["loss"]) / abs(gold["loss"])
                loss_check = {"step0_loss": l0, "reference_loss": gold["loss"], "rel_err": err,
                              "tol": LOSS_TOL, "ok": err < LOSS_TOL,
                              "source": "tests/golden/bench_step0_loss.json (compiled reference, fp32 CPU)"}
                assert err < LOSS_TOL, f"step-0 loss {l0} differs from the reference's {gold['loss']}"
            else:
                loss_check = {"ok": None, "note": "no stored reference loss for this configuration "
                                                  "or seeded weights differ"}
        h2d = sum(int(t.nbytes) for t in host)
    else:
        D = cfg["D"]
        conv = ME.MinkowskiConvolution(cfg["c_in"], cfg["c_out"], kernel_size=cfg["ks"],
                                       stride=cfg["stride"], dimension=D).to(dev)
        coords_h, feats_h = make_conv_inputs(cfg, args.voxels, seed=rank)
        host = [coords_h.pin_memory(), feats_h.pin_memory()]
        coords_d, feats_d = host[0].to(dev), host[1].to(dev).to(dtype)
        n_vox = coords_h.shape[0]

        def full(c, f):
            conv.kernel.grad = None
            x = ME.SparseTensor(f, c, requires_grad=True)   # duplicates: first occurrence kept
            y = conv(x)
            loss = y.F.float().square().mean()
            loss.backward()
            if args.dump_outputs:
                last.update(out=y.F, loss=loss, grad_kernel=conv.kernel.grad, grad_in=x.F.grad)
            return loss

        if D == 3:
            # cfg1: maps built once; the step is the layer's forward + backward alone, with an
            # L2 flush between iterations (inputs + outputs + table = 26 MB < 50 MB L2)
            x_fixed = ME.SparseTensor(feats_d, coords_d)
            y0 = conv(x_fixed)
            gout = torch.rand(y0.F.shape, device=dev).to(dtype)
            flush_l2 = True

            def step_resident():
                conv.kernel.grad = None
                f = x_fixed.F.detach().requires_grad_(True)
                y = conv(ME.SparseTensor(f, coordinate_map_key=x_fixed.coordinate_map_key,
                                         coordinate_manager=x_fixed.coordinate_manager))
                y.F.backward(gout)
                if args.dump_outputs:
                    last.update(out=y.F, grad_kernel=conv.kernel.grad, grad_in=f.grad)
                return y.F
        else:
            def step_resident():
                return full(coords_d, feats_d)

        def step_e2e():
            c = host[0].to(dev, non_blocking=True)
            f = host[1].to(dev, non_blocking=True).to(dtype)
            return float(full(c, f).item())
        h2d = sum(int(t.nbytes) for t in host)

    flush_buf = torch.empty(256 << 20, dtype=torch.uint8, device=dev) if flush_l2 else None

    def timed(fn, steps, flush=False):
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()
        l0 = ME._lib.launch_count()
        if flush:
            # per-iteration events, an L2-sized write between iterations outside the events
            total = 0.0
            for _ in range(steps):
                flush_buf.zero_()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                fn()
                e1.record()
                torch.cuda.synchronize()
                total += e0.elapsed_time(e1)
            ms = torch.tensor([total], device=dev)
        else:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(steps):
                fn()
            e1.record()
            torch.cuda.synchronize()
            ms = torch.tensor([e0.elapsed_time(e1)], device=dev)
        if world > 1:
            dist.barrier()
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        return float(ms.item()), ME._lib.launch_count() - l0

    for _ in range(max(args.warmup, 3)):
        step_resident()
    sampler = None
    if rank == 0:
        sampler = NvmlClockSampler(local_rank)
        if not sampler.start():
            sampler = ClockSampler(local_rank)
            sampler.start()
    last.clear()
    ms, launches = timed(step_resident, args.steps, flush=flush_l2)
    dumped = {k: v.detach().clone() for k, v in last.items() if v is not None}
    clocks = None
    if rank == 0:
        try:
            clocks = sampler.stop()
        except Exception as exc:                      # never lose the measurement to the sampler
            clocks = {"sm_mhz": None, "sm_max_mhz": None, "reasons": [f"sampler failed: {exc}"]}
    step_e2e()
    ms_e2e, _ = timed(step_e2e, args.steps)

    total_vox = torch.tensor([float(n_vox)], device=dev)
    if world > 1:
        dist.all_reduce(total_vox)
    total_vox = float(total_vox.item())
    value = total_vox * args.steps / (ms * 1e-3)
    e2e_value = total_vox * args.steps / (ms_e2e * 1e-3)

    # ---- roofline of the dominant kernel, measured live ---------------------------------
    # Two EXTRA steps after the timed region with every convolution / kernel-map launch
    # bracketed by CUDA events on the launch stream (torch's current stream, the one libmeb200
    # launches on).  achieved = ALGORITHMIC flops (2*P*Cin*Cout per launch) or bytes (SURVEY.md
    # 8d formulas) / summed durations.  Every rank runs the extra steps (DDP all-reduce inside).
    prof = ME.backend.profile_conv_kernels(step_resident if is_net else step_e2e, steps=2)
    if flush_l2:
        # cfg1: the convolution kernels from the cached-map step (what `value` times), the
        # kernel-map construction from the e2e step (the only one that builds maps)
        prof_res = ME.backend.profile_conv_kernels(step_resident, steps=2)
        prof["conv_fwd_dgrad"], prof["conv_wgrad"] = prof_res["conv_fwd_dgrad"], prof_res["conv_wgrad"]
    roof = None
    if rank == 0:
        peaks = load_peaks()
        step_ms = (ms if (is_net or flush_l2) else ms_e2e) / args.steps
        peak = peaks["bf16_tflops_sustained"]   # kernels timed inside a long step

        def tf(d):
            return d["flops"] / (d["ms"] * 1e-3) / 1e12 if d["ms"] > 0 else 0.0

        def gb(d):
            return d["bytes"] / (d["ms"] * 1e-3) / 1e9 if d["ms"] > 0 else 0.0

        def entry(key, kernel):
            d = prof[key]
            return {"kernel": kernel, "achieved": tf(d), "frac": tf(d) / peak,
                    "ms_per_step": d["ms"] / d["steps"], "share_of_step": d["ms"] / d["steps"] / step_ms,
                    "launches_per_step": d["launches"] / d["steps"],
                    "flops_per_step": d["flops"] / d["steps"],
                    "hbm": {"achieved_gbs": gb(d), "peak_gbs": peaks["hbm_gbs"],
                            "frac": gb(d) / peaks["hbm_gbs"],
                            "note": "compulsory bytes (SURVEY.md 8d) / same durations"}}
        fam = {"conv_fwd_dgrad": "k_conv_wg (wgmma sparse-conv forward/dgrad)",
               "conv_wgrad": "k_wgrad_wg (wgmma wgrad over compacted pair lists; its time "
                             "includes building the lists when the map is new)"}
        km = prof["kernel_map"]
        km_entry = {"kernel": "k_kernel_map (hash probes -> neighbour tables)", "bound": "hbm",
                    "achieved": gb(km), "peak": peaks["hbm_gbs"], "unit": "GB/s",
                    "frac": gb(km) / peaks["hbm_gbs"], "ms_per_step": km["ms"] / km["steps"],
                    "share_of_step": km["ms"] / km["steps"] / step_ms,
                    "launches_per_step": km["launches"] / km["steps"],
                    "probes_per_s": km["flops"] / (km["ms"] * 1e-3) if km["ms"] > 0 else 0.0,
                    "algorithmic_bytes_per_step": km["bytes"] / km["steps"],
                    "note": "algorithmic bytes = coords + one slot read per probe + both tables "
                            "written (SURVEY.md 8d); `probes` = rows x K look-ups"}
        if not is_net and cfg["D"] == 4:
            # cfg4: the hashing stress — the kernel-map probe kernel is the dominant launch
            roof = dict(km_entry)
            roof["peak_source"] = f"{peaks['source']} (MEASURED_PEAKS.json hbm_gbs)"
            roof["conv"] = [entry(k, v) for k, v in fam.items() if prof[k]["launches"]]
        else:
            live = [k for k in fam if prof[k]["launches"]]
            live.sort(key=lambda k: -prof[k]["ms"])
            if live:
                top = live[0]
                e = entry(top, fam[top])
                roof = {"bound": "tensor", "achieved": e["achieved"], "peak": peak,
                        "unit": "TFLOP/s", "frac": e["frac"],
                        "peak_source": f"{peaks['source']} (MEASURED_PEAKS.json bf16_tflops_sustained)"}
                roof.update({k: v for k, v in e.items() if k not in ("achieved", "frac")})
                roof["other"] = [entry(k, fam[k]) for k in live[1:]]
                if km["launches"]:
                    roof["kernel_map"] = km_entry

    if rank == 0:
        cpu = None if (args.no_cpu_baseline or world > 1) else cpu_baseline(args)
        if is_net:
            workload = (f"{args.model} fwd+bwd+SGD on {args.clouds} synthetic surface cloud(s) x "
                        f"{args.voxels} voxels per rank ({cfg['what']}), coordinate/kernel maps "
                        "rebuilt every step")
            l2 = ("per-step working set (activations + neighbour tables, several hundred MB or "
                  "more) exceeds the 50 MB L2; no explicit flush")
        elif cfg["D"] == 3:
            workload = (f"MinkowskiConvolution {cfg['c_in']}->{cfg['c_out']} k{cfg['ks']} "
                        f"s{cfg['stride']} on surface({args.voxels}) ({cfg['what']}): forward + "
                        "backward (dgrad + wgrad) with the maps cached; e2e rebuilds all maps from "
                        "host buffers")
            l2 = "256 MB written between timed iterations (L2 flush), each iteration event-timed"
        else:
            workload = (f"4-D MinkowskiConvolution {cfg['c_in']}->{cfg['c_out']} k{cfg['ks']} (K=81) "
                        f"on {args.voxels} coordinate draws ({cfg['what']}): dedup insert + "
                        "kernel map + forward + backward every step")
            l2 = ("neighbour tables (2 x 81 x n x 4 B = 85 MB) + features + hash table per step; "
                  "no explicit flush")
        line = {
            "metric": cfg["metric"], "value": value, "unit": UNIT, "n_gpus": world,
            "steps": args.steps, "warmup": max(args.warmup, 3), "ms_per_step": ms / args.steps,
            "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
            "dtype": args.dtype, "data": "synthetic",
            "config": {"workload": workload,
                       "global_batch_clouds": args.clouds * world, "voxels_per_step": total_vox,
                       "parallelism": f"dp{world}" if is_net else f"replicas{world}", "l2": l2,
                       "host_cpus_bound": numa_cpus,
                       **({"ablate": ablate} if ablate else {})},
            "e2e": {"value": e2e_value, "unit": UNIT, "ms_per_step": ms_e2e / args.steps,
                    "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": 4},
            "gpu_launches": int(launches),
            "clocks": clocks,
            "roofline": roof,
        }
        if loss_check is not None:
            line["loss_check"] = loss_check
        if cpu is not None:
            line["cpu_baseline"] = cpu
        if args.dump_outputs:
            dump_outputs(args.dump_outputs, dumped)
        print(json.dumps(line), flush=True)
    if world > 1:
        dist.destroy_process_group()


def main():
    args = parse_args()
    if args.impl == "reference":
        # the reference's OpenMP loops and MKL read this at first use; torchrun exports
        # OMP_NUM_THREADS=1 to its workers, which would handicap the CPU arm at N>1
        os.environ["OMP_NUM_THREADS"] = str(_ref_threads()[1])
        run_reference(args)
    else:
        run_ours(args)


if __name__ == "__main__":
    main()
