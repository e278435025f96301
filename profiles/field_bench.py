"""Times TensorField.sparse() (UNWEIGHTED_AVERAGE) and SparseTensor.slice, forward and backward, on
8 clouds x 250k points at C = 32 bf16 and C = 3 fp32, with CUDA events after a warm-up of every
timed shape, next to the torch composition (index_add_ / index_select) on the same inputs.

    python profiles/field_bench.py [--reps 20]

Prints one JSON line per case: milliseconds per call, the bytes each kernel must move (computed
here from the shapes) and their share of the 3.35 TB/s HBM3 bound of an H100 SXM."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import minkowskiengine_b200 as ME  # noqa: E402

HBM = 3.35e12


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def case(C, dtype, reps, clouds=8, per=250_000):
    g = torch.Generator().manual_seed(0)
    n = clouds * per
    pts = torch.cat([torch.arange(clouds).repeat_interleave(per)[:, None].float(),
                     torch.rand(n, 3, generator=g) * 100], 1).cuda()
    x = torch.randn(n, C, generator=g).cuda().to(dtype)
    tf = ME.TensorField(x, pts)
    st = tf.sparse()
    rec = tf._record(st.coordinate_map_key)
    rec.group()
    M, inv = len(st), rec.inverse
    es = x.element_size()
    gv = torch.randn(M, C, device="cuda").to(dtype)
    gp = torch.randn(n, C, device="cuda").to(dtype)
    Fn = ME.tensor_field.MinkowskiFieldQuantizationFunction.forward
    ctx = type("ctx", (), {})()
    res = {}
    res["sparse_fwd"] = (timed(lambda: Fn(ctx, x, rec, ME._lib.FIELD_AVG), reps),
                         n * C * es + M * C * es + 4 * n + 4 * (M + 1))
    res["sparse_bwd"] = (timed(lambda: ME.backend.field_expand(gv, inv, ME._lib.FIELD_AVG,
                                                               start=rec.group()[0]), reps),
                         M * C * es + n * C * es + 8 * n + 4 * (M + 1))
    res["slice_fwd"] = (timed(lambda: ME.backend.gather_rows(st.F, inv, n), reps),
                        M * C * es + n * C * es + 8 * n)
    res["slice_bwd"] = (timed(lambda: ME.backend.field_reduce(gp, rec.group(), M,
                                                              ME._lib.FIELD_SUM), reps),
                        n * C * es + M * C * es + 4 * n + 4 * (M + 1))

    def torch_avg():
        acc = torch.zeros(M, C, dtype=dtype, device="cuda").index_add_(0, inv, x)
        cnt = torch.zeros(M, dtype=dtype, device="cuda").index_add_(0, inv, torch.ones_like(x[:, 0]))
        return acc / cnt[:, None]
    res["torch_sparse_fwd"] = (timed(torch_avg, reps), None)
    res["torch_slice_fwd"] = (timed(lambda: st.F.index_select(0, inv), reps), None)
    res["torch_slice_bwd"] = (timed(lambda: torch.zeros(M, C, dtype=dtype, device="cuda")
                                    .index_add_(0, inv, gp), reps), None)
    for k, (ms, nbytes) in res.items():
        out = {"case": k, "C": C, "dtype": str(dtype).replace("torch.", ""), "points": n,
               "voxels": M, "ms": round(ms, 4)}
        if nbytes is not None:
            out.update(bytes=nbytes, hbm_share=round(nbytes / HBM / (ms * 1e-3), 3))
        print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "field_bench.py measures on the GPU only"
    print(json.dumps({"gpu": torch.cuda.get_device_name()}))
    case(32, torch.bfloat16, a.reps)
    case(3, torch.float32, a.reps)


if __name__ == "__main__":
    main()
