"""Times ME.spmm, spmm_average and direct max pooling, forward and backward, moving features from
8 clouds x 250k points to their voxels (the quantisation profiles/field_bench.py uses) at C = 32
and 64 in fp32 and bf16, with CUDA events after a warm-up of every timed shape, next to
torch.sparse.mm and index_add_ / scatter_reduce("amax") on the same inputs.

    python profiles/spmm_bench.py [--reps 20]

Prints the card's name and power limit, then one JSON line per case: milliseconds per call (index
check, grouping and reduction together), the same for the reduction kernel alone on a grouping
built beforehand, the bytes that kernel must move (computed here from the shapes) and its share
of the 3.35 TB/s HBM3 bound of an H100 SXM.

Direct max pooling has two backwards.  `max_bwd` is MinkowskiDirectMaxPoolingFunction's: every
pair takes the output gradient where it won (`field_expand` MAX over the pairs) and each input row
sums its pairs (`group_by_row` over in_map + a SUM `field_reduce`), P keys sorted.  `max_bwd_mask`
is the reference's entry point `direct_max_pool_bw`, which sees only the flat mask: it groups the
n_out * C output elements by their flat index (`max_bwd_mask_group`) and sums each group
(`max_bwd_mask_reduce`).  The two give the same bits here (every point has one pair)."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import minkowskiengine_b200 as ME  # noqa: E402
from minkowskiengine_b200 import _lib, backend as B  # noqa: E402

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


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    return {"gpu": torch.cuda.get_device_name(), "nvidia_smi": q.splitlines()[0] if q else None}


def cloud(clouds=8, per=250_000):
    g = torch.Generator().manual_seed(0)
    n = clouds * per
    pts = torch.cat([torch.arange(clouds).repeat_interleave(per)[:, None].float(),
                     torch.rand(n, 3, generator=g) * 100], 1).cuda()
    tf = ME.TensorField(torch.zeros(n, 1, device="cuda"), pts)
    st = tf.sparse()
    inv = tf._record(st.coordinate_map_key).inverse
    return n, len(st), inv


def case(n, M, inv, C, dtype, reps):
    es = torch.tensor([], dtype=dtype).element_size()
    g = torch.Generator().manual_seed(1)
    x = torch.randn(n, C, generator=g).to(dtype).cuda()
    w = torch.rand(n, generator=g).to(dtype).cuda()
    gv = torch.randn(M, C, generator=g).to(dtype).cuda()
    vox = inv.int()
    pts = torch.arange(n, dtype=torch.int32, device="cuda")
    size, tsize = torch.Size([M, n]), torch.Size([n, M])
    grp_vox, grp_pts = B.group_by_row(vox, M), B.group_by_row(pts, n)
    w32 = w.float()
    red_fwd = n * C * es + M * C * es + 12 * n + 4 * (M + 1)   # rows gathered, rows written, perm /
    red_bwd = M * C * es + n * C * es + 12 * n + 4 * (n + 1)   # src_row / weight, starts
    _, coo, avals = ME.spmm_average(vox, pts, size, x)
    _, mask, winner, o_rows, i_rows = B._direct_max_pool(pts, vox, x, M, True)
    res = {}
    res["spmm_fwd"] = (timed(lambda: ME.spmm(vox, pts, w, size, x), reps),
                       timed(lambda: B.field_reduce(x, grp_vox, M, _lib.FIELD_SUM, weight=w32,
                                                    src_row=pts), reps), red_fwd)
    res["spmm_bwd"] = (timed(lambda: ME.spmm(pts, vox, w, tsize, gv), reps),
                       timed(lambda: B.field_reduce(gv, grp_pts, n, _lib.FIELD_SUM, weight=w32,
                                                    src_row=vox), reps), red_bwd)
    res["avg_fwd"] = (timed(lambda: ME.spmm_average(vox, pts, size, x), reps),
                      timed(lambda: B.field_reduce(x, grp_vox, M, _lib.FIELD_AVG, src_row=pts),
                            reps), red_fwd - 4 * n)
    res["avg_bwd"] = (timed(lambda: ME.spmm(coo[1], coo[0], avals, tsize, gv), reps), None, None)
    res["max_fwd"] = (timed(lambda: B.direct_max_pool_fw(pts, vox, x, M), reps),
                      timed(lambda: B.field_reduce(x, grp_vox, M, _lib.FIELD_MAX, src_row=pts),
                            reps), red_fwd - 4 * n + 4 * M * C)
    # the autograd backward over the winning pairs
    res["max_bwd"] = (timed(lambda: B.direct_max_pool_pairs_bw(gv, winner, o_rows, i_rows, n),
                            reps), None, None)
    # the reference's entry point: group the n_out * C elements by flat argmax, one SUM over them
    assert torch.equal(B.direct_max_pool_pairs_bw(gv, winner, o_rows, i_rows, n),
                       B.direct_max_pool_bw(gv, mask, n))
    res["max_bwd_mask"] = (timed(lambda: B.direct_max_pool_bw(gv, mask, n), reps), None, None)
    flat = mask.view(-1)
    grp_flat = B.group_by_row(flat, n * C)
    res["max_bwd_mask_group"] = (timed(lambda: B.group_by_row(flat, n * C), reps), None, None)
    res["max_bwd_mask_reduce"] = (timed(lambda: B.field_reduce(gv.view(-1, 1), grp_flat, n * C,
                                                               _lib.FIELD_SUM), reps), None,
                                  M * C * es + n * C * es + 8 * M * C + 4 * (n * C + 1))
    # torch on the same inputs
    sp = torch.sparse_coo_tensor(torch.stack((inv, pts.long())), w.float(), size).coalesce()
    xf = x.float()
    res["torch_sparse_mm_fwd_fp32"] = (timed(lambda: torch.sparse.mm(sp, xf), reps), None, None)
    res["torch_index_add_fwd"] = (timed(lambda: torch.zeros(M, C, dtype=dtype, device="cuda")
                                        .index_add_(0, inv, x * w[:, None]), reps), None, None)
    res["torch_index_select_bwd"] = (timed(lambda: gv.index_select(0, inv) * w[:, None], reps),
                                     None, None)
    idx = inv[:, None].expand(n, C)
    res["torch_amax_fwd"] = (timed(lambda: torch.zeros(M, C, dtype=dtype, device="cuda")
                                   .scatter_reduce_(0, idx, x, "amax", include_self=False), reps),
                             None, None)
    for k, (ms, kms, nbytes) in res.items():
        out = {"case": k, "C": C, "dtype": str(dtype).replace("torch.", ""), "points": n,
               "voxels": M, "ms": round(ms, 4)}
        if kms is not None:
            out["reduce_ms"] = round(kms, 4)
        if nbytes is not None:
            t = kms if kms is not None else ms
            out.update(bytes=nbytes, hbm_share=round(nbytes / HBM / (t * 1e-3), 3))
        print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "spmm_bench.py measures on the GPU only"
    print(json.dumps(card()), flush=True)
    n, M, inv = cloud()
    for C in (32, 64):
        for dtype in (torch.float32, torch.bfloat16):
            case(n, M, inv, C, dtype, a.reps)


if __name__ == "__main__":
    main()
