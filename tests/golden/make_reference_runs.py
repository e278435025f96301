"""Regenerates tests/golden/ref_network.npz, ref_quantize.npz and ref_live_conv.npz: results of
the compiled reference (oracle/_ref, CPU, fp32) on the seeded inputs of test_gpu_network.py,
test_gpu_quantize.py and test_oracle.py, so that those tests compare against the reference
without needing it at run time.

    python tests/golden/make_reference_runs.py          (needs oracle/_ref, see oracle/build_ref.py)

Large outputs are stored as a SHA-256 digest (bit-exact comparisons) or as a fixed, seeded
sample of rows / elements together with the full tensor's max and rms (tolerance comparisons).
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

from helpers import digest, state_digest  # noqa: E402  (tests/ is on the path)

SAMPLE_ROWS = 1024      # logits rows kept per network case
SAMPLE_ELEMS = 2048     # gradient elements kept per parameter (all of them when fewer)

NET_CASES = [("fp32", "MinkUNet14", 6000), ("fp32", "MinkUNet34C", 4000),
             ("bf16", "MinkUNet14", 50_000), ("bf16", "MinkUNet34C", 30_000)]
NET_PARAMS = {"fp32": ("conv0p1s1.kernel", "block4.0.conv1.kernel", "final.kernel"),
              "bf16": ("conv0p1s1.kernel", "block1.0.conv2.kernel", "block4.0.conv1.kernel",
                       "convtr7p2s2.kernel", "block8.0.conv1.kernel", "final.kernel")}
QUANT_CASES = [(20000, 0.5), (50000, 1), (3000, 2.5), (1, 1), (100000, 0.25)]


def sample_index(n, k, seed):
    if n <= k:
        return np.arange(n)
    return np.sort(np.random.default_rng(seed).choice(n, k, replace=False))


def _network(REF):
    from examples.minkunet import minkunet
    import test_gpu_network as T
    from oracle import oracle_np as O
    out = {}
    for mode, name, n in NET_CASES:
        key = f"{mode}_{name}_{n}"
        torch.manual_seed(0)
        net = minkunet(name, REF, 3, 20, 3)
        if mode == "bf16":
            T._bf16_round_(net)
        # the initial weights both packages build from seed 0 (the tests check theirs against it)
        out[key + "/init_digest"] = state_digest(net)
        if mode == "fp32":
            coords = O.surface_cloud(n, seed=3)
            feats = torch.rand(n, 3, generator=torch.Generator().manual_seed(1))
            y, loss = T._run(REF, net, coords, feats, "cpu")
        else:
            coords = O.surface_cloud(n, seed=5)
            g = torch.Generator().manual_seed(2)
            feats = torch.rand(n, 3, generator=g).bfloat16()
            labels = torch.randint(0, 20, (n,), generator=g)
            y, loss = T._ce_step(REF, net, coords, feats.float(), labels, "cpu")
        F = y.F.detach().numpy().astype(np.float32)
        rows = sample_index(len(F), SAMPLE_ROWS, 1)
        out[key + "/coords_digest"] = digest(y.C)
        out[key + "/rows"] = rows.astype(np.int64)
        out[key + "/logits"] = F[rows]
        out[key + "/logits_absmax"] = np.float64(np.abs(F).max())
        out[key + "/logits_rms"] = np.float64(np.sqrt((F.astype(np.float64) ** 2).mean()))
        out[key + "/loss"] = np.float64(loss)
        params = dict(net.named_parameters())
        for p in NET_PARAMS[mode]:
            gr = params[p].grad.numpy().ravel()
            idx = sample_index(gr.size, SAMPLE_ELEMS, 2)
            out[f"{key}/{p}/idx"] = idx.astype(np.int64)
            out[f"{key}/{p}/grad"] = gr[idx].astype(np.float32)
            out[f"{key}/{p}/absmax"] = np.float64(np.abs(gr).max())
        print("network", key, "loss", loss, flush=True)
    return out


def _quantize(REF):
    import test_gpu_quantize as T
    out = {}
    for n, qs in QUANT_CASES:
        pts = T._points(n, seed=n)
        pts[:, 0] *= qs if qs != 1 else 1
        feats = torch.rand(n, 4, generator=torch.Generator().manual_seed(1))
        rc, rf, ri, rinv = REF.utils.sparse_quantize(pts, feats, return_index=True,
                                                     return_inverse=True, quantization_size=qs)
        key = f"q_{n}_{qs}"
        for nm, t in (("coords", rc), ("feats", rf), ("index", ri), ("inverse", rinv)):
            out[f"{key}/{nm}"] = digest(t)
        out[f"{key}/inverse_len"] = np.int64(len(rinv))
    n = 30000
    pts = T._points(n, seed=7, extent=24.0)
    g = torch.Generator().manual_seed(3)
    labels = torch.randint(0, 5, (n,), generator=g, dtype=torch.int32)
    labels[torch.rand(n, generator=g) < 0.02] = -100
    feats = torch.rand(n, 2, generator=g)
    rc, rf, rl, ri, rinv = REF.utils.sparse_quantize(pts, feats, labels, ignore_label=-100,
                                                     return_index=True, return_inverse=True)
    out["labels/coords"] = digest(rc)
    out["labels/feats"] = digest(rf)
    out["labels/labels"] = digest(torch.as_tensor(np.asarray(rl)))
    out["labels/index"] = np.asarray(ri).astype(np.int32)
    out["labels/inverse"] = np.asarray(rinv).astype(np.int32)
    return out


def _live_conv(REF):
    torch.manual_seed(3)
    coords = torch.cat([torch.zeros(700, 1, dtype=torch.int32),
                        torch.randint(-9, 9, (700, 3), dtype=torch.int32)], 1)
    x = REF.SparseTensor(torch.rand(700, 4), coords)
    conv = REF.MinkowskiConvolution(4, 6, kernel_size=3, stride=2, dimension=3)
    y = conv(x)
    return {"in_coords": x.C.numpy(), "in_feats": x.F.numpy(), "kernel": conv.kernel.detach().numpy(),
            "out_coords": y.C.numpy(), "out_feats": y.F.detach().numpy()}


def main():
    from oracle import ref
    REF = ref.import_reference()
    torch.set_num_threads(os.cpu_count() or 1)
    np.savez_compressed(os.path.join(HERE, "ref_live_conv.npz"), **_live_conv(REF))
    np.savez_compressed(os.path.join(HERE, "ref_quantize.npz"), **_quantize(REF))
    np.savez_compressed(os.path.join(HERE, "ref_network.npz"), **_network(REF))


if __name__ == "__main__":
    main()
