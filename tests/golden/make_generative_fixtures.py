"""Generates pruning / union / non-matching arithmetic results and one completion-network run of the
COMPILED REFERENCE (oracle/_ref, built by oracle/build_ref.py) on seeded inputs.  Run where the
reference is available:

    python tests/golden/make_generative_fixtures.py

Writes tests/golden/ref_prune.npz (a multi-cloud input, a random mask, output and gradient),
ref_union.npz (three inputs with partial overlaps), ref_binary_{add,sub,mul,div}.npz (two maps with
partial overlap, output and both gradients) and ref_completion.npz (examples/completion.py with 3
levels in fp32 train mode on the inputs of tests/test_gpu_generative.py: initial-weight digest,
per-level logits, targets and kept coordinates, loss and sampled gradients, as ref_resnet.npz
stores them).

The reference's pruned and union row orders come from its hash table, so every output is stored
with its rows sorted by coordinate, and output gradients are drawn in that canonical order."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

from helpers import state_digest  # noqa: E402  (tests/ is on the path)

SAMPLE_ELEMS = 2048
COMPLETION_PARAMS = ("enc_block_s1.0.kernel", "enc_blocks.1.0.kernel", "dec_blocks.0.0.kernel",
                     "dec_blocks.2.3.kernel", "dec_cls.2.kernel", "dec_cls.2.bias")


def canon(coords):
    """perm with coords[perm] sorted lexicographically by row."""
    c = np.asarray(coords)
    return np.lexsort(c.T[::-1])


def cloud(n, extent, seed, batches):
    g = torch.Generator().manual_seed(seed)
    c = torch.randint(-extent, extent, (n, 3), generator=g, dtype=torch.int32)
    b = torch.randint(0, batches, (n, 1), generator=g, dtype=torch.int32)
    return torch.unique(torch.cat([b, c], 1), dim=0)


def overlapping(n, seed, parts):
    """`parts` unique clouds drawn from one pool: any two share about half their rows."""
    pool = cloud(int(n * 1.6), 9, seed, 2)
    g = torch.Generator().manual_seed(seed + 1)
    out = []
    for _ in range(parts):
        sel = torch.randperm(len(pool), generator=g)[:n]
        out.append(pool[sel])
    return out


def canon_grad(shape, perm, seed):
    """A random gradient drawn in canonical row order, returned in the reference's row order."""
    g_canon = torch.rand(shape, generator=torch.Generator().manual_seed(seed))
    g_ref = torch.empty_like(g_canon)
    g_ref[perm] = g_canon
    return g_canon, g_ref


def prune_case(ME):
    C = 7
    coords = cloud(1500, 10, 30, 3)
    x = ME.SparseTensor(torch.randn(len(coords), C, generator=torch.Generator().manual_seed(31)),
                        coords, requires_grad=True)
    keep = torch.rand(len(coords), generator=torch.Generator().manual_seed(32)) < 0.5
    y = ME.MinkowskiPruning()(x, keep)
    perm = canon(y.C.numpy())
    g_canon, g_ref = canon_grad(y.F.shape, perm, 33)
    y.F.backward(g_ref)
    np.savez_compressed(os.path.join(HERE, "ref_prune.npz"), in_coords=x.C.numpy(),
                        in_feats=x.F.detach().numpy(), keep=keep.numpy(),
                        out_coords=y.C.numpy()[perm], out_feats=y.F.detach().numpy()[perm],
                        grad_out=g_canon.numpy(), grad_in=x.F.grad.numpy())
    print("wrote prune", len(coords), "->", len(y.C))


def _inputs(ME, coords_list, C, seed, scale=None):
    xs = []
    mgr = None
    for i, c in enumerate(coords_list):
        f = torch.randn(len(c), C, generator=torch.Generator().manual_seed(seed + i))
        if scale is not None:
            f = scale(f)
        x = ME.SparseTensor(f, c, coordinate_manager=mgr, requires_grad=True)
        mgr = x.coordinate_manager
        xs.append(x)
    return xs


def union_case(ME):
    coords = overlapping(900, 40, 3)
    xs = _inputs(ME, coords, 6, 41)
    assert len({x.coordinate_map_key for x in xs}) == 3
    y = ME.MinkowskiUnion()(*xs)
    perm = canon(y.C.numpy())
    g_canon, g_ref = canon_grad(y.F.shape, perm, 44)
    y.F.backward(g_ref)
    out = {"out_coords": y.C.numpy()[perm], "out_feats": y.F.detach().numpy()[perm],
           "grad_out": g_canon.numpy()}
    for i, x in enumerate(xs):
        out[f"in_coords_{i}"] = x.C.numpy()
        out[f"in_feats_{i}"] = x.F.detach().numpy()
        out[f"grad_in_{i}"] = x.F.grad.numpy()
    np.savez_compressed(os.path.join(HERE, "ref_union.npz"), **out)
    print("wrote union", [len(c) for c in coords], "->", len(y.C))


def binary_case(ME, name, seed):
    coords = overlapping(1000, seed, 2)
    # div: b away from 0 (|b| in [0.5, 2.5])
    scale = (lambda f: torch.sign(f) * (0.5 + f.abs().clamp(max=2.0))) if name == "div" else None
    a, b = _inputs(ME, coords, 5, seed + 2, scale)
    op = {"add": lambda p, q: p + q, "sub": lambda p, q: p - q, "mul": lambda p, q: p * q,
          "div": lambda p, q: p / q}[name]
    y = op(a, b)
    perm = canon(y.C.numpy())
    g_canon, g_ref = canon_grad(y.F.shape, perm, seed + 5)
    y.F.backward(g_ref)
    np.savez_compressed(os.path.join(HERE, f"ref_binary_{name}.npz"), in_coords_0=a.C.numpy(),
                        in_feats_0=a.F.detach().numpy(), in_coords_1=b.C.numpy(),
                        in_feats_1=b.F.detach().numpy(), out_coords=y.C.numpy()[perm],
                        out_feats=y.F.detach().numpy()[perm], grad_out=g_canon.numpy(),
                        grad_in_0=a.F.grad.numpy(), grad_in_1=b.F.grad.numpy())
    print("wrote binary", name, "->", len(y.C))


def completion_case(REF):
    from examples.completion import completion_net
    import test_gpu_generative as T
    out = {}
    torch.manual_seed(T.COMPLETION_SEED)
    net = completion_net(REF, T.COMPLETION_CHANNELS, T.COMPLETION_CHANNELS)
    out["init_digest"] = state_digest(net)
    out_cls, targets, final, loss = T._completion_step(REF, net, "cpu")
    for j, o in enumerate(out_cls):
        f = o.F.detach()[:, 0]
        lo = float(f.abs().min())
        print(f"completion level {j}: {len(f)} logits, min |logit| {lo:.3g}, max |logit| "
              f"{float(f.abs().max()):.3g}, {int((f > 0).sum())} positive", flush=True)
        # fp32 reordering must not be able to flip a pruning decision
        assert lo >= 1e-3, f"level {j}: a logit within 1e-3 of the pruning threshold"
        # ... and the level must still prune, and keep voxels by prediction
        assert 0 < int((f > 0).sum()) < len(f), f"level {j}: logits of one sign only"
    print("completion loss", loss, flush=True)
    for j, (o, t) in enumerate(zip(out_cls, targets)):
        perm = canon(o.C.numpy())
        out[f"level{j}/coords"] = o.C.numpy()[perm]
        out[f"level{j}/logits"] = o.F.detach().numpy()[perm, 0]
        out[f"level{j}/target"] = t.numpy()[perm]
        keep = o.F.detach().numpy()[:, 0] > 0
        if j < len(out_cls) - 1:
            keep |= t.numpy()
        kc = o.C.numpy()[keep]
        out[f"level{j}/kept_coords"] = kc[canon(kc)]
    out["final_coords"] = final.C.numpy()[canon(final.C.numpy())]
    out["loss"] = np.float64(loss)
    params = dict(net.named_parameters())
    for p in COMPLETION_PARAMS:
        gr = params[p].grad.numpy().ravel()
        idx = np.arange(gr.size) if gr.size <= SAMPLE_ELEMS else np.sort(
            np.random.default_rng(2).choice(gr.size, SAMPLE_ELEMS, replace=False))
        out[f"{p}/idx"] = idx.astype(np.int64)
        out[f"{p}/grad"] = gr[idx].astype(np.float32)
        out[f"{p}/absmax"] = np.float64(np.abs(gr).max())
    np.savez_compressed(os.path.join(HERE, "ref_completion.npz"), **out)
    print("wrote completion", [len(o.C) for o in out_cls], flush=True)


def main():
    from oracle import ref
    ME = ref.import_reference()
    torch.set_num_threads(os.cpu_count() or 1)
    which = sys.argv[1:] or ["prune", "union", "binary", "completion"]
    if "prune" in which:
        prune_case(ME)
    if "union" in which:
        union_case(ME)
    if "binary" in which:
        for i, name in enumerate(("add", "sub", "mul", "div")):
            binary_case(ME, name, 50 + 10 * i)
    if "completion" in which:
        completion_case(ME)


if __name__ == "__main__":
    main()
