"""Generates channel-wise convolution results and one ConvNeXt-style training step of the COMPILED
REFERENCE (oracle/_ref, built by oracle/build_ref.py) on seeded inputs.  Run where the reference is
available:

    python tests/golden/make_chwise_fixtures.py

Writes tests/golden/ref_chwise_<case>.npz for every case of test_gpu_chwise.CASES (a multi-cloud
input with negative coordinates, kernel, bias, output, output gradient, input gradient and kernel
gradient, fp32 on the CPU) and ref_chwise_convnext.npz (examples/convnext.py in fp32 train mode on
the inputs of tests/test_gpu_chwise.py: initial-weight digest, logits, loss and sampled gradients,
as ref_resnet.npz stores them).

The reference's output row order comes from its hash table, so every output is stored with its rows
sorted by coordinate, and output gradients are drawn in that canonical order.  Its pair order inside
an offset comes from OpenMP, so the kernel gradient can differ in the last bits between runs."""
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


def canon(coords):
    """perm with coords[perm] sorted lexicographically by row."""
    c = np.asarray(coords)
    return np.lexsort(c.T[::-1])


def layer_case(ME, name, spec, seed):
    import test_gpu_chwise as T
    coords = T.case_coords(spec, seed)
    C = spec["C"]
    torch.manual_seed(seed)
    feats = torch.randn(len(coords), C, generator=torch.Generator().manual_seed(seed + 1))
    x = ME.SparseTensor(feats, coords, requires_grad=True)
    layer = T.make_layer(ME, spec)
    if spec.get("region") == "HYPER_CROSS":
        # the reference's KernelGenerator.get_kernel raises TypeError for HYPER_CROSS
        # (convert_region_type computes `kernel_size % 2` on a list); fill its cache with what the
        # function returns for that region type, so the layer runs its own kernel map
        kg = layer.kernel_generator
        kg.cache[tuple(x.tensor_stride)] = (kg.region_type, None, kg.kernel_volume)
    y = layer(x)
    perm = canon(y.C.numpy())
    g_canon = torch.rand(y.F.shape, generator=torch.Generator().manual_seed(seed + 2)) - 0.5
    g_ref = torch.empty_like(g_canon)
    g_ref[perm] = g_canon
    y.F.backward(g_ref)
    bias = layer.bias.detach().numpy() if layer.bias is not None else np.zeros((0,), np.float32)
    np.savez_compressed(
        os.path.join(HERE, f"ref_chwise_{name}.npz"), in_coords=x.C.numpy(),
        in_feats=x.F.detach().numpy(), kernel=layer.kernel.detach().numpy(), bias=bias,
        out_coords=y.C.numpy()[perm], out_feats=y.F.detach().numpy()[perm],
        grad_out=g_canon.numpy(), grad_in=x.F.grad.numpy(), grad_kernel=layer.kernel.grad.numpy())
    print("wrote chwise", name, len(coords), "->", len(y.C), "K =", layer.kernel.shape[0],
          flush=True)


def convnext_case(REF):
    from examples.convnext import convnext
    import test_gpu_chwise as T
    out = {}
    torch.manual_seed(T.CONVNEXT_SEED)
    net = convnext(REF, 3, T.CONVNEXT_CLASSES, 3)
    out["init_digest"] = state_digest(net)
    y, loss = T._convnext_step(REF, net, "cpu")
    perm = np.argsort(y.C.numpy()[:, 0], kind="stable")
    out["out_coords"] = y.C.numpy()[perm]
    out["logits"] = y.F.detach().numpy().astype(np.float32)[perm]
    out["loss"] = np.float64(loss)
    params = dict(net.named_parameters())
    for p in T.CONVNEXT_PARAMS:
        gr = params[p].grad.numpy().ravel()
        idx = np.arange(gr.size) if gr.size <= SAMPLE_ELEMS else np.sort(
            np.random.default_rng(2).choice(gr.size, SAMPLE_ELEMS, replace=False))
        out[f"{p}/idx"] = idx.astype(np.int64)
        out[f"{p}/grad"] = gr[idx].astype(np.float32)
        out[f"{p}/absmax"] = np.float64(np.abs(gr).max())
    print("convnext loss", loss, flush=True)
    np.savez_compressed(os.path.join(HERE, "ref_chwise_convnext.npz"), **out)


def main():
    from oracle import ref
    import test_gpu_chwise as T
    ME = ref.import_reference()
    torch.set_num_threads(os.cpu_count() or 1)
    which = sys.argv[1:] or list(T.CASES) + ["convnext"]
    for i, (name, spec) in enumerate(T.CASES.items()):
        if name in which:
            layer_case(ME, name, spec, 70 + 10 * i)
    if "convnext" in which:
        convnext_case(ME)


if __name__ == "__main__":
    main()
