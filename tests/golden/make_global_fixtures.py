"""Generates the global pooling / broadcast / instance-norm results of the COMPILED REFERENCE
(oracle/_ref, built by oracle/build_ref.py) on seeded inputs.  Run where the reference is available:

    python tests/golden/make_global_fixtures.py

Writes tests/golden/ref_global_{sum,avg,max}.npz, ref_broadcast_{add,mul}.npz, ref_instnorm.npz
(small multi-cloud cases with batch indices 0..B-1, the _KERNEL pooling modes, inputs, outputs and
both gradients; they pin tests/global_oracle.py on the CPU and the CUDA path in
tests/test_gpu_global.py) and ref_resnet.npz (ResNet14 fp32 in train mode with dropout 0, and one
squeeze-excitation block, on the inputs of tests/test_gpu_global.py: initial-weight digest, logits,
loss and sampled gradients, as tests/golden/ref_network.npz stores them).

The reference's origin-map row order is implementation-defined, so per-cloud rows are stored in
ascending batch order, the order this package defines."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

from helpers import state_digest  # noqa: E402  (tests/ is on the path)

SAMPLE_ELEMS = 2048     # gradient elements kept per ResNet parameter (all of them when fewer)
RESNET_PARAMS = ("conv1.0.kernel", "layer2.0.conv1.kernel", "conv5.1.kernel", "final.linear.weight")
SE_PARAMS = ("conv1.kernel", "se.fc.0.linear.weight", "se.fc.2.linear.weight")


def cloud(n, extent, seed, D=3, batches=1):
    g = torch.Generator().manual_seed(seed)
    c = torch.randint(-extent, extent, (n, D), generator=g, dtype=torch.int32)
    b = torch.randint(0, batches, (n, 1), generator=g, dtype=torch.int32)
    return torch.cat([b, c], 1)


def sample_index(n, k, seed):
    if n <= k:
        return np.arange(n)
    return np.sort(np.random.default_rng(seed).choice(n, k, replace=False))


def _origin_perm(x):
    """perm with (reference origin rows)[perm] in ascending batch order."""
    mgr = x.coordinate_manager
    oc = mgr.get_coordinates(mgr.origin()).numpy()
    return np.argsort(oc[:, 0], kind="stable")


def global_case(ME, mode, seed):
    """Global pooling with the _KERNEL modes over 3 clouds (batch indices 0..2)."""
    D, C, n = 3, 6, 1500
    torch.manual_seed(seed)
    x = ME.SparseTensor(torch.randn(n, C), cloud(n, 10, seed, D, 3), requires_grad=True)
    pm = {"sum": ME.PoolingMode.GLOBAL_SUM_POOLING_KERNEL,
          "avg": ME.PoolingMode.GLOBAL_AVG_POOLING_KERNEL,
          "max": ME.PoolingMode.GLOBAL_MAX_POOLING_KERNEL}[mode]
    y = ME.MinkowskiGlobalPooling(pm)(x)
    perm = _origin_perm(x)
    gout = torch.rand(y.F.shape)
    y.F.backward(gout)
    np.savez_compressed(os.path.join(HERE, f"ref_global_{mode}.npz"), in_coords=x.C.numpy(),
                        in_feats=x.F.detach().numpy(), out_coords=y.C.numpy()[perm],
                        out_feats=y.F.detach().numpy()[perm], grad_out=gout.numpy()[perm],
                        grad_in=x.F.grad.numpy())
    print("wrote global", mode)


def broadcast_case(ME, mode, seed):
    D, C, n = 3, 5, 1200
    torch.manual_seed(seed)
    x = ME.SparseTensor(torch.randn(n, C), cloud(n, 10, seed, D, 4), requires_grad=True)
    key = ME.MinkowskiGlobalPooling(ME.PoolingMode.GLOBAL_AVG_POOLING_KERNEL)(x).coordinate_map_key
    perm = _origin_perm(x)
    g_canon = torch.randn(len(perm), C)
    g_ref = torch.empty_like(g_canon)
    g_ref[perm] = g_canon                      # reference row perm[k] = canonical row k
    g_ref.requires_grad_(True)
    glob = ME.SparseTensor(g_ref, coordinate_map_key=key, coordinate_manager=x.coordinate_manager)
    layer = {"add": ME.MinkowskiBroadcastAddition,
             "mul": ME.MinkowskiBroadcastMultiplication}[mode]()
    y = layer(x, glob)
    gout = torch.rand(y.F.shape)
    y.F.backward(gout)
    np.savez_compressed(os.path.join(HERE, f"ref_broadcast_{mode}.npz"), in_coords=x.C.numpy(),
                        in_feats=x.F.detach().numpy(), glob_feats=g_canon.numpy(),
                        out_feats=y.F.detach().numpy(), grad_out=gout.numpy(),
                        grad_in=x.F.grad.numpy(), grad_glob=g_ref.grad.numpy()[perm])
    print("wrote broadcast", mode)


def instnorm_case(ME, seed):
    D, C, n = 3, 8, 1600
    torch.manual_seed(seed)
    x = ME.SparseTensor(torch.randn(n, C) * 2 + 1, cloud(n, 10, seed, D, 3), requires_grad=True)
    layer = ME.MinkowskiInstanceNorm(C)
    with torch.no_grad():
        layer.weight.copy_(torch.rand(1, C) + 0.5)
        layer.bias.copy_(torch.randn(1, C))
    y = layer(x)
    gout = torch.rand(y.F.shape)
    y.F.backward(gout)
    np.savez_compressed(os.path.join(HERE, "ref_instnorm.npz"), in_coords=x.C.numpy(),
                        in_feats=x.F.detach().numpy(), weight=layer.weight.detach().numpy(),
                        bias=layer.bias.detach().numpy(), out_feats=y.F.detach().numpy(),
                        grad_out=gout.numpy(), grad_in=x.F.grad.numpy(),
                        grad_weight=layer.weight.grad.numpy(), grad_bias=layer.bias.grad.numpy())
    print("wrote instnorm")


def resnet_case(REF):
    """ResNet14 (fp32, train mode, dropout 0) and one SE block on the inputs of
    test_gpu_global.py."""
    from examples.resnet import resnet, se_basic_block
    import test_gpu_global as T
    out = {}
    torch.manual_seed(0)
    net = resnet("ResNet14", REF, 3, 40, 3, dropout=0.0)
    out["resnet/init_digest"] = state_digest(net)
    y, loss = T._resnet_step(REF, net, "cpu")
    perm = np.argsort(y.C.numpy()[:, 0], kind="stable")        # rows in ascending batch order
    out["resnet/out_coords"] = y.C.numpy()[perm]
    out["resnet/logits"] = y.F.detach().numpy().astype(np.float32)[perm]
    out["resnet/loss"] = np.float64(loss)
    params = dict(net.named_parameters())
    for p in RESNET_PARAMS:
        gr = params[p].grad.numpy().ravel()
        idx = sample_index(gr.size, SAMPLE_ELEMS, 2)
        out[f"resnet/{p}/idx"] = idx.astype(np.int64)
        out[f"resnet/{p}/grad"] = gr[idx].astype(np.float32)
        out[f"resnet/{p}/absmax"] = np.float64(np.abs(gr).max())
    print("resnet loss", loss, flush=True)
    torch.manual_seed(1)
    blk = se_basic_block(REF, 32, 32, dimension=3)
    out["se/init_digest"] = state_digest(blk)
    y, x = T._se_step(REF, blk, "cpu")
    out["se/out_feats"] = y.F.detach().numpy()
    out["se/grad_in"] = x.F.grad.numpy()
    for p, t in blk.named_parameters():
        if p in SE_PARAMS:
            out[f"se/{p}/grad"] = t.grad.numpy()
    np.savez_compressed(os.path.join(HERE, "ref_resnet.npz"), **out)


def main():
    from oracle import ref
    ME = ref.import_reference()
    torch.set_num_threads(os.cpu_count() or 1)
    for i, mode in enumerate(("sum", "avg", "max")):
        global_case(ME, mode, 20 + i)
    broadcast_case(ME, "add", 23)
    broadcast_case(ME, "mul", 24)
    instnorm_case(ME, 25)
    resnet_case(ME)


if __name__ == "__main__":
    main()
