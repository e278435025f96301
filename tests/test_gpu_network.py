"""Network-level parity on the GPU: MinkUNet through this package (CUDA) against the compiled
reference CPU path with identical weights and inputs.  The reference's results are stored in
tests/golden/ref_network.npz (tests/golden/make_reference_runs.py): the output coordinates as a
digest, a seeded sample of logit rows and of gradient elements with the full tensors' maxima.
Both packages initialise MinkUNet identically from the same seed; the reference's initial weights
are stored as a digest and checked first, so a change of initialisation is reported as such."""
import numpy as np
import pytest
import torch

from examples.minkunet import minkunet
from helpers import digest, golden, state_digest
from oracle import oracle_np as O

pytestmark = pytest.mark.gpu


def _run(MEh, net, coords, feats, dev):
    x = MEh.SparseTensor(feats.to(dev), coords.to(dev))
    out = net(x)
    loss = out.F.float().pow(2).mean()
    loss.backward()
    return out, float(loss)


@pytest.mark.parametrize("name,n", [("MinkUNet14", 6000), ("MinkUNet34C", 4000)])
def test_minkunet_fp32_matches_reference(ME, cuda, name, n):
    G, key = golden("ref_network.npz"), f"fp32_{name}_{n}"
    torch.manual_seed(0)
    net_gpu = minkunet(name, ME, 3, 20, 3)
    assert (state_digest(net_gpu) == G[key + "/init_digest"]).all(), \
        "seeded initial weights differ from the reference's"
    net_gpu = net_gpu.to(cuda)
    coords = O.surface_cloud(n, seed=3)
    feats = torch.rand(n, 3, generator=torch.Generator().manual_seed(1))
    out_g, loss_g = _run(ME, net_gpu, coords, feats, cuda)
    loss_r = float(G[key + "/loss"])
    # stride-1 output rows keep the input order on both sides
    assert (digest(out_g.C.cpu()) == G[key + "/coords_digest"]).all()
    a, b = out_g.F.detach().cpu().numpy()[G[key + "/rows"]], G[key + "/logits"]
    assert np.abs(a - b).max() / float(G[key + "/logits_absmax"]) < 1e-3
    assert abs(loss_g - loss_r) / abs(loss_r) < 1e-3
    # gradients of the first and a deep layer (reduction order differs: relative to the max)
    for pname in ("conv0p1s1.kernel", "block4.0.conv1.kernel", "final.kernel"):
        gg = dict(net_gpu.named_parameters())[pname].grad.cpu().numpy().ravel()[G[f"{key}/{pname}/idx"]]
        gr = G[f"{key}/{pname}/grad"]
        # fp32 round-off is amplified through ~30 train-mode batch-norm layers on the way back
        # to the first convolution (observed 4.5e-3 there, <1e-3 at the head); per-op parity
        # is asserted at 1e-5 in test_gpu_parity.py
        tol = 2e-3 if pname == "final.kernel" else 2e-2
        assert np.abs(gg - gr).max() / max(float(G[f"{key}/{pname}/absmax"]), 1e-20) < tol, pname


def _bf16_round_(net):
    """Round every floating parameter to a bf16-representable fp32 value (in place), so that the
    bf16 operand copies this package makes are EXACT images of the reference's fp32 weights."""
    with torch.no_grad():
        for p in net.parameters():
            p.copy_(p.bfloat16().float())


def _ce_step(MEh, net, coords, feats, labels, dev):
    x = MEh.SparseTensor(feats.to(dev), coords.to(dev))
    out = net(x)
    loss = torch.nn.functional.cross_entropy(out.F.float(), labels.to(dev))
    loss.backward()
    return out, float(loss)


# Tolerances of the bf16 path (the path bench.py times: wgmma convolutions on bf16 operands with
# fp32 accumulation, bf16 activations between layers, native bf16 batch-norm).  The reference
# runs fp32 end to end on the SAME bf16-representable inputs and weights, so the only difference
# is the rounding of every stored activation/gradient to bf16 (relative 2^-9 per rounding).
#  * logits: ~100 roundings on the longest path, re-normalised (not damped) by train-mode BN ->
#    a few 1e-2 of the rms.
#  * loss: a mean over all voxels -> errors average out.
#  * kernel.grad: the gradient of a randomly initialised, batch-normalised UNet is badly
#    conditioned on the way back — in fp32 (eps 6e-8) the first convolution's gradient already
#    differs by 4.5e-3 from the reference (test above), an amplification of ~1e5; with bf16
#    (eps 4e-3) the deep layers are therefore only asserted to point the same way (cosine),
#    the layers next to the loss tightly.  Per-LAYER parity of the same kernels is asserted at
#    2e-5 (fp32 output) in test_gpu_tc.py.  Logits are compared on the stored row sample against
#    the full reference tensor's rms / max, cosines on the stored gradient-element sample.
_BF16_TOL = {"logits_rms": 6e-2, "logits_max": 1e-1, "loss": 2e-3}
_GRAD_COS = {"final.kernel": 0.9999, "block8.0.conv1.kernel": 0.95, "convtr7p2s2.kernel": 0.95,
             "block4.0.conv1.kernel": 0.6, "block1.0.conv2.kernel": 0.6, "conv0p1s1.kernel": 0.6}


@pytest.mark.parametrize("name,n", [("MinkUNet14", 50_000), ("MinkUNet34C", 30_000)])
def test_minkunet_bf16_matches_reference(ME, cuda, name, n):
    """BASELINE configs[2] shape (MinkUNet14, 50k-voxel cloud) and the bench model, on the bf16
    path, against the compiled reference (fp32, CPU): logits, loss, first/deep/last kernel.grad."""
    G, key = golden("ref_network.npz"), f"bf16_{name}_{n}"
    torch.manual_seed(0)
    net_gpu = minkunet(name, ME, 3, 20, 3)
    _bf16_round_(net_gpu)
    assert (state_digest(net_gpu) == G[key + "/init_digest"]).all(), \
        "seeded initial weights differ from the reference's"
    net_gpu = net_gpu.to(cuda)
    coords = O.surface_cloud(n, seed=5)
    g = torch.Generator().manual_seed(2)
    feats = torch.rand(n, 3, generator=g).bfloat16()
    labels = torch.randint(0, 20, (n,), generator=g)
    out_g, loss_g = _ce_step(ME, net_gpu, coords, feats, labels, cuda)
    loss_r = float(G[key + "/loss"])
    assert out_g.F.dtype == torch.bfloat16
    assert (digest(out_g.C.cpu()) == G[key + "/coords_digest"]).all()
    a, b = out_g.F.detach().float().cpu().numpy()[G[key + "/rows"]], G[key + "/logits"]
    e_rms = np.sqrt(((a - b) ** 2).mean()) / float(G[key + "/logits_rms"])
    e_max = np.abs(a - b).max() / float(G[key + "/logits_absmax"])
    e_loss = abs(loss_g - loss_r) / abs(loss_r)
    print(f"\n[{name} bf16 vs reference fp32, {n} voxels] logits rms {e_rms:.2e} max {e_max:.2e} "
          f"loss {loss_g:.5f} vs {loss_r:.5f} ({e_loss:.2e})")
    pg = dict(net_gpu.named_parameters())
    fails = []
    if not (e_rms < _BF16_TOL["logits_rms"] and e_max < _BF16_TOL["logits_max"]):
        fails.append("logits")
    if not e_loss < _BF16_TOL["loss"]:
        fails.append("loss")
    for pname in ("conv0p1s1.kernel", "block1.0.conv2.kernel", "block4.0.conv1.kernel",
                  "convtr7p2s2.kernel", "block8.0.conv1.kernel", "final.kernel"):
        gg = pg[pname].grad.float().cpu().numpy().ravel()[G[f"{key}/{pname}/idx"]].astype(np.float64)
        gr = G[f"{key}/{pname}/grad"].astype(np.float64)
        cos = float(gg @ gr / (np.linalg.norm(gg) * np.linalg.norm(gr) + 1e-300))
        rms = float(np.linalg.norm(gg - gr) / (np.linalg.norm(gr) + 1e-300))
        print(f"    grad {pname:24s} cos {cos:.6f} rel-rms {rms:.2e}")
        if not cos > _GRAD_COS[pname]:
            fails.append(pname)
    assert not fails, fails
