"""Channel-wise (depthwise) convolution on the GPU: the native kernels (csrc/chwise.cu) against the
float64 restatement (tests/chwise_oracle.py) element by element in fp32, bf16 and fp16, the public layer
against the compiled reference's fixtures (tests/golden/ref_chwise_*, written by
tests/golden/make_chwise_fixtures.py), and one training step of examples/convnext.py against the
reference's."""
import numpy as np
import pytest
import torch

import chwise_oracle as CO
from helpers import assert_one_rounding, golden, one_rounding_ratio as _ratio, rel_err, state_digest
from oracle import oracle_np as O

pytestmark = pytest.mark.gpu

# ---- cases shared with tests/golden/make_chwise_fixtures.py (run there on the reference) ---------
CASES = {
    "d3_k3_s1": dict(D=3, k=3, s=1, d=1, C=8, bias=False),
    "d3_k3_s2": dict(D=3, k=3, s=2, d=1, C=5, bias=False),
    "d3_k2_s2": dict(D=3, k=2, s=2, d=1, C=16, bias=False),
    "d3_k5_dil2": dict(D=3, k=5, s=1, d=2, C=4, bias=False),
    "d3_cross_k5": dict(D=3, k=5, s=1, d=1, C=6, bias=False, region="HYPER_CROSS"),
    "d3_k7": dict(D=3, k=7, s=1, d=1, C=8, bias=False),
    "d2_k3_s2_bias": dict(D=2, k=3, s=2, d=1, C=3, bias=True),
    "d4_k3": dict(D=4, k=3, s=1, d=1, C=4, bias=False),
}
_EXTENT = {2: 12, 3: 8, 4: 5}
_POINTS = {2: 300, 3: 1500, 4: 1500}


def case_coords(spec, seed):
    """Unique rows of three clouds with negative coordinates."""
    D = spec["D"]
    g = torch.Generator().manual_seed(seed)
    c = torch.randint(-_EXTENT[D], _EXTENT[D], (_POINTS[D], D), generator=g, dtype=torch.int32)
    b = torch.randint(0, 3, (_POINTS[D], 1), generator=g, dtype=torch.int32)
    return torch.unique(torch.cat([b, c], 1), dim=0)


def make_layer(MEh, spec):
    rt = getattr(MEh.RegionType, spec.get("region", "HYPER_CUBE"))
    kg = MEh.KernelGenerator(kernel_size=spec["k"], stride=spec["s"], dilation=spec["d"],
                             region_type=rt, dimension=spec["D"])
    return MEh.MinkowskiChannelwiseConvolution(spec["C"], bias=spec["bias"], kernel_generator=kg,
                                               dimension=spec["D"])


CONVNEXT_SEED = 3
CONVNEXT_CLASSES = 10
CONVNEXT_PARAMS = ("stem.0.kernel", "stages.0.0.dwconv.kernel", "stages.1.2.dwconv.kernel",
                   "stages.1.2.pwconv2.linear.weight", "head.linear.weight")


def _convnext_step(MEh, net, dev):
    from examples.synthetic import surface_cloud
    coords = torch.cat([surface_cloud(1500, seed=60 + b, batch=b) for b in range(4)])
    g = torch.Generator().manual_seed(6)
    feats = torch.rand(len(coords), 3, generator=g)
    labels = torch.randint(0, CONVNEXT_CLASSES, (4,), generator=g)
    net = net.to(dev).train()
    out = net(MEh.SparseTensor(feats.to(dev), coords.to(dev)))
    loss = torch.nn.functional.cross_entropy(out.F.float(), labels.to(dev)[out.C[:, 0].long()])
    loss.backward()
    return out, float(loss.detach())


# ---- direct library calls ------------------------------------------------------------------------
def _gather(x, W, nbr):
    from minkowskiengine_b200 import _lib
    K, n_rows = nbr.shape
    C = x.shape[1]
    y = torch.empty((n_rows, C), dtype=x.dtype, device=x.device)
    _lib.check(_lib.load().meb200_chwise_gather(
        _lib.ptr(x), _lib.dtype_code(x.dtype), x.shape[0], C, _lib.ptr(W), _lib.ptr(nbr), K, n_rows,
        _lib.ptr(y), _lib.current_stream()))
    return y


def _wgrad(x, g, nbr, workspace="plan"):
    """workspace: "plan" (the size the library asks for), None, or a uint8 tensor."""
    from minkowskiengine_b200 import _lib
    lib = _lib.load()
    K, n_out = nbr.shape
    C = x.shape[1]
    code = _lib.dtype_code(x.dtype)
    if isinstance(workspace, str):
        nbytes = int(lib.meb200_chwise_wgrad_workspace_bytes(n_out, C, K, code))
        workspace = torch.empty(nbytes, dtype=torch.uint8, device=x.device) if nbytes else None
    dW = torch.empty((K, C), dtype=torch.float32, device=x.device)
    _lib.check(lib.meb200_chwise_wgrad(
        _lib.ptr(x), _lib.ptr(g), code, x.shape[0], C, _lib.ptr(nbr), K, n_out, _lib.ptr(dW),
        _lib.ptr(workspace), 0 if workspace is None else workspace.numel(), _lib.current_stream()))
    return dW


def _table(K, n_rows, n_other, density, seed, device):
    """Random k-major table [K, n_rows] with rows that have no neighbour and, for K > 2, an offset
    without any pair."""
    g = torch.Generator().manual_seed(seed)
    idx = torch.randint(0, n_other, (K, n_rows), generator=g, dtype=torch.int32)
    idx[torch.rand((K, n_rows), generator=g) > density] = -1
    idx[:, ::97] = -1
    if K > 2:
        idx[K // 2] = -1
    return idx.to(device)


def _operands(C, K, n_rows, n_other, dtype, cuda, seed):
    g = torch.Generator().manual_seed(seed)
    x = (torch.rand(n_other, C, generator=g) - 0.5).to(dtype).to(cuda)
    go = (torch.rand(n_rows, C, generator=g) - 0.5).to(dtype).to(cuda)
    W = ((torch.rand(K, C, generator=g) - 0.5) / K ** 0.5).to(cuda)
    out_nbr = _table(K, n_rows, n_other, 0.4, seed + 1, cuda)      # rows of go -> rows of x
    in_nbr = _table(K, n_other, n_rows, 0.4, seed + 2, cuda)       # rows of x -> rows of go
    return x, go, W, out_nbr, in_nbr


def _check_all(x, go, W, out_nbr, in_nbr, what):
    """Forward, input gradient and weight gradient within one rounding, each bit-identical over
    two calls.  Returns the worst ratios (fwd, dgrad, wgrad)."""
    y = _gather(x, W, out_nbr)
    ref, A = CO.gather(x, W, out_nbr)
    assert_one_rounding(y, ref, A, f"{what} forward")
    gi = _gather(go, W, in_nbr)
    refi, Ai = CO.gather(go, W, in_nbr)
    assert_one_rounding(gi, refi, Ai, f"{what} input gradient")
    dW = _wgrad(x, go, out_nbr)
    refw, Aw = CO.wgrad(x, go, out_nbr)
    assert_one_rounding(dW, refw, Aw, f"{what} weight gradient")
    assert torch.equal(y, _gather(x, W, out_nbr)), what
    assert torch.equal(gi, _gather(go, W, in_nbr)), what
    assert torch.equal(dW, _wgrad(x, go, out_nbr)), what
    return _ratio(y, ref, A), _ratio(gi, refi, Ai), _ratio(dW, refw, Aw)


# ---- the kernels, element by element -------------------------------------------------------------
# fp32 reads 4-channel vectors when C % 4 == 0 (C = 4, 12, 20 among them), bf16 / fp16 8-channel
# ones when C % 8 == 0; every other C reads single channels
@pytest.mark.parametrize("K", [1, 27, 125, 343])
@pytest.mark.parametrize("C", [1, 3, 4, 8, 12, 20, 24, 64, 96, 200, 256, 512])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16],
                         ids=["fp32", "bf16", "fp16"])
def test_kernels_one_rounding(cuda, dtype, C, K):
    ops = _operands(C, K, 700, 500, dtype, cuda, 1000 + C + K)
    r = _check_all(*ops, f"{dtype} C={C} K={K}")
    print(f"chwise ratio {dtype} C={C} K={K}: fwd {r[0]:.3f} dgrad {r[1]:.3f} wgrad {r[2]:.3f}")


@pytest.mark.parametrize("n_rows", [1, 255, 256, 257, 1023, 1024, 1025, 2049, 40_000])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
def test_row_counts_at_tile_and_split_edges(cuda, dtype, n_rows):
    ops = _operands(64, 27, n_rows, 3000, dtype, cuda, 7 + n_rows)
    _check_all(*ops, f"{dtype} n_rows={n_rows}")


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
def test_zero_rows_launch_nothing(cuda, dtype):
    from minkowskiengine_b200 import _lib
    x = torch.rand(10, 8, device=cuda).to(dtype)
    W = torch.rand(27, 8, device=cuda)
    nbr = torch.empty((27, 0), dtype=torch.int32, device=cuda)
    n0 = _lib.launch_count()
    y = _gather(x, W, nbr)
    dW = _wgrad(x, torch.empty((0, 8), dtype=dtype, device=cuda), nbr)
    torch.cuda.synchronize()
    assert _lib.launch_count() == n0
    assert y.shape == (0, 8) and torch.equal(dW, torch.zeros_like(dW))


def test_wgrad_workspace_full_small_and_none(cuda):
    """fp32 (4-channel vectors) and bf16 (8-channel vectors)."""
    from minkowskiengine_b200 import _lib
    for dtype in (torch.float32, torch.bfloat16):
        x, go, W, out_nbr, _ = _operands(64, 27, 50_000, 20_000, dtype, cuda, 5)
        nbytes = int(_lib.load().meb200_chwise_wgrad_workspace_bytes(50_000, 64, 27,
                                                                     _lib.dtype_code(dtype)))
        slot = 27 * 64 * 4
        assert nbytes >= 3 * slot, f"{dtype}: the plan should split this layer's rows"
        ref, A = CO.wgrad(x, go, out_nbr)
        full = _wgrad(x, go, out_nbr)
        small = _wgrad(x, go, out_nbr, torch.empty(2 * slot, dtype=torch.uint8, device=cuda))
        none = _wgrad(x, go, out_nbr, None)
        unaligned = _wgrad(x, go, out_nbr, torch.empty(nbytes + 16, dtype=torch.uint8,
                                                       device=cuda)[8:8 + nbytes])
        for what, dW in (("full", full), ("small", small), ("none", none),
                         ("unaligned", unaligned)):
            assert_one_rounding(dW, ref, A, f"{dtype} workspace {what}")
        assert torch.equal(none, unaligned), dtype    # an unaligned workspace means one split
        print(f"chwise wgrad ratio {dtype} one split over 50k rows: {_ratio(none, ref, A):.3f}, "
              f"planned splits: {_ratio(full, ref, A):.3f}")


# ---- the public layer ----------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(CASES))
def test_layer_matches_reference(ME, cuda, name):
    G = golden(f"ref_chwise_{name}.npz")
    spec = CASES[name]
    layer = make_layer(ME, spec).to(cuda)
    with torch.no_grad():
        layer.kernel.copy_(torch.as_tensor(G["kernel"]))
        if spec["bias"]:
            layer.bias.copy_(torch.as_tensor(G["bias"]))
    x = ME.SparseTensor(torch.as_tensor(G["in_feats"]).to(cuda),
                        torch.as_tensor(G["in_coords"]).to(cuda), requires_grad=True)
    y = layer(x)
    perm = np.lexsort(y.C.cpu().numpy().T[::-1])
    assert (y.C.cpu().numpy()[perm] == G["out_coords"]).all()
    assert rel_err(y.F.detach().cpu().numpy()[perm], G["out_feats"]) < 1e-5
    g = torch.empty_like(y.F)
    g[torch.as_tensor(perm, device=cuda)] = torch.as_tensor(G["grad_out"]).to(cuda)
    y.F.backward(g)
    assert rel_err(x.F.grad.cpu(), G["grad_in"]) < 1e-5
    assert rel_err(layer.kernel.grad.cpu(), G["grad_kernel"]) < 1e-5
    if spec["bias"]:
        assert rel_err(layer.bias.grad.cpu(), G["grad_out"].sum(0, keepdims=True)) < 1e-5


def _cloud_tensor(ME, cuda, C, dtype=torch.float32, seed=11):
    coords = case_coords(dict(D=3), seed)
    feats = (torch.rand(len(coords), C, generator=torch.Generator().manual_seed(seed + 2)) - 0.5)
    return ME.SparseTensor(feats.to(dtype).to(cuda), coords.to(cuda), requires_grad=True)


def test_shares_the_convolution_kernel_map(ME, cuda):
    x = _cloud_tensor(ME, cuda, 16)
    kms = x.coordinate_manager._manager._kernel_maps
    n0 = len(kms)
    ME.MinkowskiChannelwiseConvolution(16, kernel_size=3, stride=2, dimension=3).to(cuda)(x)
    n1 = len(kms)
    ME.MinkowskiConvolution(16, 16, kernel_size=3, stride=2, dimension=3).to(cuda)(x)
    assert n1 == n0 + 1 and len(kms) == n1


def test_coordinates_argument_gives_rows_on_that_map(ME, cuda):
    x = _cloud_tensor(ME, cuda, 8)
    want = torch.unique(x.C[::3].cpu(), dim=0)
    want = want[torch.randperm(len(want), generator=torch.Generator().manual_seed(1))]
    layer = ME.MinkowskiChannelwiseConvolution(8, kernel_size=3, dimension=3).to(cuda)
    y = layer(x, coordinates=want.to(cuda))
    assert torch.equal(y.C.cpu(), want)
    y2 = layer(x, coordinates=y)                          # a SparseTensor
    y3 = layer(x, coordinates=y.coordinate_map_key)       # a key
    assert torch.equal(y2.F, y.F) and torch.equal(y3.F, y.F)
    in_c = x.C.cpu().numpy()
    offs = O.region_offsets(O.HYPER_CUBE, [3] * 3, [1] * 3, [1] * 3)
    im, om = O.kernel_map(in_c, want.numpy(), offs)
    ref = CO.forward(x.F.detach().cpu().numpy(), layer.kernel.detach().cpu().numpy(), im, om,
                     len(want))
    assert rel_err(y.F.detach().cpu(), ref) < 1e-6


def test_adjoint_in_float64_arithmetic(ME, cuda):
    x = _cloud_tensor(ME, cuda, 24)
    layer = ME.MinkowskiChannelwiseConvolution(24, kernel_size=3, stride=2, dimension=3).to(cuda)
    y = layer(x)
    g = torch.rand(y.F.shape, generator=torch.Generator().manual_seed(3)).to(cuda) - 0.5
    y.F.backward(g)
    lhs = float((y.F.detach().double() * g.double()).sum())
    rhs = float((x.F.detach().double() * x.F.grad.double()).sum())
    assert abs(lhs - rhs) <= 1e-5 * (y.F.detach().double().abs() * g.double().abs()).sum().item()


def test_bf16_kernel_and_output_dtype(ME, cuda):
    x = _cloud_tensor(ME, cuda, 32, torch.bfloat16)
    layer = ME.MinkowskiChannelwiseConvolution(32, kernel_size=5, bias=True, dimension=3).to(cuda)
    ref_layer = ME.MinkowskiChannelwiseConvolution(32, kernel_size=5, bias=True, dimension=3)
    ref_layer = ref_layer.to(cuda)
    layer = layer.bfloat16()
    with torch.no_grad():
        ref_layer.kernel.copy_(layer.kernel.float())
        ref_layer.bias.copy_(layer.bias.float())
    y, yr = layer(x), ref_layer(x)
    assert y.F.dtype == torch.bfloat16 and yr.F.dtype == torch.bfloat16
    assert torch.equal(y.F, yr.F)        # the bf16 kernel is read as fp32: the same values
    y.F.float().sum().backward()
    assert layer.kernel.grad.dtype == torch.bfloat16 and layer.bias.grad.dtype == torch.bfloat16


def test_kernel_volume_one_runs_the_native_kernel(ME, cuda):
    from minkowskiengine_b200 import _lib
    x = _cloud_tensor(ME, cuda, 8)
    layer = ME.MinkowskiChannelwiseConvolution(8, kernel_size=1, dimension=3).to(cuda)
    layer(x)                                          # builds the (identity) kernel map
    n0 = _lib.launch_count()
    y = layer(x)
    assert _lib.launch_count() == n0 + 1
    ref = x.F.detach().double() * layer.kernel.detach().double()
    assert rel_err(y.F.detach().cpu(), ref.cpu()) < 1e-6


def test_errors(ME, cuda):
    x = _cloud_tensor(ME, cuda, 8)
    with pytest.raises(AssertionError, match="Channel size mismatch"):
        ME.MinkowskiChannelwiseConvolution(7, kernel_size=3, dimension=3).to(cuda)(x)
    x64 = ME.SparseTensor(x.F.detach().double(), coordinate_map_key=x.coordinate_map_key,
                          coordinate_manager=x.coordinate_manager)
    with pytest.raises(RuntimeError):
        ME.MinkowskiChannelwiseConvolution(8, kernel_size=3, dimension=3).to(cuda).double()(x64)
    with pytest.raises(RuntimeError):
        ME.MinkowskiChannelwiseConvolution(8, kernel_size=3, dimension=3)(x)   # CPU kernel


# ---- the network -----------------------------------------------------------------------------------
def test_convnext_fp32_step_matches_reference(ME, cuda):
    from examples.convnext import convnext
    G = golden("ref_chwise_convnext.npz")
    torch.manual_seed(CONVNEXT_SEED)
    net = convnext(ME, 3, CONVNEXT_CLASSES, 3)
    assert (state_digest(net) == G["init_digest"]).all(), \
        "seeded initial weights differ from the reference's"
    out, loss = _convnext_step(ME, net, cuda)
    assert (out.C.cpu().numpy() == G["out_coords"]).all()
    F, R = out.F.detach().cpu().numpy(), G["logits"]
    assert np.abs(F - R).max() / np.abs(R).max() < 1e-3
    assert abs(loss - float(G["loss"])) / abs(float(G["loss"])) < 1e-3
    # as for ResNet14 (test_gpu_global.py): the layers next to the loss tightly, the deeper ones,
    # below train-mode batch norms that amplify fp32 round-off, by direction
    params = dict(net.named_parameters())
    for p in CONVNEXT_PARAMS:
        gg = params[p].grad.cpu().numpy().ravel()[G[f"{p}/idx"]].astype(np.float64)
        gr = G[f"{p}/grad"].astype(np.float64)
        if p in ("stages.1.2.pwconv2.linear.weight", "head.linear.weight"):
            assert np.abs(gg - gr).max() / float(G[f"{p}/absmax"]) < 2e-3, p
        else:
            cos = float(gg @ gr / (np.linalg.norm(gg) * np.linalg.norm(gr)))
            assert cos > 0.9995 and np.abs(gg - gr).max() / float(G[f"{p}/absmax"]) < 5e-2, p
