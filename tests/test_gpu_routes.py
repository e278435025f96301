"""The convolution routes off the wgmma grid, in fp32, bf16 and fp16, against a float64
restatement on the device, element by element.

`meb200_conv_{forward,backward}` send a layer to one of several kernels by dtype and channel
counts: `k_conv_wg` / `k_wgrad_wg` (tensor cores) when every side is on the 16-channel grid,
`k_conv_gather_gemm` / `k_conv_wgrad` (SIMT) when one is not, `k_conv_small_cin_{fwd,wgrad}` for
c_in <= 4, and mixtures (forward in 256-column tensor-core slices with a SIMT wgrad for c_out >
256; SIMT dgrad with the dense-table `k_wgrad_wg` when only the wgrad qualifies).  Every case
states which route it covers through the tensor-core launch counter, so that a change of dispatch
cannot move a case to another route unnoticed.  Under torch's default matmul switch, which this
file pins, fp32 launches no tensor-core kernel in any case.

Bound (tests/helpers.py): |y - ref| <= delta = 2^-20 * A in fp32 and one rounding on top of that in
bf16 / fp16, A the same reduction over absolute values.  The weight gradients are fp32 and must be
bit-identical run to run: every split's partial sums are added in a fixed order."""
import pytest
import torch

from helpers import (_Route, _inputs, _pairs, _table, assert_one_rounding, one_rounding_ratio,
                     ref_conv, ref_wgrad)
from oracle import oracle_np as O

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def exact_fp32():
    """fp32 convolutions on the CUDA cores: torch's default matmul switch, restored afterwards."""
    saved = torch.backends.cuda.matmul.fp32_precision
    torch.backends.cuda.matmul.fp32_precision = "ieee"
    yield
    torch.backends.cuda.matmul.fp32_precision = saved


# (cin, cout, n_in, n_out, K, forward on tensor cores, dgrad on tensor cores) in bf16 / fp16
# The wgrad of every case runs on CUDA cores: k_conv_small_cin_wgrad for cin <= 4 and cout <= 64,
# else k_conv_wgrad.  The last two have cout off the 16-channel grid, so that the bf16 / fp16 stem
# kernels do not take them either.
ROUTES = {
    "head_96to20_k1": (96, 20, 200_000, 200_000, 1, False, False),    # MinkUNet head
    "cout1": (16, 1, 20_000, 20_000, 27, False, False),              # completion classifiers
    "cin20": (20, 32, 20_000, 20_000, 27, False, False),
    "cin8": (8, 16, 20_000, 20_000, 27, False, False),
    "cout272_slices": (128, 272, 8_000, 8_000, 27, True, True),        # two column slices
    "cout512_slices": (64, 512, 8_000, 8_000, 8, True, True),
    "stem_3to20_k125": (3, 20, 50_000, 50_000, 125, False, False),   # k_conv_small_cin_*
    # the small-cin forward's fallback to k_conv_gather_gemm: K * c_in * 64 fp32 weights > 200 KB
    "stem_4to56_k343": (4, 56, 20_000, 20_000, 343, False, False),
    "cin3_cout72": (3, 72, 20_000, 20_000, 27, False, False),        # c_out > 64: no small-cin
}


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16],
                         ids=["fp32", "bf16", "fp16"])
@pytest.mark.parametrize("case", list(ROUTES))
def test_route_forward_dgrad_wgrad(ME, cuda, case, dtype):
    from minkowskiengine_b200 import backend
    cin, cout, n_in, n_out, K, fwd_tc, dgrad_tc = ROUTES[case]
    if dtype == torch.float32:
        fwd_tc = dgrad_tc = False
    feats, gout, w = _inputs(cin, cout, n_in, n_out, K, dtype, cuda, seed=cin * 131 + cout)
    wl = w.to(dtype)
    out_nbr = _table(K, n_out, n_in, 0.35, seed=K + n_out, device=cuda)
    in_nbr = _table(K, n_in, n_out, 0.3, seed=K + n_in + 3, device=cuda)
    km = backend._KernelMap(out_nbr, in_nbr)
    y_ref, y_A = ref_conv(feats, wl, _pairs(out_nbr), n_out)
    with _Route(fwd_tc, f"{case} forward"):
        y = backend._conv_forward(feats, w, km)
        y2 = backend._conv_forward(feats, w, km)
        y32 = backend._conv_forward(feats, w, km, out_dtype=torch.float32)
    assert torch.equal(y, y2), f"{case} forward differs run to run"
    assert y.dtype == dtype and y32.dtype == torch.float32
    assert_one_rounding(y, y_ref, y_A, f"{case} forward")
    assert_one_rounding(y32, y_ref, y_A, f"{case} forward, fp32 output")

    gi_ref, gi_A = ref_conv(gout, wl.transpose(1, 2), _pairs(in_nbr), n_in)
    with _Route(dgrad_tc, f"{case} dgrad"):
        gi, _ = backend._conv_backward(feats, gout, w, km, need_in=True, need_w=False)
        gi2, _ = backend._conv_backward(feats, gout, w, km, need_in=True, need_w=False)
    assert gi.dtype == dtype
    assert_one_rounding(gi, gi_ref, gi_A, f"{case} dgrad")
    assert torch.equal(gi, gi2), f"{case} dgrad differs run to run"

    gw_ref, gw_A = ref_wgrad(feats, gout, _pairs(out_nbr))
    with _Route(False, f"{case} wgrad"):
        _, gw = backend._conv_backward(feats, gout, w, km, need_in=False, need_w=True)
        _, gw2 = backend._conv_backward(feats, gout, w, km, need_in=False, need_w=True)
    assert km._pairs is None, f"{case}: pair lists built for a wgrad that does not read them"
    assert gw.dtype == torch.float32
    assert_one_rounding(gw, gw_ref, gw_A, f"{case} wgrad")
    assert torch.equal(gw, gw2), f"{case} wgrad differs run to run"
    print(f"route ratio {dtype} {case}: fwd {one_rounding_ratio(y32, y_ref, y_A):.3f} "
          f"dgrad {one_rounding_ratio(gi, gi_ref, gi_A):.3f} "
          f"wgrad {one_rounding_ratio(gw, gw_ref, gw_A):.3f}")


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def test_simt_dgrad_with_tc_wgrad(ME, cuda, dtype):
    """24 -> 32: the dgrad (24 output columns) is off the grid, the wgrad is not.  Each picks its
    kernel on its own: SIMT dgrad, `k_wgrad_wg` over the pair lists, whose bits do not depend on
    whether the dgrad ran in the same call."""
    from minkowskiengine_b200 import backend
    cin, cout, n_in, n_out, K = 24, 32, 30_000, 30_000, 27
    feats, gout, w = _inputs(cin, cout, n_in, n_out, K, dtype, cuda, seed=2432)
    wl = w.to(dtype)
    out_nbr = _table(K, n_out, n_in, 0.35, seed=5, device=cuda)
    in_nbr = _table(K, n_in, n_out, 0.35, seed=6, device=cuda)
    km = backend._KernelMap(out_nbr, in_nbr)
    with _Route(False, "24->32 dgrad alone"):
        backend._conv_backward(feats, gout, w, km, need_in=True, need_w=False)
    with _Route(True, "24->32 wgrad alone"):
        _, gw_alone = backend._conv_backward(feats, gout, w, km, need_in=False, need_w=True)
    with _Route(True, "24->32 dgrad + wgrad"):
        gi, gw = backend._conv_backward(feats, gout, w, km, need_in=True, need_w=True)
        _, gw2 = backend._conv_backward(feats, gout, w, km, need_in=True, need_w=True)
    assert km._pairs is not None
    gi_ref, gi_A = ref_conv(gout, wl.transpose(1, 2), _pairs(in_nbr), n_in)
    assert_one_rounding(gi, gi_ref, gi_A, "24->32 dgrad")
    gw_ref, gw_A = ref_wgrad(feats, gout, _pairs(out_nbr))
    assert_one_rounding(gw, gw_ref, gw_A, "24->32 pair-list wgrad")
    assert torch.equal(gw, gw2)
    assert torch.equal(gw, gw_alone), "the wgrad depends on whether dgrad was requested"


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def test_dense_table_tc_wgrad_large_kernel(ME, cuda, dtype):
    """32 -> 32 with an 11^3 kernel: K > 1023 is past the pair lists' range, so the wgrad is
    `k_wgrad_wg` over the dense neighbour table (thousands of pairs per offset, as in a layer)."""
    from minkowskiengine_b200 import backend
    cin, cout, n, K = 32, 32, 3_000, 11 ** 3
    feats, gout, w = _inputs(cin, cout, n, n, K, dtype, cuda, seed=1331)
    out_nbr = _table(K, n, n, 0.9, seed=7, device=cuda)
    km = backend._KernelMap(out_nbr, torch.full((K, n), -1, dtype=torch.int32, device=cuda))
    with _Route(True, "11^3 wgrad"):
        _, gw = backend._conv_backward(feats, gout, w, km, need_in=False, need_w=True)
        _, gw2 = backend._conv_backward(feats, gout, w, km, need_in=False, need_w=True)
    assert km._pairs is None
    gw_ref, gw_A = ref_wgrad(feats, gout, _pairs(out_nbr))
    assert_one_rounding(gw, gw_ref, gw_A, "11^3 dense-table wgrad")
    assert torch.equal(gw, gw2)


# ---- transposed and generative convolution through the public API ------------------------------
def _bf16_weights_(*layers):
    with torch.no_grad():
        for m in layers:
            m.kernel.copy_(m.kernel.bfloat16().float())


def _check_layer(x_F, y, gy, w, pairs, n_out, what):
    """y = conv(x_F) over `pairs` ((in rows, out rows) per offset), gy its output gradient:
    forward, dgrad and wgrad of one layer against float64, given the layer's actual inputs."""
    y_ref, y_A = ref_conv(x_F, w, pairs, n_out)
    assert_one_rounding(y.F.detach(), y_ref, y_A, f"{what} forward")
    return ref_wgrad(x_F, gy, pairs), ref_conv(gy, w.transpose(1, 2),
                                               [(o, i) for i, o in pairs], len(x_F))


def _to_pairs(im, om, device):
    return [(torch.as_tensor(i, dtype=torch.long, device=device),
             torch.as_tensor(o, dtype=torch.long, device=device)) for i, o in zip(im, om)]


@pytest.mark.parametrize("chunk", [None, 2048], ids=["one_chunk", "chunked"])
def test_bf16_conv_then_transpose_vs_oracle_maps(ME, cuda, chunk, monkeypatch):
    """Conv k2 s2 64->96, then ConvolutionTranspose k2 s2 96->64 (the swapped tables and pair
    lists of `_KernelMap.swapped`), bf16, on the oracle's kernel maps."""
    from helpers import unique_cloud
    from minkowskiengine_b200 import backend
    if chunk is not None:
        monkeypatch.setattr(backend._KernelMap, "PAIR_CHUNK_ROWS", chunk)
    D, dt = 3, torch.bfloat16
    coords = unique_cloud(40_000, 40, seed=21, allow_negative=True)
    g = torch.Generator().manual_seed(8)
    feats = (torch.rand(len(coords), 64, generator=g) - 0.5).to(dt)
    down = ME.MinkowskiConvolution(64, 96, kernel_size=2, stride=2, dimension=D).to(cuda)
    up = ME.MinkowskiConvolutionTranspose(96, 64, kernel_size=2, stride=2, dimension=D).to(cuda)
    _bf16_weights_(down, up)
    x = ME.SparseTensor(feats, coords, device=cuda, requires_grad=True)
    y = down(x)
    y.F.retain_grad()
    z = up(y)
    assert z.coordinate_map_key == x.coordinate_map_key
    gz = (torch.rand(z.F.shape, generator=g) - 0.5).to(dt).to(cuda)
    z.F.backward(gz)
    in_c, mid_c = x.C.cpu().numpy(), y.C.cpu().numpy()
    offs = O.region_offsets(O.HYPER_CUBE, [2] * D, [1] * D, [1] * D)
    p_dn = _to_pairs(*O.kernel_map(in_c, mid_c, offs), cuda)
    p_up = _to_pairs(*O.transposed_kernel_map(mid_c, in_c, offs), cuda)
    w_dn, w_up = down.kernel.detach().to(dt), up.kernel.detach().to(dt)
    (gw, gw_A), (gi, gi_A) = _check_layer(y.F.detach(), z, gz, w_up, p_up, len(in_c), "transpose")
    assert_one_rounding(up.kernel.grad, gw, gw_A, "transpose wgrad")
    assert_one_rounding(y.F.grad, gi, gi_A, "transpose dgrad")
    (gw, gw_A), (gi, gi_A) = _check_layer(x.F.detach(), y, y.F.grad, w_dn, p_dn, len(mid_c), "conv")
    assert_one_rounding(down.kernel.grad, gw, gw_A, "conv wgrad")
    assert_one_rounding(x.F.grad, gi, gi_A, "conv dgrad")


def test_bf16_generative_transpose_vs_oracle_maps(ME, cuda):
    from helpers import unique_cloud
    D, dt = 3, torch.bfloat16
    coords = unique_cloud(20_000, 30, seed=23)
    coords[:, 1:] *= 2
    g = torch.Generator().manual_seed(9)
    feats = (torch.rand(len(coords), 96, generator=g) - 0.5).to(dt)
    up = ME.MinkowskiGenerativeConvolutionTranspose(96, 64, kernel_size=2, stride=2,
                                                    dimension=D).to(cuda)
    _bf16_weights_(up)
    x = ME.SparseTensor(feats, coords, tensor_stride=2, device=cuda, requires_grad=True)
    z = up(x)
    gz = (torch.rand(z.F.shape, generator=g) - 0.5).to(dt).to(cuda)
    z.F.backward(gz)
    in_c, out_c = x.C.cpu().numpy(), z.C.cpu().numpy()
    offs = O.region_offsets(O.HYPER_CUBE, [2] * D, [1] * D, [1] * D)
    pairs = _to_pairs(*O.transposed_kernel_map(in_c, out_c, offs), cuda)
    assert sum(len(i) for i, _ in pairs) == 8 * len(in_c)     # every offset of every input row
    (gw, gw_A), (gi, gi_A) = _check_layer(x.F.detach(), z, gz, up.kernel.detach().to(dt), pairs,
                                          len(out_c), "generative transpose")
    assert_one_rounding(up.kernel.grad, gw, gw_A, "generative transpose wgrad")
    assert_one_rounding(x.F.grad, gi, gi_A, "generative transpose dgrad")


# ---- bitwise determinism of the rewritten reductions ---------------------------------------------
def _wgrad_twice(ME, cuda, cin, cout, n, K, dtype):
    from minkowskiengine_b200 import backend
    feats, gout, w = _inputs(cin, cout, n, n, K, dtype, cuda, seed=cin + cout + K)
    km = backend._KernelMap(_table(K, n, n, 0.5, seed=n + K, device=cuda),
                            torch.full((K, n), -1, dtype=torch.int32, device=cuda))
    with _Route(False, f"{cin}->{cout} wgrad"):
        a = backend._conv_backward(feats, gout, w, km, need_in=False, need_w=True)[1]
        b = backend._conv_backward(feats, gout, w, km, need_in=False, need_w=True)[1]
    return a, b


def test_simt_wgrad_bitwise_at_800k_rows(ME, cuda):
    a, b = _wgrad_twice(ME, cuda, 96, 20, 800_000, 1, torch.bfloat16)
    assert torch.equal(a, b)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
def test_small_cin_wgrad_bitwise(ME, cuda, dtype):
    a, b = _wgrad_twice(ME, cuda, 3, 20, 300_000, 125, dtype)
    assert torch.equal(a, b)


def _grads(net):
    return {n: p.grad.detach().clone() for n, p in net.named_parameters() if p.grad is not None}


def test_minkunet14_bf16_step_bitwise(ME, cuda):
    from examples.minkunet import minkunet
    torch.manual_seed(0)
    net = minkunet("MinkUNet14", ME, 3, 20, 3).to(cuda).train()
    n = 50_000
    coords = O.surface_cloud(n, seed=5)
    feats = torch.rand(n, 3, generator=torch.Generator().manual_seed(2)).bfloat16()
    runs = []
    for _ in range(2):
        net.zero_grad(set_to_none=True)
        out = net(ME.SparseTensor(feats.to(cuda), coords.to(cuda)))
        out.F.float().pow(2).mean().backward()
        runs.append((out.F.detach().clone(), _grads(net)))
    assert torch.equal(runs[0][0], runs[1][0])
    assert runs[0][1].keys() == runs[1][1].keys() and "final.kernel" in runs[0][1]
    diff = [k for k in runs[0][1] if not torch.equal(runs[0][1][k], runs[1][1][k])]
    assert not diff, diff


def test_completion_net_wide_levels_bf16_step_bitwise(ME, cuda):
    """A completion net whose two deepest levels are 512 and 1024 channels wide: their wgrads run
    on CUDA cores (c_out > 256)."""
    from examples.completion import completion_loss, completion_net, shell_pair
    torch.manual_seed(0)
    ch = (16, 32, 64, 512, 1024)
    net = completion_net(ME, ch, ch).to(cuda).train()
    pairs = [shell_pair(16.0, seed=80 + b, batch=b) for b in range(2)]
    partial = torch.cat([p for p, _ in pairs]).to(cuda)
    full = torch.cat([f for _, f in pairs]).to(cuda)
    runs = []
    for _ in range(2):
        net.zero_grad(set_to_none=True)
        x = ME.SparseTensor(torch.ones(len(partial), 1, dtype=torch.bfloat16, device=cuda), partial)
        target_key, _ = x.coordinate_manager.insert_and_map(full, string_id="target")
        out_cls, targets, _ = net(x, target_key)
        completion_loss(out_cls, targets).backward()
        runs.append(_grads(net))
    assert len(runs[0]) > 0 and runs[0].keys() == runs[1].keys()
    diff = [k for k in runs[0] if not torch.equal(runs[0][k], runs[1][k])]
    assert not diff, diff
