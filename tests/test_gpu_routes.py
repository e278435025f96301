"""The convolution routes off the wgmma grid, in bf16 / fp16, against a float64 restatement on the
device, element by element.

`meb200_conv_{forward,backward}` send a layer to one of several kernels by dtype and channel
counts: `k_conv_wg` / `k_wgrad_wg` (tensor cores) when every side is on the 16-channel grid,
`k_conv_gather_gemm` / `k_conv_wgrad` (SIMT) when one is not, `k_conv_small_cin_{fwd,wgrad}` for
c_in <= 4, and mixtures (forward in 256-column tensor-core slices with a SIMT wgrad for c_out >
256; SIMT dgrad with the dense-table `k_wgrad_wg` when only the wgrad qualifies).  Every case
states which route it covers through the tensor-core launch counter, so that a change of dispatch
cannot move a case to another route unnoticed.

Bound (tests/helpers.py): |y - ref| <= delta = 2^-20 * A in fp32 and one rounding on top of that in
bf16 / fp16, A the same reduction over absolute values.  The weight gradients are fp32 and must be
bit-identical run to run: every split's partial sums are added in a fixed order."""
import pytest
import torch

from helpers import assert_one_rounding
from oracle import oracle_np as O

pytestmark = pytest.mark.gpu


def _table(K, n_rows, n_other, density, seed, device):
    """Random k-major neighbour table [K, n_rows] with fully empty rows and an all-empty offset."""
    g = torch.Generator().manual_seed(seed)
    idx = torch.randint(0, n_other, (K, n_rows), generator=g, dtype=torch.int32)
    idx[torch.rand((K, n_rows), generator=g) > density] = -1
    idx[:, ::97] = -1                     # rows without any neighbour
    if K > 1:
        idx[K // 2] = -1                  # an offset without any pair
    return idx.to(device)


def _pairs(nbr):
    """[(rows of the other side, table rows)] per offset of a k-major table."""
    out = []
    for k in range(nbr.shape[0]):
        o = torch.nonzero(nbr[k] >= 0).flatten()
        out.append((nbr[k][o].long(), o))
    return out


def ref_conv(x, w, pairs, n_out):
    """float64 y[o] = sum over offsets k and pairs (i, o) of x[i] @ w[k]; and the same reduction
    over |x| and |w| (the scale of the accumulation error)."""
    x, w = x.double(), w.double()
    y = torch.zeros((n_out, w.shape[2]), dtype=torch.float64, device=x.device)
    A = torch.zeros_like(y)
    for k, (i, o) in enumerate(pairs):
        if len(i):
            y.index_add_(0, o, x[i] @ w[k])
            A.index_add_(0, o, x[i].abs() @ w[k].abs())
    return y, A


def ref_wgrad(x, g, pairs):
    """float64 dW[k] = sum over pairs (i, o) of x[i]^T g[o], and over |x|, |g|."""
    x, g = x.double(), g.double()
    K = len(pairs)
    gw = torch.zeros((K, x.shape[1], g.shape[1]), dtype=torch.float64, device=x.device)
    A = torch.zeros_like(gw)
    for k, (i, o) in enumerate(pairs):
        if len(i):
            gw[k] = x[i].t() @ g[o]
            A[k] = x[i].abs().t() @ g[o].abs()
    return gw, A


def _inputs(cin, cout, n_in, n_out, K, dtype, device, seed):
    g = torch.Generator().manual_seed(seed)
    feats = (torch.rand(n_in, cin, generator=g) - 0.5).to(dtype).to(device)
    gout = (torch.rand(n_out, cout, generator=g) - 0.5).to(dtype).to(device)
    w = ((torch.rand(K, cin, cout, generator=g) - 0.5) / (cin ** 0.5)).to(device)  # fp32 master
    return feats, gout, w


class _Route:
    """Counts tensor-core launches over a block and checks the route the case is meant to take."""

    def __init__(self, tc, what):
        self.tc, self.what = tc, what

    def __enter__(self):
        from minkowskiengine_b200 import _lib
        self.n0 = _lib.tc_launch_count()
        return self

    def __exit__(self, *exc):
        from minkowskiengine_b200 import _lib
        if exc[0] is None:
            n = _lib.tc_launch_count() - self.n0
            assert (n > 0) == self.tc, \
                f"{self.what}: {n} tensor-core launches, expected {'some' if self.tc else 'none'}"


# (cin, cout, n_in, n_out, K, forward on tensor cores, dgrad on tensor cores)
# The wgrad of every case runs on CUDA cores: k_conv_small_cin_wgrad for cin <= 4, else k_conv_wgrad.
ROUTES = {
    "head_96to20_k1": (96, 20, 200_000, 200_000, 1, False, False),    # MinkUNet head
    "cout1": (16, 1, 20_000, 20_000, 27, False, False),              # completion classifiers
    "cin20": (20, 32, 20_000, 20_000, 27, False, False),
    "cin8": (8, 16, 20_000, 20_000, 27, False, False),
    "cout272_slices": (128, 272, 8_000, 8_000, 27, True, True),        # two column slices
    "cout512_slices": (64, 512, 8_000, 8_000, 8, True, True),
    "stem_3to20_k125": (3, 20, 50_000, 50_000, 125, False, False),   # k_conv_small_cin_*
}


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("case", list(ROUTES))
def test_route_forward_dgrad_wgrad(ME, cuda, case, dtype):
    from minkowskiengine_b200 import backend
    cin, cout, n_in, n_out, K, fwd_tc, dgrad_tc = ROUTES[case]
    feats, gout, w = _inputs(cin, cout, n_in, n_out, K, dtype, cuda, seed=cin * 131 + cout)
    wl = w.to(dtype)
    out_nbr = _table(K, n_out, n_in, 0.35, seed=K + n_out, device=cuda)
    in_nbr = _table(K, n_in, n_out, 0.3, seed=K + n_in + 3, device=cuda)
    km = backend._KernelMap(out_nbr, in_nbr)
    y_ref, y_A = ref_conv(feats, wl, _pairs(out_nbr), n_out)
    with _Route(fwd_tc, f"{case} forward"):
        y = backend._conv_forward(feats, w, km)
        y32 = backend._conv_forward(feats, w, km, out_dtype=torch.float32)
    assert y.dtype == dtype and y32.dtype == torch.float32
    assert_one_rounding(y, y_ref, y_A, f"{case} forward")
    assert_one_rounding(y32, y_ref, y_A, f"{case} forward, fp32 output")

    gi_ref, gi_A = ref_conv(gout, wl.transpose(1, 2), _pairs(in_nbr), n_in)
    with _Route(dgrad_tc, f"{case} dgrad"):
        gi, _ = backend._conv_backward(feats, gout, w, km, need_in=True, need_w=False)
    assert gi.dtype == dtype
    assert_one_rounding(gi, gi_ref, gi_A, f"{case} dgrad")

    gw_ref, gw_A = ref_wgrad(feats, gout, _pairs(out_nbr))
    with _Route(False, f"{case} wgrad"):
        _, gw = backend._conv_backward(feats, gout, w, km, need_in=False, need_w=True)
        _, gw2 = backend._conv_backward(feats, gout, w, km, need_in=False, need_w=True)
    assert gw.dtype == torch.float32
    assert_one_rounding(gw, gw_ref, gw_A, f"{case} wgrad")
    assert torch.equal(gw, gw2), f"{case} wgrad differs run to run"


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def test_simt_dgrad_with_dense_table_tc_wgrad(ME, cuda, dtype):
    """24 -> 32: the dgrad (24 output columns) is off the grid, the wgrad is not.  The packed
    backward is all-or-nothing, so the layer falls back to meb200_conv_backward: SIMT dgrad and
    `k_wgrad_wg` over the dense table (not the pair lists)."""
    from minkowskiengine_b200 import backend
    cin, cout, n_in, n_out, K = 24, 32, 30_000, 30_000, 27
    feats, gout, w = _inputs(cin, cout, n_in, n_out, K, dtype, cuda, seed=2432)
    wl = w.to(dtype)
    out_nbr = _table(K, n_out, n_in, 0.35, seed=5, device=cuda)
    in_nbr = _table(K, n_in, n_out, 0.35, seed=6, device=cuda)
    km = backend._KernelMap(out_nbr, in_nbr)
    with _Route(False, "24->32 dgrad alone"):
        backend._conv_backward(feats, gout, w, km, need_in=True, need_w=False)
    with _Route(True, "24->32 dgrad + wgrad"):
        gi, gw = backend._conv_backward(feats, gout, w, km, need_in=True, need_w=True)
        _, gw2 = backend._conv_backward(feats, gout, w, km, need_in=True, need_w=True)
    gi_ref, gi_A = ref_conv(gout, wl.transpose(1, 2), _pairs(in_nbr), n_in)
    assert_one_rounding(gi, gi_ref, gi_A, "24->32 dgrad")
    gw_ref, gw_A = ref_wgrad(feats, gout, _pairs(out_nbr))
    assert_one_rounding(gw, gw_ref, gw_A, "24->32 dense-table wgrad")
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
