"""fp8 training (ME.fp8_training): the e5m2 quantisation against its torch expression byte for
byte, the dgrad's e4m3 weight pack against a torch restatement, the e5m2 x e4m3 dgrad (k_conv_wg on
the transposed table) against float64 at every column width it dispatches, over reduction widths,
kernel volumes, tile orders and output dtypes, bit for bit on exactly representable inputs, the
public layers inside the context (forward, input and weight gradients, the route taken), every
fallback bit for bit, and MinkUNet training steps against bf16.

Reference of the dgrad: the float64 convolution of the dequantised operands (the e5m2 gradient times
its scale, the e4m3 weights times their per-input-channel scales) over in_nbr.  Bound (DESIGN.md §3,
"fp8 training"): the chained-accumulation model of the e4m3 forward, n * 2^-13 * A with n = K *
c_out / 32 k-steps and A the same sum over absolute values, plus the epilogue's two fp32 products
(2^-22 of |y| each) and one rounding to the output dtype.  Whether e5m2 x e4m3 accumulates like
e4m3 x e4m3 was not known before these tests: each case prints its worst err / bound."""
import contextlib

import pytest
import torch

from helpers import _pairs, _table, half_ulp, ref_conv

pytestmark = pytest.mark.gpu

FLT_MAX = torch.finfo(torch.float32).max
E5M2_MAX = 57344.0


@pytest.fixture(autouse=True)
def precision():
    saved = torch.backends.cuda.matmul.fp32_precision
    torch.backends.cuda.matmul.fp32_precision = "ieee"
    yield
    torch.backends.cuda.matmul.fp32_precision = saved


def _scales_ref(amax, fmax):
    """(scale, inv) as fp32 scalars by the formula of include/meb200.h (IEEE fp32 divisions)."""
    amax = amax.float().cpu()
    if float(amax) == 0:
        one = torch.tensor(1.0)
        return one, one
    inv = torch.tensor(fmax) / amax
    if bool(torch.isinf(inv)):
        big = torch.tensor(FLT_MAX)
        return torch.tensor(1.0) / big, big
    return amax / fmax, inv


def _finite_amax(x):
    xf = x.float()
    return torch.where(torch.isfinite(xf), xf.abs(), torch.zeros_like(xf)).max() if xf.numel() \
        else torch.zeros((), device=x.device)


def _e5m2_ref(x):
    """(e5m2 bytes, scale, inv) of x by the pinned torch expression (the clamp stands for
    satfinite: torch rounds values past 57344 to inf; it keeps NaN)."""
    scale, inv = _scales_ref(_finite_amax(x), E5M2_MAX)
    q = (x.float() * inv.to(x.device)).clamp(-E5M2_MAX, E5M2_MAX).to(torch.float8_e5m2)
    return q.view(torch.uint8), scale, inv


def _nan_e5m2(b):
    return ((b & 0x7C) == 0x7C) & ((b & 0x03) != 0)     # exponent all ones, mantissa not zero


def _nan_e4m3(b):
    return (b & 0x7F) == 0x7F


def _same_bytes(got, want, what, is_nan):
    """Equal bytes, NaN compared as NaN (its encoding may differ)."""
    nan_w, nan_g = is_nan(want), is_nan(got)
    assert torch.equal(nan_w, nan_g), f"{what}: NaN positions differ"
    assert torch.equal(got[~nan_w], want[~nan_w]), \
        f"{what}: {int((got != want)[~nan_w].sum())} bytes differ"


def _inputs(kind, shape, dtype, device, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(shape, generator=g) * 3
    if kind == "zero":
        x.zero_()
    elif kind == "special":
        flat = x.view(-1)
        idx = torch.randperm(flat.numel(), generator=g)[:40]
        flat[idx[:10]] = float("nan")
        flat[idx[10:20]] = float("inf")
        flat[idx[20:30]] = float("-inf")
        flat[idx[30:]] = 0.0
    elif kind == "big":                      # finite values past 57344 set the amax
        x = x * 3e4
    elif kind == "tiny":
        x = x * 1e-38                        # 57344 / amax overflows: inv is FLT_MAX
    return x.to(dtype).to(device)


# ---- 1. e5m2 quantisation -------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["random", "zero", "special", "big", "tiny"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16],
                         ids=["fp32", "bf16", "fp16"])
@pytest.mark.parametrize("n,c,offset", [(5000, 64, 0), (777, 32, 0), (3, 5, 0), (1000, 64, 1)],
                         ids=["5000x64", "777x32", "3x5", "1000x64_misaligned"])
def test_quantize_e5m2_bytes(ME, cuda, kind, dtype, n, c, offset):
    from minkowskiengine_b200 import backend
    if kind == "tiny" and dtype == torch.float16:
        pytest.skip("fp16 has no values this small")
    if kind == "big" and dtype == torch.float16:
        pytest.skip("fp16 overflows past 65504")
    x = _inputs(kind, (n * c + offset,), dtype, cuda, seed=n + c + 1)[offset:].view(n, c)
    q, scale = backend._quantize_dynamic(x, "meb200_quantize_e5m2")
    want_q, want_scale, want_inv = _e5m2_ref(x)
    _same_bytes(q, want_q, f"{kind} {dtype}", _nan_e5m2)
    assert scale.cpu().tolist() == [want_scale.item(), want_inv.item()]
    if kind == "special":                    # +-inf saturates to +-57344
        xf = x.float()
        sat = q.view(torch.float8_e5m2).float()
        assert bool((sat[torch.isposinf(xf)] == E5M2_MAX).all())
        assert bool((sat[torch.isneginf(xf)] == -E5M2_MAX).all())
        assert bool(torch.isnan(sat[torch.isnan(xf)]).all())
    q2, scale2 = backend._quantize_dynamic(x, "meb200_quantize_e5m2")
    assert torch.equal(q, q2) and torch.equal(scale, scale2)
    # the shared workspace is left zero: the e4m3 quantiser after it is unchanged
    qe, se = backend._quantize_e4m3(x)
    q3, s3 = backend._quantize_dynamic(x, "meb200_quantize_e5m2")
    assert torch.equal(q3, q) and torch.equal(s3, scale)
    assert float(se[1]) == float(_scales_ref(_finite_amax(x), 448.0)[1])


# ---- 2. the dgrad's weight pack -------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["random", "special"])
@pytest.mark.parametrize("K,c_in,c_out", [(27, 64, 96), (8, 32, 16), (1, 384, 256), (3, 5, 7),
                                          (125, 32, 300)])
def test_dgrad_pack_bytes(ME, cuda, kind, K, c_in, c_out):
    from minkowskiengine_b200 import backend
    w = _inputs(kind, (K, c_in, c_out), torch.float32, cuda, seed=K * c_in + c_out)
    w[:, 0, :] = 0.0                                   # a zero input channel: scale 1
    w_c, w_scale = backend._fp8_dgrad_weights(w)
    wf = w.transpose(0, 1).reshape(c_in, K * c_out)
    amax = torch.where(torch.isfinite(wf), wf.abs(), torch.zeros_like(wf)).max(1).values.cpu()
    scales = [_scales_ref(a, 448.0) for a in amax]
    want_scale = torch.stack([s for s, _ in scales])
    inv = torch.stack([i for _, i in scales]).to(cuda)
    want = (w * inv[None, :, None]).clamp(-448, 448).to(torch.float8_e4m3fn).view(torch.uint8)
    _same_bytes(w_c, want, f"dgrad weights {kind}", _nan_e4m3)
    assert torch.equal(w_scale.cpu(), want_scale)
    assert w_c.shape == (K, c_in, c_out)


# ---- 3. the dgrad against float64 -----------------------------------------------------------------
def _deq(gout, w):
    """float64 dequantised operands: the gradient [n_out, c_out], the weights [K, c_in, c_out]."""
    from minkowskiengine_b200 import backend
    q, s = backend._quantize_dynamic(gout.contiguous(), "meb200_quantize_e5m2")
    w_c, w_scale = backend._fp8_dgrad_weights(w)
    gd = q.view(torch.float8_e5m2).double() * s[0].double()
    wd = w_c.view(torch.float8_e4m3fn).double() * w_scale.double()[None, :, None]
    return gd, wd


def _expected(gd, wd, in_nbr, n_in, steps, out_dtype):
    ref, A = ref_conv(gd, wd.transpose(1, 2), _pairs(in_nbr), n_in)
    delta = A * (steps * 2.0 ** -13) + 2.0 ** -21 * ref.abs()
    if out_dtype != torch.float32:
        delta = half_ulp(ref.abs() + delta, out_dtype) + delta
    return ref, delta


def _check(y, y_ref, bound, what):
    err = (y.double() - y_ref).abs()
    bad = ~(err <= bound)
    ratio = float((err / bound.clamp(min=1e-300)).max())
    if bool(bad.any()):
        j = int(torch.nonzero(bad.flatten())[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements outside the "
                             f"bound (worst err / bound {ratio:.2f}); first at flat index {j}: got "
                             f"{y.flatten()[j].item()!r}, float64 {y_ref.flatten()[j].item()!r}")
    return ratio


def _dmap(K, n_out, n_in, seed, device):
    """A map whose dgrad table in_nbr [K, n_in] is random (rows and an offset without neighbours)."""
    from minkowskiengine_b200 import backend
    in_nbr = _table(K, n_in, n_out, 0.35, seed, device)
    assert bool((in_nbr < 0).all(0).any())
    return backend._KernelMap(torch.full((K, n_out), -1, dtype=torch.int32, device=device), in_nbr)


def _grad(n, c, dtype, device, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(n, c, generator=g) * 1e-3).to(dtype).to(device)


def _weights(K, cin, cout, device, seed):
    g = torch.Generator().manual_seed(seed)
    return ((torch.rand(K, cin, cout, generator=g) - 0.5) / cin ** 0.5).to(device)


def _run(case, gout, w, km, dtype):
    from minkowskiengine_b200 import _lib, backend
    n0 = _lib.tc_launch_count()
    y = backend._conv_dgrad_fp8(gout, w, km, dtype)
    y2 = backend._conv_dgrad_fp8(gout, w, km, dtype)
    assert _lib.tc_launch_count() > n0, f"{case}: no tensor-core launch"
    assert y.dtype == dtype and torch.equal(y, y2), f"{case}: differs run to run"
    gd, wd = _deq(gout, w)
    y_ref, bound = _expected(gd, wd, km.in_nbr, km.n_in, km.K * gout.shape[1] // 32, dtype)
    ratio = _check(y, y_ref, bound, case)
    print(f"{case}: worst err / bound {ratio:.4f}")
    empty = (km.in_nbr < 0).all(0)          # (every row of a stride-1 map has its centre)
    assert not y[empty].any(), f"{case}: rows without neighbours"
    return ratio


DTYPES = [torch.float32, torch.bfloat16, torch.float16]
DT_IDS = ["fp32", "bf16", "fp16"]
# every (NI, NT) of MEB_COLS_DISPATCH (c_in = 16 i), and two widths past one launch
COLS = [16 * i for i in range(1, 17)] + [272, 512]


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("cin", COLS)
def test_dgrad_columns_against_float64(ME, cuda, dtype, cin):
    K, cout, n = 8, 32, 2000
    _run(f"dgrad {dtype} {cout}->{cin} K={K}", _grad(n, cout, dtype, cuda, cin),
         _weights(K, cin, cout, cuda, cin + 1), _dmap(K, n, n, cin + 2, cuda), dtype)


@pytest.mark.parametrize("K", [1, 8, 27, 125])
@pytest.mark.parametrize("cout", [32, 96, 128, 384])
def test_dgrad_reductions_against_float64(ME, cuda, K, cout):
    """32-byte (c_out 32, 96), 128-byte (128) and multi-stage (384) rows of the reduction."""
    n = 3000 if K <= 27 else 1200
    dtype = torch.bfloat16
    _run(f"dgrad bf16 {cout}->64 K={K}", _grad(n, cout, dtype, cuda, K + cout),
         _weights(K, 64, cout, cuda, K * cout), _dmap(K, n, n, K + 3 * cout, cuda), dtype)


def _cloud(ME, n, c, dtype, device, seed):
    from oracle import oracle_np as O
    coords = O.surface_cloud(n, seed=seed)
    feats = (torch.rand(len(coords), c, generator=torch.Generator().manual_seed(seed)) - 0.5) * 4
    return ME.SparseTensor(feats.to(dtype).to(device), coords.to(device))


def _real_map(ME, x, stride=1):
    key = x.coordinate_map_key
    mgr = x.coordinate_manager._manager
    if stride == 1:
        return mgr._kernel_map(key, key, [3] * 3, [1] * 3, [1] * 3, ME.RegionType.HYPER_CUBE,
                               None, False, False)
    from minkowskiengine_b200 import backend
    out_key = ME.CoordinateMapKey(4)
    backend._set_strided_key(mgr, key, out_key, [2] * 3)
    return mgr._kernel_map(key, out_key, [2] * 3, [2] * 3, [1] * 3, ME.RegionType.HYPER_CUBE,
                           None, False, False)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("cout", [64, 384])
def test_dgrad_tile_order_against_float64(ME, cuda, dtype, cout):
    """A real kernel map carries the dgrad's tile order (in_order): with it and without it."""
    from minkowskiengine_b200 import backend
    x = _cloud(ME, 20_000, 4, torch.float32, cuda, seed=11)
    km = _real_map(ME, x)
    assert km.in_order is not None
    plain = backend._KernelMap(km.out_nbr, km.in_nbr)
    gout = _grad(km.n_out, cout, dtype, cuda, 5)
    w = _weights(27, 96, cout, cuda, 12)
    ys = [_run(f"dgrad {what} {dtype} {cout}->96", gout, w, m, dtype)
          for m, what in ((km, "ordered"), (plain, "unordered"))]
    assert all(r <= 1 for r in ys)


# ---- 4. exact inputs ------------------------------------------------------------------------------
EXACT = [("table", 8, 64, 16), ("table", 8, 32, 96), ("table", 8, 64, 272), ("table", 27, 96, 64),
         ("table", 27, 384, 128), ("ordered", 27, 96, 64), ("ordered", 27, 384, 32)]


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("kind,K,cout,cin", EXACT,
                         ids=[f"{c[0]}_K{c[1]}_{c[2]}to{c[3]}" for c in EXACT])
def test_exact_inputs_equal_float64(ME, cuda, dtype, kind, K, cout, cin):
    """Gradients and weights in {-1, 0, 1} plus one 7 in the gradient and a 7 in every weight row,
    so every amax is 7 = 1.75 * 2^2: the e5m2 scale is 2^-13, the e4m3 ones 2^-6, and every value is
    exact in its format.  The 7s multiply only zeros (gradient channel 0 meets zero weights, weight
    column 1 zero gradients), so each partial sum is a small integer.  The dgrad is float64's,
    rounded once to the output dtype."""
    from minkowskiengine_b200 import backend
    g = torch.Generator().manual_seed(K * cin + cout)
    if kind == "table":
        n = 2000
        maps = [_dmap(K, n, n, cout, cuda)]
    else:
        x = _cloud(ME, 20_000, 4, torch.float32, cuda, seed=cin)
        km = _real_map(ME, x)
        assert km.in_order is not None
        n = km.n_out
        maps = [km, backend._KernelMap(km.out_nbr, km.in_nbr)]
    gout = torch.randint(-1, 2, (n, cout), generator=g).float()
    gout[:, :2] = 0
    gout[n // 2, 0] = 7
    w = torch.randint(-1, 2, (K, cin, cout), generator=g).float()
    w[:, :, 0] = 0
    w[K // 3, :, 1] = 7
    gout, w = gout.to(dtype).to(cuda), w.to(cuda)
    _, s = backend._quantize_dynamic(gout, "meb200_quantize_e5m2")
    _, w_scale = backend._fp8_dgrad_weights(w)
    assert float(s[0]) == 2.0 ** -13 and bool((w_scale == 2.0 ** -6).all())
    for m in maps:
        ref, _ = ref_conv(gout, w.transpose(1, 2), _pairs(m.in_nbr), m.n_in)
        y = backend._conv_dgrad_fp8(gout, w, m, dtype)
        assert torch.equal(y, ref.to(dtype)), \
            f"{kind} {dtype} K={K} {cout}->{cin} ordered={m.in_order is not None}"


# ---- 5. the public layers -------------------------------------------------------------------------
class _Routes:
    """Counts the e4m3 forwards and fp8 dgrads run inside fp8_training(), and keeps the dgrads'
    arguments and results."""

    def __init__(self):
        self.fwd, self.dgrad = 0, []

    def __enter__(self):
        import minkowskiengine_b200 as ME
        from minkowskiengine_b200 import backend
        self._f, self._d = backend._conv_forward_fp8, backend._conv_dgrad_fp8

        def f(*a, **k):
            self.fwd += 1
            return self._f(*a, **k)

        def d(*a, **k):
            out = self._d(*a, **k)
            self.dgrad.append((a, out))
            return out
        backend._conv_forward_fp8, backend._conv_dgrad_fp8 = f, d
        self._ctx = ME.fp8_training()
        self._ctx.__enter__()
        return self

    def __exit__(self, *exc):
        from minkowskiengine_b200 import backend
        self._ctx.__exit__(*exc)
        backend._conv_forward_fp8, backend._conv_dgrad_fp8 = self._f, self._d
        return False


def _layer(ME, name, C, device):
    torch.manual_seed(1)
    cls = {"conv": ME.MinkowskiConvolution, "conv_bias": ME.MinkowskiConvolution,
           "transpose": ME.MinkowskiConvolutionTranspose,
           "generative": ME.MinkowskiGenerativeConvolutionTranspose}[name]
    conv_like = name.startswith("conv")
    return cls(C, C, kernel_size=3 if conv_like else 2, stride=1 if conv_like else 2,
               bias=name == "conv_bias", dimension=3).to(device)


def _fwd_bwd(layer, x, gout):
    """(output, input gradient, kernel gradient, bias gradient) of layer(x) against gout."""
    xf = x.F.detach().clone().requires_grad_(True)
    layer.zero_grad(set_to_none=True)
    y = layer(x.__class__(xf, coordinate_map_key=x.coordinate_map_key,
                          coordinate_manager=x.coordinate_manager))
    y.F.backward(gout(y))
    return (y, xf.grad, layer.kernel.grad.clone(),
            None if layer.bias is None else layer.bias.grad.clone())


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("name", ["conv", "conv_bias", "transpose", "generative"])
def test_public_layers(ME, cuda, name, dtype):
    C = 64
    x = _cloud(ME, 8000, C, dtype, cuda, seed=3)
    if name in ("transpose", "generative"):
        down = ME.MinkowskiConvolution(C, C, kernel_size=2, stride=2, dimension=3).to(cuda)
        with torch.no_grad():
            x = down(x)
    layer = _layer(ME, name, C, cuda)
    gen = torch.Generator(device=cuda).manual_seed(7)
    cache = {}

    def gout(y):                         # the same dOut inside and outside the block
        if "g" not in cache:
            cache["g"] = (torch.randn(y.F.shape, generator=gen, device=cuda) * 1e-2).to(dtype)
        return cache["g"]

    want = _fwd_bwd(layer, x, gout)
    with _Routes() as r:
        got = _fwd_bwd(layer, x, gout)
    assert r.fwd == 1 and len(r.dgrad) == 1
    y, gi, gw, gb = got
    # forward: a bias-free layer gives the bits of fp8_inference() on the same input and weights
    if layer.bias is None:
        with torch.no_grad(), ME.fp8_inference():
            assert torch.equal(y.F, layer(x).F)
    rel = float((y.F.double() - want[0].F.double()).norm() / want[0].F.double().norm())
    assert rel < 0.1, rel
    if name != "generative":
        assert y.coordinate_map_key == want[0].coordinate_map_key
    # input gradient: within the bound of item 3, on the layer's own dgrad arguments
    (gout_d, kernel, km, dt), out = r.dgrad[0]
    assert torch.equal(out, gi) and dt == dtype
    gd, wd = _deq(gout_d, kernel)
    y_ref, bound = _expected(gd, wd, km.in_nbr, km.n_in, km.K * C // 32, dtype)
    print(f"layer {name} {dtype}: dgrad worst err / bound {_check(gi, y_ref, bound, name):.4f}")
    # weight (and bias) gradient: the bits of the same layer outside the block
    assert torch.equal(gw, want[2]), f"{name}: weight gradient"
    if gb is not None:
        assert torch.equal(gb, want[3])


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_empty_maps(ME, cuda, dtype):
    """An empty output map: the input gradient is zero, and no dgrad launches.  An empty input
    map: the forward's output rows have no neighbours (zero), the input gradient has no rows."""
    from minkowskiengine_b200 import _lib, backend
    K, cin, cout = 27, 64, 32
    w = _weights(K, cin, cout, cuda, 1)
    none = lambda *s: torch.full(s, -1, dtype=torch.int32, device=cuda)     # noqa: E731
    km = backend._KernelMap(none(K, 0), none(K, 50))                      # no output rows
    n0 = _lib.tc_launch_count()
    gi = backend._conv_dgrad_fp8(torch.zeros(0, cout, dtype=dtype, device=cuda), w, km, dtype)
    assert gi.shape == (50, cin) and gi.dtype == dtype and not gi.any()
    assert _lib.tc_launch_count() == n0
    km = backend._KernelMap(none(K, 40), none(K, 0))                      # no input rows
    gi = backend._conv_dgrad_fp8(_grad(40, cout, dtype, cuda, 2), w, km, dtype)
    assert gi.shape == (0, cin)
    y = backend._conv_forward(torch.zeros(0, cin, dtype=dtype, device=cuda), w, km, fp8=True)
    assert y.shape == (40, cout) and not y.any()


# ---- 6. fallbacks ----------------------------------------------------------------------------------
def _same_training(ME, fn, params):
    """fn() forward and backward outside and inside fp8_training(): the same bits, no fp8 route."""
    def run():
        for p in params:
            p.grad = None
        x, y = fn()
        if y.F.requires_grad:
            y.F.float().square().sum().backward()
        return [y.F] + [t.grad for t in [x] + params if t is not None and t.grad is not None]
    want = run()
    with _Routes() as r:
        got = run()
    assert r.fwd == 0 and not r.dgrad
    assert len(got) == len(want) and all(torch.equal(a, b) for a, b in zip(got, want))


def test_fallbacks_are_bit_identical(ME, cuda):
    torch.manual_seed(2)
    C = 32

    def leaf(c, seed, n=4000):
        x = _cloud(ME, n, c, torch.bfloat16, cuda, seed)
        xf = x.F.detach().clone().requires_grad_(True)
        return xf, ME.SparseTensor(xf, coordinate_map_key=x.coordinate_map_key,
                                   coordinate_manager=x.coordinate_manager)

    cases = {
        "c_in 48": (ME.MinkowskiConvolution(48, 64, kernel_size=3, dimension=3), 48),
        "c_out 40": (ME.MinkowskiConvolution(C, 40, kernel_size=3, dimension=3), C),
        "c_out 16 (dgrad off the grid)": (ME.MinkowskiConvolution(C, 16, kernel_size=3, dimension=3), C),
        "stem": (ME.MinkowskiConvolution(3, 32, kernel_size=5, dimension=3), 3),
        "use_mm": (ME.MinkowskiConvolution(C, 64, kernel_size=1, dimension=3), C),
        "channelwise": (ME.MinkowskiChannelwiseConvolution(C, kernel_size=3, dimension=3), C),
        "pooling": (ME.MinkowskiMaxPooling(kernel_size=2, stride=2, dimension=3), C),
        "batch norm": (ME.MinkowskiBatchNorm(C), C),
    }
    for i, (name, (mod, c)) in enumerate(cases.items()):
        mod = mod.to(cuda)
        params = list(mod.parameters())

        def fn(mod=mod, c=c, i=i):
            xf, x = leaf(c, 5 + i)
            return xf, mod(x)
        _same_training(ME, fn, params)
    # no gradient needed: grad mode off, or nothing requires one
    conv = ME.MinkowskiConvolution(C, 64, kernel_size=3, dimension=3).to(cuda)
    with torch.no_grad():
        _same_training(ME, lambda: (None, conv(leaf(C, 20)[1])), [])
    for p in conv.parameters():
        p.requires_grad_(False)
    x = _cloud(ME, 4000, C, torch.bfloat16, cuda, 21)
    _same_training(ME, lambda: (None, conv(x)), [])


# ---- 7. MinkUNet34C training steps ----------------------------------------------------------------
class _LayerAudit:
    """Inside the fp8 step, checks every selected layer on its own inputs as it runs: the e4m3
    forward and the e5m2 dgrad against float64 of their dequantised operands within the bounds of
    items 3 and 5, and the weight gradient against the same call outside fp8, bit for bit."""

    def __init__(self):
        self.fwd, self.dgrad, self.wgrad = [], [], 0

    def __enter__(self):
        from minkowskiengine_b200 import backend
        self._f, self._b = backend._conv_forward_fp8, backend._conv_backward_impl
        backend._conv_forward_fp8, backend._conv_backward_impl = self._forward, self._backward
        return self

    def __exit__(self, *exc):
        from minkowskiengine_b200 import backend
        backend._conv_forward_fp8, backend._conv_backward_impl = self._f, self._b
        return False

    def _forward(self, in_feat, kernel, km, epilogue, act=None, shadow=None):
        from minkowskiengine_b200 import backend
        assert epilogue is None and act is None and shadow is None
        y = self._f(in_feat, kernel, km, epilogue, act, shadow)
        q, a = backend._quantize_e4m3(in_feat)               # the bytes the forward multiplied
        w_t, w_scale = backend._fp8_weights(kernel)
        xd = q.view(torch.float8_e4m3fn).double() * a[0].double()
        wd = w_t.view(torch.float8_e4m3fn).double().transpose(1, 2) * w_scale.double()
        ref, A = ref_conv(xd, wd, _pairs(km.out_nbr), km.n_out)
        bound = A * (km.K * in_feat.shape[1] // 32 * 2.0 ** -13) + 2.0 ** -21 * ref.abs()
        if y.dtype != torch.float32:
            bound = half_ulp(ref.abs() + bound, y.dtype) + bound
        self.fwd.append(_check(y, ref, bound, f"forward {tuple(kernel.shape)}"))
        return y

    def _backward(self, in_feat, grad_out, kernel, km, need_in=True, need_w=True, fp8=False):
        gi, gw = self._b(in_feat, grad_out, kernel, km, need_in, need_w, fp8)
        if not fp8:
            return gi, gw
        if need_in:
            g = grad_out.to(in_feat.dtype).contiguous()
            gd, wd = _deq(g, kernel)
            y_ref, bound = _expected(gd, wd, km.in_nbr, km.n_in, km.K * g.shape[1] // 32, gi.dtype)
            self.dgrad.append(_check(gi, y_ref, bound, f"dgrad {tuple(kernel.shape)}"))
        if need_w:
            _, want = self._b(in_feat, grad_out, kernel, km, False, True, False)
            assert torch.equal(gw, want), f"wgrad {tuple(kernel.shape)}"
            self.wgrad += 1
        return gi, gw


def _steps(ME, net, coords, feats, labels, fp8, steps=2, grads_of=(), audit=None):
    opt = torch.optim.SGD(net.parameters(), lr=1e-2)
    crit = torch.nn.CrossEntropyLoss()
    losses, grads = [], {}
    names = dict(net.named_parameters())
    for s in range(steps):
        opt.zero_grad(set_to_none=True)
        with contextlib.ExitStack() as stack:
            if fp8:
                stack.enter_context(ME.fp8_training())
            if audit is not None:
                stack.enter_context(audit)
            out = net(ME.SparseTensor(feats, coords))
            loss = crit(out.F.float(), labels)
            loss.backward()
        losses.append(loss.detach().double())
        for n, p in names.items():
            assert p.grad is None or bool(torch.isfinite(p.grad).all()), f"step {s} {n}"
        if s == 0:
            grads = {n: names[n].grad.detach().double().clone() for n in grads_of}
        opt.step()
    return torch.stack(losses), grads


# Step-0 weight-gradient cosines against the exact fp32 step, for the stem, a middle layer
# (block4.2.conv1) and the final layer.  Measured on an H100 80GB HBM3 (700 W): bf16 0.966, 0.809,
# 0.99997; fp8 0.852, 0.160, 0.99925.  Every selected layer passes its own audit, so the middle
# layer's loss is the e5m2 noise of a gradient whose terms mostly cancel (bf16 already loses a
# fifth of it there): DESIGN.md §3, "fp8 training".
COS_MIN = (0.75, 0.05, 0.995)


def _cos(a, b):
    return float(torch.nn.functional.cosine_similarity(a.flatten(), b.flatten(), 0))


def test_minkunet34c_steps(ME, cuda):
    """Two SGD steps of bench.py's cfg3 network (MinkUNet34C, bf16) on its clouds, inside and
    outside fp8_training(), from the same state; every selected layer of the first fp8 run is
    audited on its own inputs.  The weight gradients are also compared with the exact fp32 step's,
    which separates what bf16 already loses from what fp8 adds.  Limits: DESIGN.md §3."""
    from examples.minkunet import minkunet
    from examples.synthetic import surface_cloud
    # bench.py's batch (make_batch): 8 surface clouds of 100k voxels, features U(0, 1), labels 0
    coords = torch.cat([surface_cloud(100_000, j, batch=j) for j in range(8)], 0)
    feats = torch.rand(len(coords), 3, generator=torch.Generator().manual_seed(0))
    labels = torch.zeros(len(coords), dtype=torch.int64)
    coords, feats, labels = coords.to(cuda), feats.to(cuda), labels.to(cuda)
    torch.manual_seed(0)
    net = minkunet("MinkUNet34C", ME, 3, 20, 3).to(cuda)
    state = {k: v.clone() for k, v in net.state_dict().items()}
    names = [n for n, p in net.named_parameters() if p.dim() == 3]
    picks = [names[0], names[len(names) // 2], names[-1]]
    l32, g32 = _steps(ME, net, coords, feats, labels, False, grads_of=picks, steps=1)
    net.load_state_dict(state)
    base, gb = _steps(ME, net, coords, feats.bfloat16(), labels, False, grads_of=picks)
    runs, audit = [], _LayerAudit()
    for i in range(2):
        net.load_state_dict(state)
        runs.append(_steps(ME, net, coords, feats.bfloat16(), labels, True, grads_of=picks,
                           audit=audit if i == 0 else None))
    (l8, g8), (l8b, g8b) = runs
    assert torch.equal(l8, l8b) and all(torch.equal(g8[n], g8b[n]) for n in picks)
    assert bool(torch.isfinite(l8).all())
    # 2 steps x (46 K = 27 and 8 K = 8 selected layers): the stem's input needs no gradient and
    # its c_in is off the grid; the final layer is a K = 1 matrix product
    assert len(audit.fwd) == len(audit.dgrad) == audit.wgrad == 2 * 54, \
        (len(audit.fwd), len(audit.dgrad), audit.wgrad)
    rel = float((l8[0] - base[0]).abs() / base[0].abs())
    cos = {n: (_cos(gb[n], g32[n]), _cos(g8[n], g32[n]), _cos(g8[n], gb[n])) for n in picks}
    print(f"MinkUNet34C step-0 loss fp32 {float(l32[0]):.6f} bf16 {float(base[0]):.6f} fp8 "
          f"{float(l8[0]):.6f} (rel to bf16 {rel:.2e}); step 1 bf16 {float(base[1]):.6f} fp8 "
          f"{float(l8[1]):.6f}; audit worst err / bound forward {max(audit.fwd):.4f} dgrad "
          f"{max(audit.dgrad):.4f}; weight-gradient cosines (bf16 vs fp32, fp8 vs fp32, fp8 vs "
          f"bf16) {cos}")
    assert rel < 2e-3, rel                     # measured 2.46e-4 (4.533210 against 4.532097)
    assert max(audit.fwd) <= 1 and max(audit.dgrad) <= 1      # measured 0.80 and 0.86
    for n, (c_b, c_8, _) in cos.items():
        assert c_8 > COS_MIN[picks.index(n)], (n, c_b, c_8)


# ---- 8. a short training run ----------------------------------------------------------------------
def test_minkunet14_fits_a_batch(ME, cuda):
    """MinkUNet14 fits one small fixed batch for 40 SGD steps in bf16 and in fp8: the fp8 loss
    decreases and ends near bf16's."""
    from examples.minkunet import minkunet
    from examples.synthetic import surface_cloud
    coords = torch.cat([surface_cloud(20_000, 50 + j, batch=j) for j in range(2)], 0).to(cuda)
    g = torch.Generator().manual_seed(3)
    feats = torch.rand(len(coords), 3, generator=g).to(cuda).bfloat16()
    labels = (coords[:, 1] // 8 % 4 + 4 * (feats[:, 0].float() > 0.5).long()).to(cuda)
    finals = {}
    for fp8 in (False, True):
        torch.manual_seed(0)
        net = minkunet("MinkUNet14", ME, 3, 8, 3).to(cuda)
        losses, _ = _steps(ME, net, coords, feats, labels, fp8, steps=40)
        finals[fp8] = losses
        print(f"MinkUNet14 {'fp8' if fp8 else 'bf16'} loss: " +
              " ".join(f"{float(v):.4f}" for v in losses[::5]) + f" ... {float(losses[-1]):.4f}")
    l8, lb = finals[True], finals[False]
    assert bool(torch.isfinite(l8).all())
    # measured on an H100 80GB HBM3 (700 W): bf16 2.744 -> 1.884, fp8 2.744 -> 1.917 (1.8 % above)
    assert float(l8[-5:].mean()) < 0.8 * float(l8[:5].mean())
    assert float(l8[-1]) < float(lb[-1]) * 1.1 + 0.02
