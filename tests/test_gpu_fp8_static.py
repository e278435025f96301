"""Static fp8 scales and shadows (ME.Fp8Calibration, ME.fp8_inference(calibration)) on the GPU: the
amax accumulation, the scales and the static conversion against their torch expressions byte for
byte; the shadow every k_conv_wg_q family writes against the static conversion of the output it
stored, byte for byte; a consumer reading a shadow against the same consumer converting its input;
links through real modules; batch invariance of a calibrated layer; and MinkUNet34C against the
exact fp32 network."""
import pytest
import torch

from helpers import _table
from test_gpu_fp8 import (_cloud, _epilogue, _feats, _inputs, _minkunet, _norm, _quant_ref,
                          _same_bytes, _scales_ref, _weights)

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def precision():
    saved = torch.backends.cuda.matmul.fp32_precision
    torch.backends.cuda.matmul.fp32_precision = "ieee"
    yield
    torch.backends.cuda.matmul.fp32_precision = saved


def _static_ref(x, scale_dev):
    """e4m3 bytes of x at a given (scale, inv), by the torch expression of DESIGN.md §3."""
    inv = scale_dev[1].float()
    return (x.float() * inv).clamp(-448, 448).to(torch.float8_e4m3fn).view(torch.uint8)


def _bits(t):
    return t.float().view(torch.int32)


# ---- the static-scale kernels -------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["random", "zero", "special", "tiny"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16],
                         ids=["fp32", "bf16", "fp16"])
@pytest.mark.parametrize("n,c,offset", [(5000, 64, 0), (777, 32, 0), (3, 5, 0), (1000, 64, 1)],
                         ids=["5000x64", "777x32", "3x5", "1000x64_misaligned"])
def test_amax_scales_and_static_conversion(ME, cuda, kind, dtype, n, c, offset):
    from minkowskiengine_b200 import backend
    amax = torch.zeros(1, dtype=torch.float32, device=cuda)
    xs = []
    for b in range(3):                      # three batches into one running amax
        buf = _inputs(kind, (n * c + offset,), dtype, cuda, seed=n + c + b)
        x = buf[offset:].view(n, c)
        if kind == "random":
            x = x * (b + 1)
        backend.amax_accumulate(x, amax)
        xs.append(x)
    allx = torch.cat([x.float().flatten() for x in xs])
    fin = allx[torch.isfinite(allx)]
    want = fin.abs().max() if fin.numel() else torch.zeros((), device=cuda)
    assert torch.equal(_bits(amax[0]), _bits(want)), f"amax {float(amax[0])} != {float(want)}"
    scale = backend.e4m3_scales(amax)
    s_ref, inv_ref = _scales_ref(want)
    assert torch.equal(_bits(scale.cpu()), _bits(torch.stack([s_ref, inv_ref]))), "scales"
    for x in xs:
        q = backend.quantize_e4m3_static(x, scale)
        _same_bytes(q, _static_ref(x, scale), f"{kind} {dtype} {n}x{c}+{offset}")
    # the static scale of one tensor is the dynamic scale: the same bytes as meb200_quantize_e4m3
    one = torch.zeros(1, dtype=torch.float32, device=cuda)
    backend.amax_accumulate(xs[0], one)
    q_dyn, s_dyn = backend._quantize_e4m3(xs[0])
    q_st = backend.quantize_e4m3_static(xs[0], backend.e4m3_scales(one))
    assert torch.equal(q_dyn, q_st)
    assert torch.equal(_quant_ref(xs[0])[0][~((q_dyn & 0x7F) == 0x7F)], q_st[~((q_dyn & 0x7F) == 0x7F)])


def test_static_scale_saturates_above_the_calibrated_amax(ME, cuda):
    from minkowskiengine_b200 import backend
    amax = torch.full((1,), 2.0, device=cuda)
    x = torch.tensor([[-10.0, -2.0, 1.0, 2.0, 3.0, float("inf"), float("-inf"), 0.0]], device=cuda)
    q = backend.quantize_e4m3_static(x, backend.e4m3_scales(amax))
    deq = q.view(torch.float8_e4m3fn).float() * (2.0 / 448)
    assert deq.tolist()[0] == [-2.0, -2.0, 1.0, 2.0, 2.0, 2.0, -2.0, 0.0]


# ---- shadows --------------------------------------------------------------------------------------
def _km(K, n_out, n_in, seed, device):
    from minkowskiengine_b200 import backend
    return backend._KernelMap(_table(K, n_out, n_in, 0.35, seed, device),
                              torch.full((K, n_in), -1, dtype=torch.int32, device=device))


def _shadow_scale(y, frac=0.5):
    """A static scale whose amax is a fraction of the output's: some values saturate."""
    from minkowskiengine_b200 import backend
    amax = (y.float().abs().max() * frac).reshape(1).contiguous()
    return backend.e4m3_scales(amax)


def _check_shadow(case, feats, w, km, epi, fp8, out_dtype=None):
    """The forward with a shadow stores the same output as without, and the shadow is the static
    conversion of the stored output, byte for byte."""
    from minkowskiengine_b200 import backend
    want = backend._conv_forward(feats, w, km, out_dtype=out_dtype, epilogue=epi, fp8=fp8)
    scale = _shadow_scale(want)
    out, q = backend._conv_forward(feats, w, km, out_dtype=out_dtype, epilogue=epi, fp8=fp8,
                                   shadow=scale)
    assert q is not None, f"{case}: no shadow"
    assert torch.equal(out, want), f"{case}: the output changed"
    _same_bytes(q, backend.quantize_e4m3_static(out, scale), f"{case}: shadow")
    _same_bytes(q, _static_ref(out, scale), f"{case}: shadow vs torch")
    empty = (km.out_nbr < 0).all(0)
    assert bool(empty.any()), f"{case}: the table has rows without neighbours"


# every (NI, NT) of MEB_COLS_DISPATCH, two launches of column blocks (272, 512)
COLS = [16 * i for i in range(1, 17)] + [272, 512]


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16],
                         ids=["fp32", "bf16", "fp16"])
@pytest.mark.parametrize("cout", COLS)
def test_shadow_e4m3_operands(ME, cuda, dtype, cout):
    """e4m3 operands; the output in the feature dtype (fp32 features: an fp32 output)."""
    feats = _feats(2000, 32, dtype, cuda, cout)
    w = _weights(8, 32, cout, cuda, cout + 1)
    km = _km(8, 2000, 2000, cout + 2, cuda)
    epi = _epilogue(cout, 2000, dtype, cuda, cout + 3, with_res=True, relu=True)
    _check_shadow(f"e4m3 {dtype} ->{cout}", feats, w, km, epi, fp8=True)


@pytest.mark.parametrize("out_dtype", [None, torch.float32], ids=["same", "fp32"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("cout", COLS)
def test_shadow_16_bit_operands(ME, cuda, dtype, cout, out_dtype):
    feats = _feats(2000, 32, dtype, cuda, cout)
    w = _weights(8, 32, cout, cuda, cout + 1)
    km = _km(8, 2000, 2000, cout + 2, cuda)
    epi = _epilogue(cout, 2000, out_dtype or dtype, cuda, cout + 3, with_res=True, relu=True)
    _check_shadow(f"{dtype} ->{cout} out {out_dtype}", feats, w, km, epi, fp8=False,
                  out_dtype=out_dtype)


@pytest.mark.parametrize("with_res,relu", [(False, False), (False, True), (True, False)],
                         ids=["affine", "relu", "residual"])
@pytest.mark.parametrize("fp8", [True, False], ids=["e4m3", "bf16"])
def test_shadow_epilogue_variants(ME, cuda, with_res, relu, fp8):
    feats = _feats(3000, 64, torch.bfloat16, cuda, 5)
    w = _weights(27, 64, 96, cuda, 6)
    km = _km(27, 3000, 3000, 7, cuda)
    epi = _epilogue(96, 3000, torch.bfloat16, cuda, 8, with_res, relu)
    _check_shadow(f"res={with_res} relu={relu} fp8={fp8}", feats, w, km, epi, fp8=fp8)


@pytest.mark.parametrize("fp8", [True, False], ids=["e4m3", "bf16"])
@pytest.mark.parametrize("cout", [64, 256])
def test_shadow_tile_order_and_column_slices(ME, cuda, cout, fp8):
    """A real map: with its tile order (rows stored through slot_row) and without; 1000 rows on a
    wide layer run in column slices (tc::fwd_col_slice)."""
    from minkowskiengine_b200 import backend
    for n, seed in ((20_000, 11), (1000, 12)):
        x = _cloud(ME, n, 64, torch.bfloat16, cuda, seed=seed)
        key = x.coordinate_map_key
        km = x.coordinate_manager._manager._kernel_map(
            key, key, [3] * 3, [1] * 3, [1] * 3, ME.RegionType.HYPER_CUBE, None, False, False)
        assert km.out_order is not None
        w = _weights(27, 64, cout, cuda, 12)
        epi = _epilogue(cout, km.n_out, torch.bfloat16, cuda, 13, True, True)
        for m in (km, backend._KernelMap(km.out_nbr, km.in_nbr)):
            want = backend._conv_forward(x.F, w, m, epilogue=epi, fp8=fp8)
            scale = _shadow_scale(want)
            out, q = backend._conv_forward(x.F, w, m, epilogue=epi, fp8=fp8, shadow=scale)
            assert torch.equal(out, want)
            _same_bytes(q, backend.quantize_e4m3_static(out, scale),
                        f"n={n} ->{cout} ordered={m.out_order is not None}")


@pytest.mark.parametrize("out_dtype", [None, torch.float32], ids=["same", "fp32"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def test_shadow_stem(ME, cuda, dtype, out_dtype):
    from minkowskiengine_b200 import backend
    x = _cloud(ME, 8000, 3, dtype, cuda, seed=21)
    key = x.coordinate_map_key
    km = x.coordinate_manager._manager._kernel_map(
        key, key, [5] * 3, [1] * 3, [1] * 3, ME.RegionType.HYPER_CUBE, None, False, False)
    w = _weights(125, 3, 32, cuda, 22)
    assert backend._is_stem(w, dtype)
    epi = _epilogue(32, km.n_out, out_dtype or dtype, cuda, 23, True, True)
    want = backend._conv_forward(x.F, w, km, out_dtype=out_dtype, epilogue=epi)
    scale = _shadow_scale(want)
    out, q = backend._conv_forward(x.F, w, km, out_dtype=out_dtype, epilogue=epi, shadow=scale)
    assert torch.equal(out, want)
    _same_bytes(q, backend.quantize_e4m3_static(out, scale), f"stem {dtype}")


def test_routes_without_shadows(ME, cuda):
    """Exact fp32 (SIMT) and TF32 return no shadow and the output they return without one."""
    from minkowskiengine_b200 import backend
    feats = _feats(2000, 32, torch.float32, cuda, 1)
    w = _weights(8, 32, 64, cuda, 2)
    km = _km(8, 2000, 2000, 3, cuda)
    epi = _epilogue(64, 2000, torch.float32, cuda, 4, True, True)
    for prec in ("ieee", "tf32"):
        torch.backends.cuda.matmul.fp32_precision = prec
        want = backend._conv_forward(feats, w, km, epilogue=epi)
        out, q = backend._conv_forward(feats, w, km, epilogue=epi, shadow=_shadow_scale(want))
        assert q is None and torch.equal(out, want), prec


# ---- the public API -----------------------------------------------------------------------------
class _Pair(torch.nn.Module):
    def __init__(self, ME, C=64):
        super().__init__()
        self.a = ME.MinkowskiConvolution(C, C, kernel_size=3, dimension=3)
        self.b = ME.MinkowskiConvolution(C, C, kernel_size=3, dimension=3)
        self.c = ME.MinkowskiConvolution(C, C, kernel_size=3, dimension=3)


def _pair(ME, cuda, C=64):
    torch.manual_seed(1)
    net = _Pair(ME, C).to(cuda).eval()
    norms = [_norm(ME, C, cuda, s) for s in (2, 3, 4)]
    return net, norms


def _fwd(ME, net, norms, x):
    y = ME.fused_conv_bn_relu(net.a, norms[0], x)
    return y, ME.fused_conv_bn_relu(net.b, norms[1], y)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
def test_consumer_reading_a_shadow_equals_converting(ME, cuda, dtype):
    from minkowskiengine_b200 import backend, fp8_calibration as FC
    net, norms = _pair(ME, cuda)
    calib = ME.Fp8Calibration(net)
    with torch.no_grad():
        with calib.observe():
            for s in (31, 32):
                _fwd(ME, net, norms, _cloud(ME, 6000, 64, dtype, cuda, seed=s))
        assert calib.state_dict()["a"]["feeds"] == ["b"]
        x = _cloud(ME, 6000, 64, dtype, cuda, seed=33)
        calls = {"dyn": 0, "static": 0}
        real_dyn, real_st = backend._quantize_e4m3, backend.quantize_e4m3_static

        def dyn(*a):
            calls["dyn"] += 1
            return real_dyn(*a)

        def st(*a):
            calls["static"] += 1
            return real_st(*a)
        backend._quantize_e4m3, backend.quantize_e4m3_static = dyn, st
        try:
            with ME.fp8_inference(calib):
                y, z = _fwd(ME, net, norms, x)
                assert calls == {"dyn": 0, "static": 1}          # a's input only
                q, scale = FC.fresh_shadow(y)
                _same_bytes(q, real_st(y.F, scale), "shadow of a's output")
                # the same consumer on a new tensor (no shadow) converts at its static scale
                y2 = ME.SparseTensor(y.F, coordinate_map_key=y.coordinate_map_key,
                                     coordinate_manager=y.coordinate_manager)
                z2 = ME.fused_conv_bn_relu(net.b, norms[1], y2)
                assert calls == {"dyn": 0, "static": 2}
        finally:
            backend._quantize_e4m3, backend.quantize_e4m3_static = real_dyn, real_st
        assert torch.equal(z.F, z2.F)
        # an uncalibrated layer inside fp8_inference(calib) is today's fp8_inference()
        with ME.fp8_inference(calib):
            u1 = ME.fused_conv_bn_relu(net.c, norms[2], y)
            p1 = net.c(y)
        with ME.fp8_inference():
            u2 = ME.fused_conv_bn_relu(net.c, norms[2], y)
            p2 = net.c(y)
        assert torch.equal(u1.F, u2.F) and torch.equal(p1.F, p2.F)
        # a stale shadow is ignored: b converts the modified features
        with ME.fp8_inference(calib):
            y, _ = _fwd(ME, net, norms, x)
            y.F.mul_(0.5)
            z3 = ME.fused_conv_bn_relu(net.b, norms[1], y)
            z4 = ME.fused_conv_bn_relu(net.b, norms[1], ME.SparseTensor(
                y.F, coordinate_map_key=y.coordinate_map_key,
                coordinate_manager=y.coordinate_manager))
        assert torch.equal(z3.F, z4.F)


def test_links_through_real_modules(ME, cuda):
    """a (64 -> 32) feeds b32 (32 -> 64) directly, or through a module or a new tensor; b64 takes
    ME.cat(y, y)."""
    torch.manual_seed(4)
    net = torch.nn.ModuleDict({
        "a": ME.MinkowskiConvolution(64, 32, kernel_size=3, dimension=3),
        "b32": ME.MinkowskiConvolution(32, 64, kernel_size=3, dimension=3),
        "b64": ME.MinkowskiConvolution(64, 64, kernel_size=3, dimension=3)}).to(cuda).eval()
    na, nb = _norm(ME, 32, cuda, 1), _norm(ME, 64, cuda, 2)
    relu = ME.MinkowskiReLU(inplace=True)
    new = lambda y: ME.SparseTensor(y.F, coordinate_map_key=y.coordinate_map_key,     # noqa: E731
                                    coordinate_manager=y.coordinate_manager)
    cases = {"direct": ("b32", lambda y: y), "relu": ("b32", relu), "new": ("b32", new),
             "cat": ("b64", lambda y: ME.cat(y, y))}
    with torch.no_grad():
        for name, (b, between) in cases.items():
            calib = ME.Fp8Calibration(net)
            with calib.observe():
                y = ME.fused_conv_bn_relu(net["a"], na, _cloud(ME, 3000, 64, torch.float32, cuda, 5))
                ME.fused_conv_bn_relu(net[b], nb, between(y))
            sd = calib.state_dict()
            assert sd[b]["amax"] is not None, name
            assert sd["a"]["feeds"] == (["b32"] if name == "direct" else []), name


def test_batch_invariance(ME, cuda):
    """A calibrated K = 125 layer (no tile order) gives each cloud the same bits alone and in a
    batch of 8, rows matched by coordinate."""
    from examples.synthetic import surface_cloud
    torch.manual_seed(3)
    conv = ME.MinkowskiConvolution(32, 64, kernel_size=5, dimension=3).to(cuda).eval()
    norm = _norm(ME, 64, cuda, 5)
    clouds = [surface_cloud(20_000, 100 + j, batch=j) for j in range(8)]
    feats = [(torch.rand(len(c), 32, generator=torch.Generator().manual_seed(j)) - 0.5) * 4
             for j, c in enumerate(clouds)]
    calib = ME.Fp8Calibration(conv)
    with torch.no_grad():
        with calib.observe():
            for j in range(2):
                c = surface_cloud(20_000, 900 + j, batch=0)
                conv(ME.SparseTensor(torch.randn(len(c), 32).to(cuda), c.to(cuda)))
        with ME.fp8_inference(calib):
            xb = ME.SparseTensor(torch.cat(feats).to(cuda), torch.cat(clouds).to(cuda))
            yb = ME.fused_conv_bn_relu(conv, norm, xb)
            alone = []
            for j in range(8):
                c0 = clouds[j].clone()
                c0[:, 0] = 0
                alone.append(ME.fused_conv_bn_relu(
                    conv, norm, ME.SparseTensor(feats[j].to(cuda), c0.to(cuda))))
        with ME.fp8_inference():            # the dynamic scale: the batch changes the bits
            yd = ME.fused_conv_bn_relu(conv, norm, xb)

    def by_coord(y):
        C = y.C.long().cpu()
        key = ((C[:, 1] + 2 ** 19) * 2 ** 20 + (C[:, 2] + 2 ** 19)) * 2 ** 20 + (C[:, 3] + 2 ** 19)
        return C[:, 0], key, y.F.cpu()
    b_idx, b_key, b_F = by_coord(yb)
    _, _, d_F = by_coord(yd)
    dyn_differs = False
    for j in range(8):
        _, k1, F1 = by_coord(alone[j])
        m = b_idx == j
        kb, Fb, Fd = b_key[m], b_F[m], d_F[m]
        o1, ob = torch.argsort(k1), torch.argsort(kb)
        assert torch.equal(k1[o1], kb[ob])
        assert torch.equal(F1[o1], Fb[ob]), f"cloud {j}: alone and batched differ"
        dyn_differs |= not torch.equal(F1[o1], Fd[ob])
    print(f"dynamic scales: alone and batched differ for some cloud: {dyn_differs}")


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
def test_minkunet_calibrated(ME, cuda, dtype):
    """MinkUNet34C in eval, calibrated on two clouds other than the test clouds: the logits against
    the exact fp32 network within the limits of the dynamic test; no amax pass; conversions only
    where no shadow reaches (the four layers after ME.cat, and on fp32 features the layer after the
    exact-fp32 stem)."""
    from examples.synthetic import surface_cloud
    from minkowskiengine_b200 import backend
    coords = torch.cat([surface_cloud(50_000, j, batch=j) for j in range(2)], 0)
    feats = torch.rand(len(coords), 3, generator=torch.Generator().manual_seed(0))
    net = _minkunet(ME, cuda)
    with torch.no_grad():
        for _ in range(3):
            net.train()(ME.SparseTensor(feats.to(cuda), coords.to(cuda)))
    net.eval()
    calib = ME.Fp8Calibration(net)
    with torch.no_grad():
        with calib.observe():
            for s in (7, 8):
                c = torch.cat([surface_cloud(50_000, 10 * s + j, batch=j) for j in range(2)], 0)
                f = torch.rand(len(c), 3, generator=torch.Generator().manual_seed(s))
                net(ME.SparseTensor(f.to(dtype).to(cuda), c.to(cuda)))
        x32 = ME.SparseTensor(feats.to(cuda), coords.to(cuda))
        want = net(x32).F.double()
        x = ME.SparseTensor(feats.to(dtype).to(cuda), coords.to(cuda))
        calls = {"dyn": 0, "static": []}
        real_dyn, real_st = backend._quantize_e4m3, backend.quantize_e4m3_static

        def dyn(*a):
            calls["dyn"] += 1
            return real_dyn(*a)

        def st(f, s):
            calls["static"].append(f.shape[1])
            return real_st(f, s)
        backend._quantize_e4m3, backend.quantize_e4m3_static = dyn, st
        try:
            with ME.fp8_inference(calib):
                y = net(x).F.double()
                again = net(x).F.double()
        finally:
            backend._quantize_e4m3, backend.quantize_e4m3_static = real_dyn, real_st
    assert torch.equal(y, again)
    sd = calib.state_dict()
    n_cal = sum(1 for v in sd.values() if v["amax"] is not None)
    n_links = sum(len(v["feeds"]) for v in sd.values())
    assert calls["dyn"] == 0
    # per forward: the four layers after ME.cat, and the layer after the stem when the stem runs
    # the exact-fp32 kernels (which write no shadow)
    n_static = 4 + (dtype == torch.float32)
    assert len(calls["static"]) == 2 * n_static, calls["static"]
    print(f"static conversions per forward, by c_in: {calls['static'][:n_static]}")
    rms = float((y - want).pow(2).mean().sqrt() / want.pow(2).mean().sqrt())
    agree = float((y.argmax(1) == want.argmax(1)).double().mean())
    print(f"MinkUNet34C eval fp8 static ({dtype}) vs exact fp32: logits rms {rms:.3e}, argmax "
          f"agreement {agree:.4f}; {n_cal} calibrated layers, {n_links} links")
    assert bool(torch.isfinite(y).all())
    assert rms < 4.5e-2 and agree > 0.96
