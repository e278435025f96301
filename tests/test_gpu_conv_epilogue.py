"""The convolution epilogue (meb200_conv_epilogue: eval batch norm as a per-channel affine map, a
residual and the ReLU applied to the fp32 accumulator) on every forward route, and
ME.fused_conv_bn_relu through the public API.

Routes, each checked through the tensor-core launch counter: `k_conv_wg` in bf16 / fp16 at every
column width it dispatches (16 ... 256, and 272 / 512 over two launches of column slices), TF32,
the exact-fp32 and bf16 SIMT gather-GEMM, the small-cin kernel and the bf16 / fp16 network stem.

Bound: the accumulator is the route's own, within acc * 2^-20 * A of float64 (tests/helpers.py,
DESIGN.md §6); the epilogue scales that error by |scale| <= max|scale| and adds its two fp32
roundings (the fused multiply-add, the residual add: 2^-24 each, relative to the largest term) and
one rounding to the output dtype.  On the exactly summable operands of tests/test_gpu_fp32_conv.py
with power-of-two scales the exact-fp32 routes must equal float64 bit for bit."""
import pytest
import torch

from helpers import TC_ACC, _Route, _pairs, _table, half_ulp, ref_conv

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def precision():
    saved = torch.backends.cuda.matmul.fp32_precision
    torch.backends.cuda.matmul.fp32_precision = "ieee"
    yield
    torch.backends.cuda.matmul.fp32_precision = saved


def _tf32_exact(t):
    return (t.contiguous().view(torch.int32) & ~0x1FFF).view(torch.float32)


def _operands(cin, cout, n_in, n_out, K, dtype, device, seed, tf32=False):
    g = torch.Generator().manual_seed(seed)
    feats = torch.rand(n_in, cin, generator=g) - 0.5
    w = (torch.rand(K, cin, cout, generator=g) - 0.5) / (cin ** 0.5)
    if tf32:
        feats, w = _tf32_exact(feats), _tf32_exact(w)
    return feats.to(dtype).to(device), w.to(device)


def _epilogue(cout, n_out, out_dtype, device, seed, with_res, relu, exact=False):
    """(scale, shift, residual, relu): signed scales of mixed magnitude, shifts around zero so that
    the ReLU clamps part of every channel."""
    g = torch.Generator().manual_seed(seed)
    if exact:          # powers of two, multiples of 1/128, multiples of 1/8
        scale = 2.0 ** torch.randint(-2, 2, (cout,), generator=g).float() * \
            (torch.randint(0, 2, (cout,), generator=g) * 2 - 1)
        shift = torch.randint(-64, 65, (cout,), generator=g) / 128.0
        res = torch.randint(-8, 9, (n_out, cout), generator=g) / 8.0
    else:
        scale = (torch.rand(cout, generator=g) * 3 + 0.1) * (torch.randint(0, 2, (cout,), generator=g) * 2 - 1)
        shift = torch.randn(cout, generator=g) * 0.3
        res = torch.randn(n_out, cout, generator=g) * 0.5
    res = res.to(out_dtype).to(device) if with_res else None
    return scale.to(device), shift.to(device), res, relu


def _expected(ref, A, epi, out_dtype, acc):
    """float64 result of the epilogue on the float64 convolution, and the per-element bound."""
    scale, shift, res, relu = epi
    s, b = scale.double(), shift.double()
    pre = ref * s + b
    mag = (ref * s).abs() + b.abs()
    if res is not None:
        pre = pre + res.double()
        mag = mag + res.double().abs()
    y = pre.clamp(min=0) if relu else pre
    delta = A.double() * (acc * 2.0 ** -20) * float(s.abs().max()) + 2.0 ** -22 * mag
    if out_dtype != torch.float32:
        delta = half_ulp(y.abs() + delta, out_dtype) + delta
    return y, delta


def _check(y, y_ref, bound, what):
    err = (y.double() - y_ref).abs()
    bad = ~(err <= bound)
    if bool(bad.any()):
        j = int(torch.nonzero(bad.flatten())[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements outside the "
                             f"bound; first at flat index {j}: got {y.flatten()[j].item()!r}, "
                             f"float64 {y_ref.flatten()[j].item()!r}, |err| "
                             f"{err.flatten()[j].item():.3e} > {bound.flatten()[j].item():.3e}")


def _run(case, feats, w, km, epi, out_dtype, tc, acc):
    """The fused forward twice (bit-identical), against float64 within the route's bound, empty
    rows included."""
    from minkowskiengine_b200 import backend
    with _Route(tc, case):
        y = backend._conv_forward(feats, w, km, out_dtype=out_dtype, epilogue=epi)
        y2 = backend._conv_forward(feats, w, km, out_dtype=out_dtype, epilogue=epi)
    assert y.dtype == out_dtype
    assert torch.equal(y, y2), f"{case}: differs run to run"
    wl = w if feats.dtype == torch.float32 else w.to(feats.dtype)
    ref, A = ref_conv(feats, wl, _pairs(km.out_nbr), km.n_out)
    y_ref, bound = _expected(ref, A, epi, out_dtype, acc)
    _check(y, y_ref, bound, case)
    empty = (km.out_nbr < 0).all(0)
    assert bool(empty.any()), "the tables have rows without neighbours"
    return y


# (cin, cout, n_out, K, stem) for the bf16 / fp16 tensor-core routes: every column width of
# MEB_COLS_DISPATCH, two with column slices past 256, the stem
TC_WIDTHS = [(32, 16 * i, 2000, 8, False) for i in range(1, 17)] + \
    [(64, 272, 3000, 27, False), (32, 512, 1500, 8, False), (3, 32, 5000, 125, True),
     (4, 96, 3000, 27, True)]


def _km(K, n_out, n_in, seed, device):
    from minkowskiengine_b200 import backend
    out_nbr = _table(K, n_out, n_in, 0.35, seed, device)
    return backend._KernelMap(out_nbr, torch.full((K, n_in), -1, dtype=torch.int32, device=device))


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("cin,cout,n_out,K,stem", TC_WIDTHS,
                         ids=[f"{c[0]}to{c[1]}_K{c[3]}" + ("_stem" if c[4] else "") for c in TC_WIDTHS])
def test_tensor_core_widths(ME, cuda, dtype, cin, cout, n_out, K, stem):
    from minkowskiengine_b200 import backend
    n_in = n_out
    feats, w = _operands(cin, cout, n_in, n_out, K, dtype, cuda, seed=cin + cout + K)
    assert backend._is_stem(w, dtype) == stem
    km = _km(K, n_out, n_in, cout + K, cuda)
    case = f"{dtype} {cin}->{cout} K={K}"
    epi = _epilogue(cout, n_out, dtype, cuda, cout, with_res=True, relu=True)
    _run(case, feats, w, km, epi, dtype, True, TC_ACC)


@pytest.mark.parametrize("with_res,relu", [(False, False), (False, True), (True, False)],
                         ids=["affine", "relu", "residual"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def test_tensor_core_residual_and_relu(ME, cuda, dtype, with_res, relu):
    feats, w = _operands(64, 96, 3000, 3000, 27, dtype, cuda, seed=5)
    km = _km(27, 3000, 3000, 6, cuda)
    epi = _epilogue(96, 3000, dtype, cuda, 7, with_res, relu)
    _run(f"{dtype} res={with_res} relu={relu}", feats, w, km, epi, dtype, True, TC_ACC)


def test_tensor_core_fp32_output(ME, cuda):
    """bf16 operands, fp32 output and an fp32 residual."""
    feats, w = _operands(32, 64, 2000, 2000, 27, torch.bfloat16, cuda, seed=8)
    km = _km(27, 2000, 2000, 9, cuda)
    epi = _epilogue(64, 2000, torch.float32, cuda, 10, True, True)
    _run("bf16 -> fp32", feats, w, km, epi, torch.float32, True, TC_ACC)


@pytest.mark.parametrize("cout", [48, 272])
def test_tf32(ME, cuda, cout):
    torch.backends.cuda.matmul.fp32_precision = "tf32"
    feats, w = _operands(32, cout, 3000, 3000, 27, torch.float32, cuda, seed=cout, tf32=True)
    km = _km(27, 3000, 3000, cout + 1, cuda)
    epi = _epilogue(cout, 3000, torch.float32, cuda, cout + 2, True, True)
    _run(f"tf32 32->{cout}", feats, w, km, epi, torch.float32, True, TC_ACC)


# (cin, cout, K, dtypes) off the tensor cores: SIMT gather-GEMM, small-cin (c_in <= 4, c_out <= 64,
# one and two 32-channel slabs), the small-cin fallback to the gather-GEMM (4 -> 56, K = 343)
CUDA_CORE = {"simt_20to40": (20, 40, 27), "simt_64to130": (64, 130, 27),
             "small_cin_3to20": (3, 20, 125), "small_cin_4to40": (4, 40, 27),
             "small_cin_fallback_4to56": (4, 56, 343)}


@pytest.mark.parametrize("with_res,relu", [(True, True), (False, False)], ids=["res_relu", "affine"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16],
                         ids=["fp32", "bf16", "fp16"])
@pytest.mark.parametrize("case", list(CUDA_CORE))
def test_cuda_core_routes(ME, cuda, case, dtype, with_res, relu):
    from minkowskiengine_b200 import backend
    cin, cout, K = CUDA_CORE[case]
    feats, w = _operands(cin, cout, 3000, 3000, K, dtype, cuda, seed=cin * 7 + cout)
    assert not backend._is_stem(w, dtype)
    km = _km(K, 3000, 3000, cin + cout, cuda)
    epi = _epilogue(cout, 3000, dtype, cuda, cout, with_res, relu)
    _run(f"{case} {dtype}", feats, w, km, epi, dtype, False, 1.0)


@pytest.mark.parametrize("case", list(CUDA_CORE))
def test_exact_fp32_equals_float64(ME, cuda, case):
    """Operands k / 8 and k / 16 (|k| <= 8), power-of-two scales, shifts k / 128, residuals k / 8:
    every fma of the convolution and of the epilogue is exact, so the output is float64's."""
    from minkowskiengine_b200 import backend
    cin, cout, K = CUDA_CORE[case]
    g = torch.Generator().manual_seed(cin + cout)
    feats = (torch.randint(-8, 9, (2000, cin), generator=g) / 8.0).to(cuda)
    w = (torch.randint(-8, 9, (K, cin, cout), generator=g) / 16.0).to(cuda)
    km = _km(K, 2000, 2000, cout, cuda)
    for with_res, relu in [(True, True), (False, False), (True, False)]:
        epi = _epilogue(cout, 2000, torch.float32, cuda, K, with_res, relu, exact=True)
        with _Route(False, case):
            y = backend._conv_forward(feats, w, km, epilogue=epi)
        ref, _ = ref_conv(feats, w, _pairs(km.out_nbr), 2000)
        y_ref, _ = _expected(ref, torch.zeros_like(ref), epi, torch.float32, 1.0)
        assert torch.equal(y.double(), y_ref), f"{case} res={with_res} relu={relu}"


def test_null_epilogue_is_the_plain_forward(ME, cuda):
    """meb200_conv_forward called the old way (no epilogue argument) and with NULL: the same bits."""
    from minkowskiengine_b200 import _lib, backend
    lib = _lib.load()
    feats, w = _operands(32, 64, 2000, 2000, 27, torch.bfloat16, cuda, seed=11)
    km = _km(27, 2000, 2000, 12, cuda)
    y = backend._conv_forward(feats, w, km)
    w_cast, w_t = backend._packed_weights(w, torch.bfloat16)
    out = torch.empty_like(y)
    _lib.check(lib.meb200_conv_forward(
        _lib.ptr(feats), _lib.BF16, 2000, 32, _lib.ptr(w_cast), _lib.ptr(w_t), 27, 64,
        _lib.ptr(km.out_nbr), 2000, _lib.ptr(out), _lib.BF16, None, _lib.current_stream()))
    assert torch.equal(out, y)


# ---- the public function ----------------------------------------------------------------------
def _cloud(ME, n, c, dtype, device, seed):
    from oracle import oracle_np as O
    coords = O.surface_cloud(n, seed=seed)
    feats = torch.rand(len(coords), c, generator=torch.Generator().manual_seed(seed)) - 0.5
    return ME.SparseTensor(feats.to(dtype).to(device), coords.to(device))


def _norm(ME, C, device, seed, affine=True):
    norm = ME.MinkowskiBatchNorm(C, affine=affine).to(device)
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        norm.bn.running_mean.copy_(torch.randn(C, generator=g) * 0.2)
        norm.bn.running_var.copy_(torch.rand(C, generator=g) + 0.5)
        if affine:
            norm.bn.weight.copy_(torch.randn(C, generator=g))
            norm.bn.bias.copy_(torch.randn(C, generator=g) * 0.3)
    return norm.eval()


def _unfused(conv, norm, x, residual, relu):
    from minkowskiengine_b200.normalization import _bn_tail
    out = conv(x)
    if residual is None and not relu:
        return out, norm(out)
    return out, _bn_tail(norm, out, residual, relu)


LAYERS = {"conv_k3": lambda ME, c, d: ME.MinkowskiConvolution(c, c, kernel_size=3, dimension=d),
          "conv_k2s2": lambda ME, c, d: ME.MinkowskiConvolution(c, c, kernel_size=2, stride=2,
                                                                  dimension=d),
          "conv_k3_bias": lambda ME, c, d: ME.MinkowskiConvolution(c, c, kernel_size=3, bias=True,
                                                                     dimension=d),
          "transpose_k2s2": lambda ME, c, d: ME.MinkowskiConvolutionTranspose(
              c, c, kernel_size=2, stride=2, dimension=d),
          "generative_k2s2": lambda ME, c, d: ME.MinkowskiGenerativeConvolutionTranspose(
              c, c, kernel_size=2, stride=2, dimension=d)}


@pytest.mark.parametrize("affine", [True, False], ids=["affine", "no_affine"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("layer", list(LAYERS))
def test_public_fused_against_composition(ME, cuda, layer, dtype, affine):
    """Fused against the two-pass composition: the same accumulator, so they differ by the
    composition's extra rounding of the convolution output (scaled by |scale|), one rounding of
    each output and the fp32 epilogue's roundings."""
    from minkowskiengine_b200 import _lib
    torch.manual_seed(0)
    C = 32
    x = _cloud(ME, 4000, C, dtype, cuda, seed=3)
    if layer.startswith(("transpose", "generative")):
        x = ME.MinkowskiConvolution(C, C, kernel_size=2, stride=2, dimension=3).to(cuda)(x).detach()
    conv = LAYERS[layer](ME, C, 3).to(cuda)
    if conv.bias is not None:
        with torch.no_grad():
            conv.bias.normal_()
    norm = _norm(ME, C, cuda, 4, affine)
    scale = norm.bn.running_var.rsqrt() * (norm.bn.weight.detach() if affine else 1.0)
    with torch.no_grad():
        c = conv(x)
        cases = [(None, True), (None, False)]
        if not layer.startswith("generative"):   # a generative layer's output map is a new one
            cases += [(ME.SparseTensor(torch.randn_like(c.F), coordinate_map_key=c.coordinate_map_key,
                                       coordinate_manager=c.coordinate_manager), True)]
        s_max = float(scale.abs().max())
        b_max = float(conv.bias.abs().max()) if conv.bias is not None else 0.0
        for residual, relu in cases:
            y = ME.fused_conv_bn_relu(conv, norm, x, residual, relu)
            n0 = _lib.launch_count()
            y2 = ME.fused_conv_bn_relu(conv, norm, x, residual, relu)
            n_fused = _lib.launch_count() - n0
            assert torch.equal(y.F, y2.F)
            n0 = _lib.launch_count()
            c_out, want = _unfused(conv, norm, x, residual, relu)
            if not layer.startswith("generative"):
                assert _lib.launch_count() - n0 == n_fused + 1, "the fused call saves one pass"
                assert y.coordinate_map_key == want.coordinate_map_key
            assert y.F.shape == want.F.shape and y.F.dtype == dtype
            c = c_out.F.double().abs()
            r = residual.F.double().abs() if residual is not None else 0.0
            # the composition rounds the convolution output (and, with a bias, the bias and the
            # sum) to the dtype; both round the output once; fp32 roundings of the epilogue
            t1 = 3 * s_max * half_ulp(c + b_max, dtype) if dtype != torch.float32 else 0.0
            t2 = 2.0 ** -20 * (c * s_max + r + 1.0)
            tol = t1 + t2
            if dtype != torch.float32:
                tol = tol + 2 * half_ulp(want.F.double().abs() + tol, dtype)
            err = (y.F.double() - want.F.double()).abs()
            assert bool((err <= tol).all()), f"{layer} res={residual is not None} relu={relu}: " \
                f"max err {float(err.max()):.3e}"


def test_zero_convolution_gives_the_shift(ME, cuda):
    """A zero accumulator (as on a row without neighbours, which the route tests above cover on
    their tables) gives relu(shift), what the composition gives for a zero convolution output."""
    torch.manual_seed(1)
    C = 32
    coords = torch.tensor([[0, 0, 0, 0], [0, 1, 0, 0], [0, 9, 9, 9]], dtype=torch.int32)
    x = ME.SparseTensor(torch.randn(3, C).to(cuda), coords.to(cuda))
    conv = ME.MinkowskiConvolutionTranspose(C, C, kernel_size=3, stride=1, dimension=3).to(cuda)
    with torch.no_grad():
        conv.kernel.zero_()
        norm = _norm(ME, C, cuda, 2)
        y = ME.fused_conv_bn_relu(conv, norm, x, None, True)
        _, want = _unfused(conv, norm, x, None, True)
    assert torch.allclose(y.F, want.F, rtol=1e-6, atol=1e-6)
    from minkowskiengine_b200.normalization import _eval_scale_shift
    _, shift = _eval_scale_shift(norm.bn)
    assert torch.equal(y.F, shift.clamp(min=0).expand_as(y.F))


def _fallback_equal(ME, conv, norm, x, residual=None, relu=True):
    from minkowskiengine_b200 import _lib
    y = ME.fused_conv_bn_relu(conv, norm, x, residual, relu)
    n0 = _lib.launch_count()
    _, want = _unfused(conv, norm, x, residual, relu)
    n_composition = _lib.launch_count() - n0
    n0 = _lib.launch_count()
    y2 = ME.fused_conv_bn_relu(conv, norm, x, residual, relu)
    assert _lib.launch_count() - n0 == n_composition, "a fallback launches the composition"
    assert torch.equal(y.F, want.F) and torch.equal(y2.F, want.F)
    assert y.coordinate_map_key == want.coordinate_map_key


def test_fallbacks_are_the_composition(ME, cuda):
    torch.manual_seed(2)
    C = 32
    x = _cloud(ME, 3000, C, torch.bfloat16, cuda, seed=5)
    conv = ME.MinkowskiConvolution(C, C, kernel_size=3, dimension=3).to(cuda)
    norm = _norm(ME, C, cuda, 6)
    res = ME.SparseTensor(torch.randn_like(x.F), coordinate_map_key=x.coordinate_map_key,
                          coordinate_manager=x.coordinate_manager)
    # gradients needed: grad mode on and the parameters require them
    _fallback_equal(ME, conv, norm, x, res)
    _fallback_equal(ME, conv, norm, x, None, False)
    with torch.no_grad():
        # a training norm (its running statistics move: compare on copies of one state)
        norm.train()
        state = {k: v.clone() for k, v in norm.state_dict().items()}
        y = ME.fused_conv_bn_relu(conv, norm, x, res)
        norm.load_state_dict(state)
        _, want = _unfused(conv, norm, x, res, True)
        assert torch.equal(y.F, want.F)
        norm.eval()
        # a K = 1 stride-1 layer (a matrix product)
        _fallback_equal(ME, ME.MinkowskiConvolution(C, C, kernel_size=1, dimension=3).to(cuda),
                        norm, x, res)
        # a channel count the native batch norm does not take
        conv20 = ME.MinkowskiConvolution(C, 20, kernel_size=3, dimension=3).to(cuda)
        _fallback_equal(ME, conv20, _norm(ME, 20, cuda, 7), x)
        # a residual in another dtype, and one on another map
        _fallback_equal(ME, conv, norm, x, ME.SparseTensor(
            res.F.float(), coordinate_map_key=x.coordinate_map_key,
            coordinate_manager=x.coordinate_manager))
        down = ME.MinkowskiConvolution(C, C, kernel_size=2, stride=2, dimension=3).to(cuda)(x)
        with pytest.raises(AssertionError, match="same coordinate map"):
            ME.fused_conv_bn_relu(conv, norm, x, down)


# ---- the network ------------------------------------------------------------------------------
class _Unfused:
    """The package as a module handle without fused_conv_bn_relu: the examples then build the
    two-pass composition."""

    def __init__(self, ME):
        self._ME = ME

    def __getattr__(self, name):
        if name == "fused_conv_bn_relu":
            raise AttributeError(name)
        return getattr(self._ME, name)


def _minkunet(ME, handle, device):
    from examples.minkunet import minkunet
    torch.manual_seed(0)
    return minkunet("MinkUNet34C", handle, 3, 20, 3).to(device)


def test_minkunet_eval_fused_against_composition(ME, cuda):
    from oracle import oracle_np as O
    coords = torch.cat([O.surface_cloud(40_000, seed=s) for s in (1, 2)])
    coords[40_000:, 0] = 1
    feats = torch.rand(len(coords), 3, generator=torch.Generator().manual_seed(3)).bfloat16()
    fused, plain = _minkunet(ME, ME, cuda), _minkunet(ME, _Unfused(ME), cuda)
    with torch.no_grad():          # running statistics of a few batches, the same in both nets
        for _ in range(3):
            fused(ME.SparseTensor(feats.to(cuda), coords.to(cuda)))
    plain.load_state_dict(fused.state_dict())
    fused.eval(), plain.eval()
    with torch.no_grad():
        y = fused(ME.SparseTensor(feats.to(cuda), coords.to(cuda))).F.double()
        y2 = fused(ME.SparseTensor(feats.to(cuda), coords.to(cuda))).F.double()
        want = plain(ME.SparseTensor(feats.to(cuda), coords.to(cuda))).F.double()
    assert torch.equal(y, y2)
    rms = float((y - want).pow(2).mean().sqrt() / want.pow(2).mean().sqrt())
    mx = float((y - want).abs().max() / want.abs().max())
    agree = float((y.argmax(1) == want.argmax(1)).double().mean())
    print(f"MinkUNet34C eval bf16 fused vs composition: logits rms {rms:.2e}, max {mx:.2e} of the "
          f"composition's; per-point argmax agreement {agree:.4f}")
    assert rms < 6e-2 and mx < 1e-1
    assert agree > 0.9


def test_minkunet_training_is_the_composition(ME, cuda):
    """In training the fused call is the composition: the same loss and gradients, bit for bit."""
    from oracle import oracle_np as O
    coords = O.surface_cloud(30_000, seed=4)
    feats = torch.rand(len(coords), 3, generator=torch.Generator().manual_seed(5)).bfloat16()
    grads, losses = [], []
    for handle in (ME, _Unfused(ME)):
        net = _minkunet(ME, handle, cuda).train()
        out = net(ME.SparseTensor(feats.to(cuda), coords.to(cuda)))
        loss = out.F.float().pow(2).mean()
        loss.backward()
        losses.append(loss.detach())
        grads.append([p.grad.clone() for p in net.parameters()])
    assert torch.equal(losses[0], losses[1])
    assert all(torch.equal(a, b) for a, b in zip(*grads))
