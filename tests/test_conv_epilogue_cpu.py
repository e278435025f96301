"""fused_conv_bn_relu without a GPU: when a convolution takes eval batch norm, a residual and the
ReLU into its epilogue (case by case), the fp32 scale and shift it folds them into (against
float64), how the host hands the epilogue to meb200_conv_forward (a recording stub of the native
library), and the TypeError for modules it does not fuse."""
import ctypes

import pytest
import torch

import minkowskiengine_b200 as ME
from minkowskiengine_b200 import backend as B
from minkowskiengine_b200 import convolution as CV


@pytest.fixture
def native_ok(monkeypatch):
    """The native batch norm's shape / device check, which needs CUDA tensors, as a switch; records
    what it was asked about."""
    state = {"ok": True, "asked": []}

    def fake(bn, x):
        state["asked"].append((bn, tuple(x.shape), x.dtype))
        return state["ok"]
    monkeypatch.setattr(CV, "_native_ok", fake)
    return state


def _layers(c_in=16, c_out=32, bias=False, affine=True, kernel_size=3, stride=1):
    conv = ME.MinkowskiConvolution(c_in, c_out, kernel_size=kernel_size, stride=stride, bias=bias,
                                   dimension=3)
    norm = ME.MinkowskiBatchNorm(c_out, affine=affine).eval()
    return conv, norm


def test_eval_without_gradients_fuses(native_ok):
    conv, norm = _layers()
    x = torch.randn(10, 16)
    with torch.no_grad():
        assert CV._fuses(conv, norm, x, None)
        assert CV._fuses(conv, norm, x, torch.randn(7, 32))
    # grad mode on but nothing requires a gradient
    for p in list(conv.parameters()) + list(norm.parameters()):
        p.requires_grad_(False)
    assert CV._fuses(conv, norm, x, None)
    assert native_ok["asked"][-1] == (norm.bn, (0, 32), torch.float32)


def test_training_norm_does_not_fuse(native_ok):
    conv, norm = _layers()
    norm.train()
    with torch.no_grad():
        assert not CV._fuses(conv, norm, torch.randn(10, 16), None)


@pytest.mark.parametrize("which", ["input", "kernel", "bias", "bn_weight", "bn_bias", "residual"])
def test_a_tensor_needing_a_gradient_does_not_fuse(native_ok, which):
    conv, norm = _layers(bias=True)
    for p in list(conv.parameters()) + list(norm.parameters()):
        p.requires_grad_(False)
    x, res = torch.randn(10, 16), torch.randn(10, 32)
    t = {"input": x, "kernel": conv.kernel, "bias": conv.bias, "bn_weight": norm.bn.weight,
         "bn_bias": norm.bn.bias, "residual": res}[which]
    assert CV._fuses(conv, norm, x, res)
    t.requires_grad_(True)
    assert not CV._fuses(conv, norm, x, res)
    with torch.no_grad():                  # grad mode off: nothing needs a gradient
        assert CV._fuses(conv, norm, x, res)


def test_matrix_product_layer_does_not_fuse(native_ok):
    conv, norm = _layers(kernel_size=1)
    assert conv.use_mm
    with torch.no_grad():
        assert not CV._fuses(conv, norm, torch.randn(10, 16), None)
    conv, norm = _layers(kernel_size=1, stride=2)       # K = 1 with a stride runs the kernels
    assert not conv.use_mm
    with torch.no_grad():
        assert CV._fuses(conv, norm, torch.randn(10, 16), None)


def test_native_batch_norm_check_decides(native_ok):
    conv, norm = _layers()
    native_ok["ok"] = False
    with torch.no_grad():
        assert not CV._fuses(conv, norm, torch.randn(10, 16).bfloat16(), None)
    assert native_ok["asked"][-1] == (norm.bn, (0, 32), torch.bfloat16)


def test_residual_in_another_dtype_does_not_fuse(native_ok):
    conv, norm = _layers()
    x = torch.randn(10, 16).bfloat16()
    with torch.no_grad():
        assert CV._fuses(conv, norm, x, torch.randn(10, 32).bfloat16())
        assert not CV._fuses(conv, norm, x, torch.randn(10, 32))


def test_native_ok_rejects_what_the_epilogue_cannot_take():
    """The real check: CPU features and a norm without running statistics fail."""
    from minkowskiengine_b200.normalization import _native_ok
    bn = torch.nn.BatchNorm1d(32).eval()
    assert not _native_ok(bn, torch.empty(0, 32))                     # not CUDA
    assert not _native_ok(torch.nn.BatchNorm1d(32, track_running_stats=False), torch.empty(0, 32))


def test_unsupported_modules_raise_type_error():
    conv, norm = _layers()
    with pytest.raises(TypeError, match="MinkowskiConvolution"):
        ME.fused_conv_bn_relu(torch.nn.Linear(16, 32), norm, None)
    with pytest.raises(TypeError, match="MinkowskiConvolution"):
        ME.fused_conv_bn_relu(ME.MinkowskiChannelwiseConvolution(32, 3, dimension=3), norm, None)
    with pytest.raises(TypeError, match="MinkowskiBatchNorm"):
        ME.fused_conv_bn_relu(conv, ME.MinkowskiInstanceNorm(32), None)
    with pytest.raises(TypeError, match="MinkowskiBatchNorm"):
        ME.fused_conv_bn_relu(conv, torch.nn.BatchNorm1d(32), None)


@pytest.mark.parametrize("affine", [True, False], ids=["affine", "no_affine"])
@pytest.mark.parametrize("bias", [False, True], ids=["no_bias", "bias"])
def test_scale_shift_folding_against_float64(affine, bias):
    from minkowskiengine_b200.normalization import _eval_scale_shift
    g = torch.Generator().manual_seed(3)
    C = 48
    bn = torch.nn.BatchNorm1d(C, eps=1e-3, affine=affine).eval()
    bn.running_mean.copy_(torch.randn(C, generator=g) * 3)
    bn.running_var.copy_(torch.rand(C, generator=g) * 4 + 0.01)
    if affine:
        with torch.no_grad():
            bn.weight.copy_(torch.randn(C, generator=g))
            bn.bias.copy_(torch.randn(C, generator=g))
    conv_bias = torch.randn(1, C, generator=g) if bias else None
    scale, shift = _eval_scale_shift(bn, conv_bias)
    assert scale.dtype == shift.dtype == torch.float32 and scale.shape == shift.shape == (C,)
    assert scale.is_contiguous() and shift.is_contiguous()
    d = lambda t: t.detach().double()                                   # noqa: E731
    invstd = 1.0 / torch.sqrt(d(bn.running_var) + bn.eps)
    s64 = invstd * d(bn.weight) if affine else invstd
    b64 = d(bn.bias) if affine else torch.zeros(C, dtype=torch.float64)
    sh64 = b64 - d(bn.running_mean) * s64
    if bias:
        sh64 = sh64 + d(conv_bias).flatten() * s64
    # a few fp32 roundings: rsqrt (<= 2 ulp), the product, and each term of the shift
    assert torch.allclose(scale.double(), s64, rtol=2 ** -20, atol=0)
    mag = (d(bn.running_mean) * s64).abs() + b64.abs() + (d(conv_bias).flatten() * s64).abs() \
        if bias else (d(bn.running_mean) * s64).abs() + b64.abs()
    assert bool(((shift.double() - sh64).abs() <= 2 ** -20 * mag).all())
    # y = x * scale + shift is eval batch norm after the bias: the composition in float64
    x = torch.randn(100, C, generator=g).double()
    xb = x + (d(conv_bias) if bias else 0)
    want = (xb - d(bn.running_mean)) * invstd * (d(bn.weight) if affine else 1) + b64
    got = x * scale.double() + shift.double()
    assert torch.allclose(got, want, rtol=0, atol=1e-5 * float(want.abs().max()))


class _Stub:
    """Stands in for the library: records every call, and the epilogue struct the forward got
    (read during the call, while the host keeps it alive)."""

    def __init__(self, calls):
        self.calls = calls

    def __getattr__(self, name):
        def fn(*args):
            rec = None
            if name == "meb200_conv_forward" and args[-2] is not None:
                e = B._ConvEpilogue.from_address(args[-2])
                rec = (e.scale, e.shift, e.residual, e.relu)
            self.calls.append((name, args, rec))
            return 0
        return fn


class _Map:
    K, n_in, n_out, n_pairs = 27, 10, 12, 40
    out_nbr = in_nbr = out_order = in_order = None


@pytest.fixture
def stub(monkeypatch):
    from minkowskiengine_b200 import _lib
    calls = []
    monkeypatch.setattr(_lib, "load", lambda: _Stub(calls))
    monkeypatch.setattr(_lib, "current_stream", lambda: None)
    saved = torch.backends.cuda.matmul.fp32_precision
    torch.backends.cuda.matmul.fp32_precision = "ieee"          # exact fp32: no weight packing
    yield calls
    torch.backends.cuda.matmul.fp32_precision = saved


def test_forward_passes_null_without_epilogue(stub):
    B._conv_forward_impl(torch.randn(10, 32), torch.randn(27, 32, 64), _Map())
    (name, args, rec), = [c for c in stub if c[0] == "meb200_conv_forward"]
    assert len(args) == 15 and args[-2] is None and rec is None


@pytest.mark.parametrize("relu", [True, False])
@pytest.mark.parametrize("with_res", [True, False])
def test_forward_passes_the_epilogue(stub, relu, with_res):
    scale, shift = torch.rand(64), torch.rand(64)
    res = torch.randn(12, 64) if with_res else None
    B._conv_forward_impl(torch.randn(10, 32), torch.randn(27, 32, 64), _Map(),
                         epilogue=(scale, shift, res, relu))
    (name, args, rec), = [c for c in stub if c[0] == "meb200_conv_forward"]
    assert rec == (scale.data_ptr(), shift.data_ptr(), res.data_ptr() if with_res else None,
                   int(relu))


@pytest.mark.parametrize("bad", ["scale_shape", "shift_dtype", "res_shape", "res_dtype"])
def test_forward_rejects_a_malformed_epilogue(stub, bad):
    scale, shift, res = torch.rand(64), torch.rand(64), torch.randn(12, 64)
    if bad == "scale_shape":
        scale = torch.rand(32)
    elif bad == "shift_dtype":
        shift = shift.double()
    elif bad == "res_shape":
        res = torch.randn(10, 64)
    else:
        res = res.bfloat16()
    with pytest.raises(RuntimeError, match="epilogue"):
        B._conv_forward_impl(torch.randn(10, 32), torch.randn(27, 32, 64), _Map(),
                             epilogue=(scale, shift, res, True))
    assert not [c for c in stub if c[0] == "meb200_conv_forward"]


def test_epilogue_struct_layout():
    """_ConvEpilogue is meb200_conv_epilogue: three pointers, then the int32 flag."""
    P = ctypes.sizeof(ctypes.c_void_p)
    assert B._ConvEpilogue.relu.offset == 3 * P
    assert ctypes.sizeof(B._ConvEpilogue) == 4 * P
