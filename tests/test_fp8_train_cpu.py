"""fp8 training without a GPU: which layers ME.fp8_training() selects (case by case), the context's
rules, the arguments the host hands the library for the e4m3 forward, the e5m2 x e4m3 dgrad and the
unchanged weight gradient (a stub that records every call), and the e5m2 scale formula against
float64 at its edges."""
import ctypes
import threading

import numpy as np
import pytest
import torch

import minkowskiengine_b200 as ME
from minkowskiengine_b200 import backend as B
from minkowskiengine_b200 import convolution as CV

E5M2_MAX = 57344.0
FLT_MAX = np.finfo(np.float32).max


def _conv(c_in=32, c_out=64, kernel_size=3, stride=1, bias=False, cls=ME.MinkowskiConvolution):
    return cls(c_in, c_out, kernel_size=kernel_size, stride=stride, bias=bias, dimension=3)


def _x(c=32, dtype=torch.float32, grad=True):
    return torch.randn(10, c).to(dtype).requires_grad_(grad)


# ---- the context ---------------------------------------------------------------------------------
def test_off_by_default_and_nests():
    conv = _conv()
    assert not B.fp8_training_enabled() and not CV._fp8_train(conv, _x())
    with ME.fp8_training():
        assert CV._fp8_train(conv, _x())
        with ME.fp8_training():
            assert B.fp8_training_enabled()
        assert B.fp8_training_enabled()
    assert not B.fp8_training_enabled() and not CV._fp8_train(conv, _x())


def test_survives_exceptions():
    with pytest.raises(ValueError):
        with ME.fp8_training():
            raise ValueError
    assert not B.fp8_training_enabled()


def test_thread_local():
    seen = []
    with ME.fp8_training():
        t = threading.Thread(target=lambda: seen.append(B.fp8_training_enabled()))
        t.start()
        t.join()
        assert B.fp8_training_enabled()
    assert seen == [False]


def test_independent_of_fp8_inference_and_calibration():
    """fp8_inference() selects layers that need no gradient, fp8_training() layers that need one:
    nested either way, each keeps its own selection."""
    conv = _conv()
    with ME.fp8_inference():
        assert not B.fp8_training_enabled()
        with ME.fp8_training():
            assert B.fp8_enabled() and B.fp8_training_enabled()
            assert CV._fp8_train(conv, _x()) and not CV._fp8(conv, _x())
            with torch.no_grad():
                assert CV._fp8(conv, _x()) and not CV._fp8_train(conv, _x())
        assert B.fp8_enabled() and not B.fp8_training_enabled()
    with ME.fp8_training():
        with ME.fp8_inference():
            assert CV._fp8_train(conv, _x())
        assert not B.fp8_enabled()
    net = torch.nn.Sequential(conv)
    calib = ME.Fp8Calibration(net)
    with calib.observe():
        with ME.fp8_training():
            assert B.fp8_observer() is calib and CV._fp8_train(conv, _x())
        assert B.fp8_observer() is calib and not B.fp8_training_enabled()
    assert B.fp8_observer() is None


# ---- the selection rule ----------------------------------------------------------------------------
@pytest.mark.parametrize("which", ["input", "kernel", "bias"])
def test_one_tensor_needing_a_gradient_selects(which):
    conv = _conv(bias=True)
    for p in conv.parameters():
        p.requires_grad_(False)
    x = _x(grad=False)
    t = {"input": x, "kernel": conv.kernel, "bias": conv.bias}[which]
    with ME.fp8_training():
        assert not CV._fp8_train(conv, x)
        t.requires_grad_(True)
        assert CV._fp8_train(conv, x)
        with torch.no_grad():               # grad mode off: nothing needs a gradient
            assert not CV._fp8_train(conv, x)


@pytest.mark.parametrize("c_in,c_out,ok", [
    (32, 32, True), (32, 64, True), (64, 96, True), (96, 1024, True), (1024, 1024, True),
    (384, 256, True), (32, 16, False), (32, 48, False), (48, 64, False), (16, 64, False),
    (32, 1040, False), (1056, 32, False), (3, 32, False), (4, 64, False)],
    ids=lambda v: str(v))
def test_grid_both_ways(c_in, c_out, ok):
    """c_in -> c_out for the forward and c_out -> c_in for the dgrad: both multiples of 32, at most
    1024.  The stem (c_in <= 4) is off the grid whether or not its input needs a gradient."""
    assert (B.fp8_supported(c_in, c_out) and B.fp8_supported(c_out, c_in)) == ok
    conv = _conv(c_in, c_out, kernel_size=5 if c_in <= 4 else 3)
    with ME.fp8_training():
        assert CV._fp8_train(conv, _x(c_in)) == ok
        assert CV._fp8_train(conv, _x(c_in, grad=False)) == ok      # the kernel needs one


def test_matrix_product_layer_is_not_selected():
    with ME.fp8_training():
        conv = _conv(kernel_size=1)
        assert conv.use_mm and not CV._fp8_train(conv, _x())
        conv = _conv(kernel_size=1, stride=2)        # K = 1 with a stride runs the kernels
        assert not conv.use_mm and CV._fp8_train(conv, _x())


@pytest.mark.parametrize("dtype,ok", [(torch.float32, True), (torch.bfloat16, True),
                                      (torch.float16, True), (torch.float64, False)],
                         ids=["fp32", "bf16", "fp16", "fp64"])
def test_feature_dtype(dtype, ok):
    with ME.fp8_training():
        assert CV._fp8_train(_conv(), _x(dtype=dtype)) == ok


@pytest.mark.parametrize("cls", [ME.MinkowskiConvolution, ME.MinkowskiConvolutionTranspose,
                                 ME.MinkowskiGenerativeConvolutionTranspose])
def test_all_three_layer_classes_are_selected(cls):
    with ME.fp8_training():
        assert CV._fp8_train(_conv(kernel_size=2, stride=2, cls=cls), _x())


def test_other_layers_have_no_fp8_route():
    """Channel-wise convolution, pooling and normalisation never consult the rule: their
    modules take no fp8 argument and run as outside the block."""
    for cls in (ME.MinkowskiChannelwiseConvolution, ME.MinkowskiMaxPooling, ME.MinkowskiBatchNorm):
        assert not issubclass(cls, CV.MinkowskiConvolutionBase)


# ---- the e5m2 scale formula -----------------------------------------------------------------------
def e5m2_scales(amax):
    """(scale, inv) by the kernels' formula, in fp32 (numpy rounds fp32 divisions to nearest)."""
    amax = np.float32(amax)
    if amax == 0:
        return np.float32(1), np.float32(1)
    with np.errstate(over="ignore"):
        inv = np.float32(E5M2_MAX) / amax
    if np.isinf(inv):
        return np.float32(1) / FLT_MAX, FLT_MAX
    return amax / np.float32(E5M2_MAX), inv


@pytest.mark.parametrize("amax", [0.0, 1.0, 1.75, 3e-3, 57344.0, 1e30, FLT_MAX, 1e-30,
                                  np.float32(E5M2_MAX) / FLT_MAX, 1.5e-34, 1e-38, 1e-45])
def test_e5m2_scales_against_float64(amax):
    """scale and inv are the fp32 roundings of the float64 quotients, except at amax = 0 (both 1)
    and where 57344 / amax overflows fp32 (inv = FLT_MAX, scale = 1 / FLT_MAX)."""
    a = float(np.float32(amax))
    s, inv = e5m2_scales(a)
    if a == 0:
        assert (s, inv) == (1, 1)
        return
    q = E5M2_MAX / a
    if q >= float(FLT_MAX) * (1 + 2 ** -25):      # rounds to inf in fp32
        assert inv == FLT_MAX and s == np.float32(1 / float(FLT_MAX))
        assert float(s) * float(inv) == pytest.approx(1, rel=2 ** -23)
        return
    assert inv == np.float32(q) and s == np.float32(a / E5M2_MAX)
    assert abs(float(s) * float(inv) - 1) <= 2 ** -22        # q * scale approximates x


# ---- a stub library -------------------------------------------------------------------------------
def _f32(ptr, n):
    return np.ctypeslib.as_array((ctypes.c_float * n).from_address(ptr))


class _Stub:
    """Records every call; the e4m3 packings write their scales, the quantisations fixed scales."""

    def __init__(self, calls, real):
        self.calls, self.real = calls, real

    def __getattr__(self, name):
        def fn(*args):
            if name == "meb200_conv_fp8_supported":
                return self.real.meb200_conv_fp8_supported(*args)
            if name == "meb200_quantize_e4m3_workspace_bytes":
                return 16
            if name == "meb200_conv_pack_weights_e4m3":
                _f32(args[5], args[3])[:] = 0.125
            elif name == "meb200_conv_pack_weights_e4m3_dgrad":
                _f32(args[5], args[2])[:] = 0.0625
            elif name == "meb200_quantize_e4m3":
                _f32(args[5], 2)[:] = [0.5, 2.0]
            elif name == "meb200_quantize_e5m2":
                _f32(args[5], 2)[:] = [0.25, 4.0]
            self.calls.append((name, args))
            return 0
        return fn


class _Map:
    K, n_in, n_out, n_pairs = 27, 10, 12, 40
    out_nbr = in_nbr = out_order = in_order = None


class _TMap(_Map):
    """A map with (fake) tables, so that the pointers passed can be told apart."""

    def __init__(self):
        self.out_nbr = torch.zeros(27, 12, dtype=torch.int32)
        self.in_nbr = torch.zeros(27, 10, dtype=torch.int32)
        self.out_order = torch.zeros(8, dtype=torch.int32)
        self.in_order = torch.zeros(8, dtype=torch.int32)


@pytest.fixture
def stub(monkeypatch):
    from minkowskiengine_b200 import _lib
    real = _lib.load()
    calls = []
    monkeypatch.setattr(_lib, "load", lambda: _Stub(calls, real))
    monkeypatch.setattr(_lib, "current_stream", lambda: None)
    for name in ("_QUANT_WS", "_PACKED", "_PACK_TABLES"):
        monkeypatch.setattr(B, name, {})
    saved = torch.backends.cuda.matmul.fp32_precision
    torch.backends.cuda.matmul.fp32_precision = "ieee"
    yield calls
    torch.backends.cuda.matmul.fp32_precision = saved


def _named(calls, name):
    return [c for c in calls if c[0] == name]


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
def test_forward_gets_e4m3_operands(stub, dtype):
    """The forward of a selected layer is the e4m3 forward without an epilogue."""
    x, w = torch.randn(10, 32).to(dtype), torch.randn(27, 32, 64)
    y = B._conv_forward(x, w, _Map(), fp8=True)
    assert y.dtype == dtype and y.shape == (12, 64)
    (_, qa), = _named(stub, "meb200_quantize_e4m3")
    (_, fa), = _named(stub, "meb200_conv_forward_fp8")
    assert qa[0] == x.data_ptr() and fa[0] == qa[4] and fa[1] == qa[5]
    assert not _named(stub, "meb200_conv_forward") and not _named(stub, "meb200_conv_pack_weights")


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
def test_dgrad_gets_e5m2_operands(stub, dtype):
    km = _TMap()
    x, w = torch.randn(10, 32).to(dtype), torch.randn(27, 32, 64)
    g = torch.randn(12, 64).to(dtype)
    gi, gw = B._conv_backward(x, g, w, km, need_in=True, need_w=False, fp8=True)
    assert gw is None and gi.shape == (10, 32) and gi.dtype == dtype
    (_, pk), = _named(stub, "meb200_conv_pack_weights_e4m3_dgrad")
    (_, qa), = _named(stub, "meb200_quantize_e5m2")
    (_, da), = _named(stub, "meb200_conv_dgrad_fp8")
    assert pk[1:4] == (27, 32, 64)
    assert qa[0] == g.data_ptr() and qa[1] == ME._lib.dtype_code(dtype) and qa[2:4] == (12, 64)
    assert qa[6] is not None                                          # the shared workspace
    assert da[0] == qa[4] and da[1] == qa[5]                          # e5m2 bytes and scale
    assert da[2:4] == (12, 64) and da[4] == pk[4] and da[5] == pk[5]  # packed weights, w_scale
    assert da[6:8] == (27, 32) and da[8] == km.in_nbr.data_ptr() and da[9] == 10
    assert da[10] == gi.data_ptr() and da[11] == ME._lib.dtype_code(dtype)
    assert da[12] == km.in_order.data_ptr()
    assert not _named(stub, "meb200_conv_backward") and not _named(stub, "meb200_conv_pack_weights")
    assert not _named(stub, "meb200_quantize_e4m3")


def _wgrad_args(a):
    """The arguments of meb200_conv_backward a weight gradient reads (not its output pointer)."""
    return (a[0], a[2], a[3], a[4], a[6], a[7], a[8], a[10], a[12], a[14], a[15], a[16], a[17],
            a[19])


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
def test_wgrad_arguments_are_those_outside_the_block(stub, dtype):
    km = _TMap()
    x, w, g = torch.randn(10, 32).to(dtype), torch.randn(27, 32, 64), torch.randn(12, 64).to(dtype)
    B._conv_backward(x, g, w, km, need_in=False, need_w=True)                 # outside, wgrad only
    B._conv_backward(x, g, w, km, need_in=True, need_w=True)                  # outside, both
    n0 = len(stub)
    gi, gw = B._conv_backward(x, g, w, km, need_in=True, need_w=True, fp8=True)
    assert gi is not None and gw.shape == (27, 32, 64)
    alone, both, fp8 = [c[1] for c in _named(stub, "meb200_conv_backward")]
    assert _wgrad_args(fp8) == _wgrad_args(alone) == _wgrad_args(both)
    assert fp8[5] is None and fp8[9] is None and fp8[11] is None and fp8[20] is None   # no dgrad
    assert alone[5] is None                        # a wgrad-only call packs no w_cast ...
    assert both[5] is not None                     # ... the call with a dgrad reads one
    packs = _named(stub, "meb200_conv_pack_weights")
    assert len(packs) == (0 if dtype == torch.float32 else 1)      # (exact fp32 packs nothing)
    assert not _named(stub[n0:], "meb200_conv_pack_weights")
    # the dgrad launched before the wgrad, on the same gradient
    names = [c[0] for c in stub[n0:]]
    assert names.index("meb200_conv_dgrad_fp8") < names.index("meb200_conv_backward")


def test_wgrad_only_call_packs_nothing(stub):
    """A layer whose input needs no gradient: the wgrad alone, no e5m2, no packs."""
    x, w, g = torch.randn(10, 32).bfloat16(), torch.randn(27, 32, 64), torch.randn(12, 64).bfloat16()
    gi, gw = B._conv_backward(x, g, w, _TMap(), need_in=False, need_w=True, fp8=True)
    assert gi is None and gw is not None
    assert not [c for c in stub if c[0].startswith(("meb200_conv_pack", "meb200_quant"))]
    assert not _named(stub, "meb200_conv_dgrad_fp8")
    (_, a), = _named(stub, "meb200_conv_backward")
    assert a[5] is None and a[9] is None and a[11] is None


def test_each_pack_once_per_parameter_version(stub):
    w = torch.randn(27, 32, 64)
    x, g = torch.randn(10, 32).bfloat16(), torch.randn(12, 64).bfloat16()
    for _ in range(3):
        B._conv_forward(x, w, _Map(), fp8=True)
        B._conv_backward(x, g, w, _TMap(), need_in=True, need_w=True, fp8=True)
    assert len(_named(stub, "meb200_conv_pack_weights_e4m3")) == 1
    assert len(_named(stub, "meb200_conv_pack_weights_e4m3_dgrad")) == 1
    assert len(_named(stub, "meb200_quantize_e5m2")) == 3             # dOut: every step
    assert not _named(stub, "meb200_conv_pack_weights")
    with torch.no_grad():
        w.sub_(0.1)                                                   # the optimizer stepped
    B._conv_forward(x, w, _Map(), fp8=True)
    B._conv_backward(x, g, w, _TMap(), need_in=True, need_w=True, fp8=True)
    assert len(_named(stub, "meb200_conv_pack_weights_e4m3")) == 2
    assert len(_named(stub, "meb200_conv_pack_weights_e4m3_dgrad")) == 2
    # the dgrad pack is its own entry of the cache, beside the forward's
    assert {e[3] for e in B._PACKED.values()} == {B.FP8, B.FP8_DGRAD}


def test_empty_maps_launch_no_dgrad(stub):
    class Empty(_Map):
        n_out = 0
    w = torch.randn(27, 32, 64)
    gi, _ = B._conv_backward(torch.randn(10, 32), torch.zeros(0, 64), w, Empty(), need_in=True,
                             need_w=False, fp8=True)
    assert gi.shape == (10, 32) and not gi.any()
    assert not _named(stub, "meb200_conv_dgrad_fp8") and not _named(stub, "meb200_quantize_e5m2")


def test_without_fp8_the_call_is_unchanged(stub):
    km = _TMap()
    x, w, g = torch.randn(10, 32).bfloat16(), torch.randn(27, 32, 64), torch.randn(12, 64).bfloat16()
    with ME.fp8_training():                       # the flag, not the context, picks the route
        B._conv_backward(x, g, w, km, need_in=True, need_w=True)
    (_, a), = _named(stub, "meb200_conv_backward")
    assert a[5] is not None and a[9] == km.in_nbr.data_ptr() and a[20] == km.in_order.data_ptr()
    assert not _named(stub, "meb200_conv_dgrad_fp8") and not _named(stub, "meb200_quantize_e5m2")
    assert not _named(stub, "meb200_conv_pack_weights_e4m3_dgrad")


def test_functions_carry_the_decision(monkeypatch):
    """The layer decides once in its forward and hands the flag to the autograd Function as one
    extra non-tensor argument; the backward passes it to the native backward."""
    seen = {}

    def fwd(*a, fp8=False, **k):
        seen["fwd"] = fp8
        return torch.zeros(12, a[1].shape[2], dtype=a[0].dtype)

    def bwd(*a, fp8=False, need_in=True, need_w=True, **k):
        seen["bwd"] = (fp8, need_in, need_w)
        return (torch.zeros_like(a[0]) if need_in else None,
                torch.zeros_like(a[2]) if need_w else None)

    monkeypatch.setattr(B, "ConvolutionForwardGPU", fwd)
    monkeypatch.setattr(B, "ConvolutionBackwardGPU", bwd)

    class Mgr:
        _manager = None

    for flag in (False, True):
        x = torch.randn(10, 32, requires_grad=True)
        k = torch.randn(27, 32, 64, requires_grad=True)
        y = CV.MinkowskiConvolutionFunction.apply(x, k, ME.KernelGenerator(3, dimension=3), None,
                                                  object(), object(), Mgr(), flag)
        y.sum().backward()
        assert seen == {"fwd": flag, "bwd": (flag, True, True)}
