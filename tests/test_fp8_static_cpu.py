"""Static fp8 scales without a GPU: which layers Fp8Calibration observes and links (case by case),
the calls the host makes inside fp8_inference(calibration) (a stub of the native library that
computes the amax and the scales as the kernels do), the state_dict round trip, stale shadows, and
the context rules.  The layers run on CPU stand-ins for the sparse tensors: the native forward is
replaced by a function that records what it was handed."""
import ctypes
import threading
import types

import numpy as np
import pytest
import torch

import minkowskiengine_b200 as ME
from minkowskiengine_b200 import backend as B
from minkowskiengine_b200 import convolution as CV
from minkowskiengine_b200 import fp8_calibration as FC


def _scales(amax):
    """(scale, inv) by the kernels' formula, in fp32."""
    amax = np.float32(amax)
    if amax == 0:
        return np.float32(1), np.float32(1)
    with np.errstate(over="ignore"):
        inv = np.float32(448) / amax
    if np.isinf(inv):
        big = np.finfo(np.float32).max
        return np.float32(1) / big, big
    return amax / np.float32(448), inv


def _f32(ptr, n):
    return np.ctypeslib.as_array((ctypes.c_float * n).from_address(ptr))


class _Stub:
    """Records every call.  On CPU tensors it computes what the static-scale entries write: the
    running amax, the scales, and (as a marker) the conversion's output bytes = 7."""

    def __init__(self, calls, real):
        self.calls, self.real = calls, real

    def __getattr__(self, name):
        def fn(*args):
            if name == "meb200_conv_fp8_supported":
                return self.real.meb200_conv_fp8_supported(*args)
            if name == "meb200_quantize_e4m3_workspace_bytes":
                return 16
            if name == "meb200_amax_accumulate":
                x, dt, n, c, a = args[:5]
                assert dt == ME._lib.F32
                v = _f32(x, n * c)
                m = np.abs(v[np.isfinite(v)]).max(initial=0)
                _f32(a, 1)[0] = max(_f32(a, 1)[0], m)
            elif name == "meb200_e4m3_scales":
                _f32(args[1], 2)[:] = _scales(_f32(args[0], 1)[0])
            elif name == "meb200_quantize_e4m3":
                _f32(args[5], 2)[:] = [0.5, 2.0]
            elif name == "meb200_quantize_e4m3_static":
                n, c = args[2], args[3]
                ctypes.memset(args[4], 7, n * c)
            elif name == "meb200_conv_pack_weights_e4m3":
                _f32(args[5], args[3])[:] = 1
            self.calls.append((name, args))
            return 0
        return fn


@pytest.fixture
def stub(monkeypatch):
    from minkowskiengine_b200 import _lib
    real = _lib.load()
    calls = []
    monkeypatch.setattr(_lib, "load", lambda: _Stub(calls, real))
    monkeypatch.setattr(_lib, "current_stream", lambda: None)
    for name in ("_QUANT_WS", "_PACKED", "_PACK_TABLES"):
        monkeypatch.setattr(B, name, {})
    yield calls


def _named(calls, name):
    return [c for c in calls if c[0] == name]


class _Map:
    K, n_in, n_out, n_pairs = 27, 6, 6, 40
    out_nbr = in_nbr = out_order = in_order = None


class _ST(ME.SparseTensor):
    """A CPU stand-in for a SparseTensor: its features and nothing else."""

    def __init__(self, feats, coordinate_map_key=None, coordinate_manager=None):
        self._F = feats
        self._manager = types.SimpleNamespace(_manager=None)
        self._D = 3

    @property
    def coordinate_map_key(self):
        return None


@pytest.fixture
def layers(monkeypatch, stub):
    """The layers' forwards on CPU: the native forward calls _conv_forward_impl with the stub
    library and a map of 6 rows; the batch norm check passes."""
    def forward(in_feat, kernel, *a, epilogue=None, fp8=False, act=None, shadow=None):
        return B._conv_forward_impl(in_feat, kernel, _Map(), epilogue=epilogue, fp8=fp8, act=act,
                                    shadow=shadow)

    def plain(in_feat, kernel, *a, **k):
        return torch.zeros(6, kernel.shape[2])

    monkeypatch.setattr(B, "ConvolutionForwardGPU", forward)
    monkeypatch.setattr(B, "ConvolutionTransposeForwardGPU", forward)
    monkeypatch.setattr(CV._C, "ConvolutionForwardGPU", forward)
    monkeypatch.setattr(CV.MinkowskiConvolutionFunction, "forward",
                        staticmethod(lambda ctx, f, k, *a: plain(f, k)))
    monkeypatch.setattr(CV, "SparseTensor", _ST)
    monkeypatch.setattr(CV, "_get_coordinate_map_key", lambda *a, **k: None)
    monkeypatch.setattr(CV, "_output_key", lambda conv, input: "out")
    monkeypatch.setattr(CV, "_native_ok", lambda bn, x: True)
    monkeypatch.setattr(B, "_is_stem", lambda kernel, dtype: False)
    return stub


class _Net(torch.nn.Module):
    """a -> b -> c, all 32 -> 32 (on the e4m3 grid), with eval batch norms for the fused calls."""

    def __init__(self, c_a=32):
        super().__init__()
        self.a = ME.MinkowskiConvolution(c_a, 32, kernel_size=3, dimension=3)
        self.b = ME.MinkowskiConvolution(32, 32, kernel_size=3, dimension=3)
        self.c = ME.MinkowskiConvolution(32, 32, kernel_size=3, dimension=3)
        self.na = ME.MinkowskiBatchNorm(32).eval()
        self.nb = ME.MinkowskiBatchNorm(32).eval()
        self.nc = ME.MinkowskiBatchNorm(32).eval()


def _x(c=32, scale=1.0, seed=0):
    g = torch.Generator().manual_seed(seed)
    return _ST(torch.randn(6, c, generator=g) * scale)


# ---- observing: amax and links -----------------------------------------------------------------
def test_direct_link_and_running_amax(layers):
    net = _Net()
    calib = ME.Fp8Calibration(net)
    xs = [_x(scale=s, seed=i) for i, s in enumerate((1.0, 3.0, 2.0))]
    with torch.no_grad(), calib.observe():
        for x in xs:
            y = ME.fused_conv_bn_relu(net.a, net.na, x)
            ME.fused_conv_bn_relu(net.b, net.nb, y)
    sd = calib.state_dict()
    want = max(float(x.F.abs().max()) for x in xs)
    assert float(sd["a"]["amax"]) == np.float32(want)
    assert sd["a"]["feeds"] == ["b"] and sd["b"]["feeds"] == []
    assert sd["b"]["amax"] is not None          # (of whatever the stub's forward left)
    # one accumulation per selected layer and batch, no conversion, no dynamic quantisation
    assert len(_named(layers, "meb200_amax_accumulate")) == 6
    assert not _named(layers, "meb200_quantize_e4m3")
    assert not _named(layers, "meb200_quantize_e4m3_static")


def test_observe_runs_the_layers_as_outside_fp8(layers):
    net = _Net()
    calib = ME.Fp8Calibration(net)
    with torch.no_grad(), calib.observe():
        ME.fused_conv_bn_relu(net.a, net.na, _x())
        net.b(_x())
    assert not _named(layers, "meb200_conv_forward_fp8")
    assert not _named(layers, "meb200_conv_forward_fp8_q")
    assert _named(layers, "meb200_conv_forward")          # the fused call's usual route


@pytest.mark.parametrize("how", ["new_tensor", "features_op"])
def test_a_new_object_breaks_the_link(layers, how):
    net = _Net()
    calib = ME.Fp8Calibration(net)
    with torch.no_grad(), calib.observe():
        y = ME.fused_conv_bn_relu(net.a, net.na, _x())
        y2 = _ST(y.F) if how == "new_tensor" else _ST(torch.relu(y.F))
        ME.fused_conv_bn_relu(net.b, net.nb, y2)
    sd = calib.state_dict()
    assert "b" in sd and sd["b"]["amax"] is not None
    assert "a" not in sd or sd["a"]["feeds"] == []


def test_plain_layers_link(layers):
    """A MinkowskiConvolution the fp8 rule selects is a producer too (in fp8 it runs the e4m3
    route, which writes shadows)."""
    net = _Net()
    calib = ME.Fp8Calibration(net)
    with torch.no_grad(), calib.observe():
        net.c(net.b(net.a(_x())))
    sd = calib.state_dict()
    assert sd["a"]["feeds"] == ["b"] and sd["b"]["feeds"] == ["c"]


def test_one_producer_two_consumers(layers):
    net = _Net()
    calib = ME.Fp8Calibration(net)
    with torch.no_grad(), calib.observe():
        y = ME.fused_conv_bn_relu(net.a, net.na, _x())
        ME.fused_conv_bn_relu(net.b, net.nb, y)
        ME.fused_conv_bn_relu(net.c, net.nc, y)
    assert calib.state_dict()["a"]["feeds"] == ["b", "c"]


def test_layers_off_the_rule_are_not_observed(layers):
    """The stem (c_in 4, off the e4m3 grid) is a producer but no consumer; a layer whose kernel
    needs a gradient is neither; layers of another model are not bound."""
    net = _Net(c_a=4)
    calib = ME.Fp8Calibration(net)
    other = ME.MinkowskiConvolution(32, 32, kernel_size=3, dimension=3)
    with torch.no_grad(), calib.observe():
        y = ME.fused_conv_bn_relu(net.a, net.na, _x(c=4))
        ME.fused_conv_bn_relu(net.b, net.nb, y)
        other(_x())
    sd = calib.state_dict()
    assert sd["a"] == {"amax": None, "feeds": ["b"]} and sd["b"]["amax"] is not None
    assert len(_named(layers, "meb200_amax_accumulate")) == 1
    net.b.kernel.requires_grad_(True)
    calib2 = ME.Fp8Calibration(net)
    with calib2.observe():                  # grad mode on, the kernel needs a gradient
        net.b(_x())
    assert calib2.state_dict() == {}


# ---- inference with a calibration --------------------------------------------------------------
def _calibrated(layers, feeds=True):
    net = _Net()
    calib = ME.Fp8Calibration(net)
    with torch.no_grad(), calib.observe():
        y = ME.fused_conv_bn_relu(net.a, net.na, _x(scale=2.0))
        ME.fused_conv_bn_relu(net.b, net.nb, y if feeds else _ST(y.F.clone()))
    layers.clear()
    return net, calib


def test_static_input_and_shadow_arguments(layers):
    net, calib = _calibrated(layers)
    sd = calib.state_dict()
    x = _x()
    with torch.no_grad(), ME.fp8_inference(calib):
        y = ME.fused_conv_bn_relu(net.a, net.na, x)
        z = ME.fused_conv_bn_relu(net.b, net.nb, y)
    assert not _named(layers, "meb200_quantize_e4m3")            # no amax pass anywhere
    (_, qa), = _named(layers, "meb200_quantize_e4m3_static")     # a's input, at a's scale
    (_, fa), = _named(layers, "meb200_conv_forward_fp8_q")       # a writes b's shadow
    (_, fb), = _named(layers, "meb200_conv_forward_fp8")         # b reads it, writes none
    assert qa[0] == x.F.data_ptr() and qa[2:4] == (6, 32)
    a_scale = _f32(qa[5], 2)
    assert tuple(a_scale) == _scales(np.float32(sd["a"]["amax"]))
    assert fa[0] == qa[4] and fa[1] == qa[5]                     # a: the static bytes and scale
    q_shadow, s_shadow = fa[13], fa[14]
    assert tuple(_f32(s_shadow, 2)) == _scales(np.float32(sd["b"]["amax"]))
    assert fb[0] == q_shadow and fb[1] == s_shadow               # b: the shadow and its scale
    sh = FC.fresh_shadow(y)
    assert sh is not None and sh[0].data_ptr() == q_shadow and sh[0].shape == (6, 32)
    assert FC.fresh_shadow(z) is None
    # the scales are computed once per layer and reused
    n_scales = len(_named(layers, "meb200_e4m3_scales"))
    with torch.no_grad(), ME.fp8_inference(calib):
        ME.fused_conv_bn_relu(net.b, net.nb, ME.fused_conv_bn_relu(net.a, net.na, _x()))
    assert len(_named(layers, "meb200_e4m3_scales")) == n_scales == 2


def test_stale_shadow_is_ignored(layers):
    net, calib = _calibrated(layers)
    with torch.no_grad(), ME.fp8_inference(calib):
        y = ME.fused_conv_bn_relu(net.a, net.na, _x())
        assert FC.fresh_shadow(y) is not None
        y.F.mul_(2)                                             # modified in place
        assert FC.fresh_shadow(y) is None
        layers.clear()
        ME.fused_conv_bn_relu(net.b, net.nb, y)
    (_, qb), = _named(layers, "meb200_quantize_e4m3_static")    # b converts its input itself
    (_, fb), = _named(layers, "meb200_conv_forward_fp8")
    assert qb[0] == y.F.data_ptr() and fb[0] == qb[4]
    # replacing the features is stale too
    with torch.no_grad(), ME.fp8_inference(calib):
        y = ME.fused_conv_bn_relu(net.a, net.na, _x())
        y._F = y.F.clone()
        assert FC.fresh_shadow(y) is None


def test_unlinked_consumer_converts_with_its_static_scale(layers):
    net, calib = _calibrated(layers, feeds=False)
    assert calib.state_dict()["a"]["feeds"] == []
    with torch.no_grad(), ME.fp8_inference(calib):
        ME.fused_conv_bn_relu(net.b, net.nb, ME.fused_conv_bn_relu(net.a, net.na, _x()))
    assert len(_named(layers, "meb200_quantize_e4m3_static")) == 2
    assert not _named(layers, "meb200_conv_forward_fp8_q")
    assert not _named(layers, "meb200_quantize_e4m3")


def test_uncalibrated_layer_keeps_the_dynamic_path(layers):
    """c has no entry: its call is today's fp8_inference() call, shadow or not on its input."""
    net, calib = _calibrated(layers)
    x = _x()
    runs = []
    for c in (None, calib):
        layers.clear()
        B._PACKED.clear()
        with torch.no_grad(), ME.fp8_inference(c):
            ME.fused_conv_bn_relu(net.c, net.nc, x)
        runs.append([n for n, _ in layers])
        (_, qa), = _named(layers, "meb200_quantize_e4m3")
        assert qa[:4] == (x.F.data_ptr(), ME._lib.F32, 6, 32)
    assert runs[0] == runs[1] == ["meb200_conv_pack_weights_e4m3", "meb200_quantize_e4m3",
                                  "meb200_conv_forward_fp8"]


def test_producer_off_the_e4m3_grid_writes_its_shadow_on_the_16_bit_route(layers):
    """A bf16 stem-like producer (c_in 4) runs meb200_conv_forward_q with the consumer's scale;
    the route returns MEB200_ERR_UNSUPPORTED for fp32 features (no shadow: the consumer
    converts)."""
    net = _Net(c_a=4).to(torch.float32)
    calib = ME.Fp8Calibration(net)
    with torch.no_grad(), calib.observe():
        ME.fused_conv_bn_relu(net.b, net.nb, ME.fused_conv_bn_relu(net.a, net.na, _x(c=4)))
    layers.clear()
    xb = _ST(torch.randn(6, 4).bfloat16())
    with torch.no_grad(), ME.fp8_inference(calib):
        y = ME.fused_conv_bn_relu(net.a, net.na, xb)
    (_, fa), = _named(layers, "meb200_conv_forward_q")
    assert fa[1] == ME._lib.BF16 and fa[14] == FC.fresh_shadow(y)[0].data_ptr()
    assert not _named(layers, "meb200_conv_forward")


def test_observe_inside_fp8_inference_raises():
    calib = ME.Fp8Calibration(_Net())
    with ME.fp8_inference():
        with pytest.raises(RuntimeError):
            with calib.observe():
                pass
    with calib.observe():
        with pytest.raises(RuntimeError):
            with ME.fp8_inference(calib):
                pass
    assert B.fp8_observer() is None and not B.fp8_enabled()


def test_context_nesting_and_thread_locality():
    calib = ME.Fp8Calibration(_Net())
    seen = []
    with ME.fp8_inference(calib):
        assert B.fp8_calibration() is calib
        with ME.fp8_inference():
            assert B.fp8_calibration() is None and B.fp8_enabled()
        assert B.fp8_calibration() is calib
        t = threading.Thread(target=lambda: seen.append((B.fp8_enabled(), B.fp8_calibration(),
                                                         B.fp8_observer())))
        t.start()
        t.join()
    assert seen == [(False, None, None)]
    assert B.fp8_calibration() is None and not B.fp8_enabled()
    with calib.observe():
        t = threading.Thread(target=lambda: seen.append(B.fp8_observer()))
        t.start()
        t.join()
        assert B.fp8_observer() is calib
    assert seen[-1] is None


def test_state_dict_round_trip(layers, tmp_path):
    net, calib = _calibrated(layers)
    sd = calib.state_dict()
    path = tmp_path / "calib.pt"
    torch.save(sd, path)
    other = _Net()
    calib2 = ME.Fp8Calibration(other)
    calib2.load_state_dict(torch.load(path))
    sd2 = calib2.state_dict()
    assert sd2.keys() == sd.keys()
    for k in sd:
        assert sd2[k]["feeds"] == sd[k]["feeds"]
        assert (sd2[k]["amax"] is None) == (sd[k]["amax"] is None)
        if sd[k]["amax"] is not None:
            assert sd2[k]["amax"].dtype == torch.float32
            assert sd2[k]["amax"].view(torch.int32) == sd[k]["amax"].view(torch.int32)
    with pytest.raises(KeyError):
        ME.Fp8Calibration(torch.nn.Sequential()).load_state_dict(sd)
