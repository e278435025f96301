"""fp8 inference without a GPU: which layers ME.fp8_inference() runs on e4m3 operands (case by
case), how the weight scale, the conv bias and eval batch norm fold into the epilogue (against
float64), the arguments the host hands the library (a stub that computes the scales the way the
kernels do), and the launch configuration of csrc/tc_config.h at an element size of one byte."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

import minkowskiengine_b200 as ME
from minkowskiengine_b200 import backend as B
from minkowskiengine_b200 import convolution as CV

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _conv(c_in=32, c_out=64, kernel_size=3, stride=1, bias=False, cls=ME.MinkowskiConvolution):
    return cls(c_in, c_out, kernel_size=kernel_size, stride=stride, bias=bias, dimension=3)


# ---- the selection rule -------------------------------------------------------------------------
def test_context_off_never_selects():
    conv = _conv()
    with torch.no_grad():
        assert not CV._fp8(conv, torch.randn(10, 32))
        with ME.fp8_inference():
            assert CV._fp8(conv, torch.randn(10, 32))
        assert not CV._fp8(conv, torch.randn(10, 32))


def test_context_nests_and_survives_exceptions():
    with ME.fp8_inference():
        with ME.fp8_inference():
            assert B.fp8_enabled()
        assert B.fp8_enabled()
    assert not B.fp8_enabled()
    with pytest.raises(ValueError):
        with ME.fp8_inference():
            raise ValueError
    assert not B.fp8_enabled()


def test_context_is_thread_local():
    import threading
    seen = []
    with ME.fp8_inference():
        t = threading.Thread(target=lambda: seen.append(B.fp8_enabled()))
        t.start()
        t.join()
        assert B.fp8_enabled()
    assert seen == [False]


@pytest.mark.parametrize("which", ["input", "kernel", "bias"])
def test_a_tensor_needing_a_gradient_does_not_select(which):
    conv = _conv(bias=True)
    for p in conv.parameters():
        p.requires_grad_(False)
    x = torch.randn(10, 32)
    t = {"input": x, "kernel": conv.kernel, "bias": conv.bias}[which]
    with ME.fp8_inference():
        assert CV._fp8(conv, x)
        t.requires_grad_(True)
        assert not CV._fp8(conv, x)
        with torch.no_grad():               # grad mode off: nothing needs a gradient
            assert CV._fp8(conv, x)


@pytest.mark.parametrize("c_in,c_out,ok", [
    (32, 16, True), (32, 64, True), (64, 96, True), (96, 1024, True), (384, 256, True),
    (16, 64, False), (48, 64, False), (33, 64, False), (32, 40, False), (32, 8, False),
    (32, 1040, False), (3, 32, False), (4, 64, False)],
    ids=lambda v: str(v))
def test_grid(c_in, c_out, ok):
    """c_in in whole 32-byte k-steps, c_out in multiples of 16 up to 1024; the stem (c_in <= 4) is
    off the grid."""
    assert B.fp8_supported(c_in, c_out) == ok
    conv = _conv(c_in, c_out, kernel_size=5 if c_in <= 4 else 3)
    with torch.no_grad(), ME.fp8_inference():
        assert CV._fp8(conv, torch.randn(10, c_in)) == ok


def test_matrix_product_layer_is_not_selected():
    with torch.no_grad(), ME.fp8_inference():
        conv = _conv(kernel_size=1)
        assert conv.use_mm and not CV._fp8(conv, torch.randn(10, 32))
        conv = _conv(kernel_size=1, stride=2)        # K = 1 with a stride runs the kernels
        assert not conv.use_mm and CV._fp8(conv, torch.randn(10, 32))


@pytest.mark.parametrize("dtype,ok", [(torch.float32, True), (torch.bfloat16, True),
                                      (torch.float16, True), (torch.float64, False)],
                         ids=["fp32", "bf16", "fp16", "fp64"])
def test_feature_dtype(dtype, ok):
    with torch.no_grad(), ME.fp8_inference():
        assert CV._fp8(_conv(), torch.randn(10, 32).to(dtype)) == ok


@pytest.mark.parametrize("cls", [ME.MinkowskiConvolutionTranspose,
                                 ME.MinkowskiGenerativeConvolutionTranspose])
def test_transposed_layers_are_selected(cls):
    with torch.no_grad(), ME.fp8_inference():
        assert CV._fp8(_conv(kernel_size=2, stride=2, cls=cls), torch.randn(10, 32))


# ---- a stub library that computes the scales as the kernels do ----------------------------------
def _f32(ptr, n):
    return np.ctypeslib.as_array((ctypes.c_float * n).from_address(ptr)) if n else np.zeros(0, np.float32)


def _scales(amax):
    """(scale, inv) by the kernels' formula, in fp32 (numpy rounds fp32 divisions to nearest)."""
    amax = np.float32(amax)
    if amax == 0:
        return np.float32(1), np.float32(1)
    with np.errstate(over="ignore"):
        inv = np.float32(448) / amax
    if np.isinf(inv):
        big = np.finfo(np.float32).max
        return np.float32(1) / big, big
    return amax / np.float32(448), inv


class _Stub:
    """Records every call; the e4m3 weight packing writes w_scale and the quantisation the
    activation scales (the bytes are not modelled), the fp8 forward's epilogue is read during the
    call."""

    def __init__(self, calls, real):
        self.calls, self.real = calls, real

    def __getattr__(self, name):
        def fn(*args):
            rec = None
            if name == "meb200_conv_fp8_supported":
                return self.real.meb200_conv_fp8_supported(*args)
            if name == "meb200_quantize_e4m3_workspace_bytes":
                return 16
            if name == "meb200_conv_pack_weights_e4m3":
                w, K, c_in, c_out, _, ws_ptr, _ = args
                W = _f32(w, K * c_in * c_out).reshape(K * c_in, c_out)
                _f32(ws_ptr, c_out)[:] = [_scales(a)[0] for a in np.abs(W).max(0)]
            elif name == "meb200_quantize_e4m3":
                _f32(args[5], 2)[:] = [0.5, 2.0]
            elif name == "meb200_conv_forward_fp8":
                e = B._ConvEpilogue.from_address(args[-2])
                c_out = args[6]
                rec = (_f32(e.scale, c_out).copy(), _f32(e.shift, c_out).copy(), e.residual, e.relu)
            self.calls.append((name, args, rec))
            return 0
        return fn


class _Map:
    K, n_in, n_out, n_pairs = 27, 10, 12, 40
    out_nbr = in_nbr = out_order = in_order = None


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


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
def test_forward_arguments(stub, dtype):
    x, w = torch.randn(10, 32).to(dtype), torch.randn(27, 32, 64)
    res = torch.randn(12, 64).to(dtype)
    scale, shift = torch.rand(64) + 0.5, torch.randn(64)
    y = B._conv_forward(x, w, _Map(), epilogue=(scale, shift, res, True), fp8=True)
    assert y.shape == (12, 64) and y.dtype == dtype
    (_, pk, _), = _named(stub, "meb200_conv_pack_weights_e4m3")
    (_, qa, _), = _named(stub, "meb200_quantize_e4m3")
    (_, fa, rec), = _named(stub, "meb200_conv_forward_fp8")
    assert not _named(stub, "meb200_conv_forward")
    assert qa[0] == x.data_ptr() and qa[1] == ME._lib.dtype_code(dtype) and qa[2:4] == (10, 32)
    assert qa[6] is not None                                   # the workspace
    assert fa[0] == qa[4] and fa[1] == qa[5]                   # the quantised features and scale
    assert fa[2:4] == (10, 32) and fa[4] == pk[4] and fa[5:7] == (27, 64)
    assert fa[8] == 12 and fa[9] == y.data_ptr() and fa[10] == ME._lib.dtype_code(dtype)
    assert rec[2] == res.data_ptr() and rec[3] == 1
    # epi.scale = w_scale * scale (one fp32 rounding), epi.shift = shift
    w_scale = np.array([_scales(a)[0] for a in w.abs().reshape(-1, 64).max(0).values.numpy()],
                       np.float32)
    assert np.array_equal(rec[0], w_scale * scale.numpy())
    assert np.array_equal(rec[1], shift.numpy())


def test_plain_layer_epilogue(stub):
    """No epilogue: the scale is the weight scale alone and the shift zero."""
    w = torch.randn(27, 32, 16)
    B._conv_forward(torch.randn(10, 32), w, _Map(), fp8=True)
    (_, _, rec), = _named(stub, "meb200_conv_forward_fp8")
    assert np.array_equal(rec[0], np.array([_scales(a)[0] for a in
                                            w.abs().reshape(-1, 16).max(0).values.numpy()], np.float32))
    assert not rec[1].any() and rec[2] is None and rec[3] == 0


def test_weights_are_packed_once_per_version(stub):
    w = torch.randn(27, 32, 64)
    for _ in range(3):
        B._conv_forward(torch.randn(10, 32), w, _Map(), fp8=True)
    assert len(_named(stub, "meb200_conv_pack_weights_e4m3")) == 1
    assert len(_named(stub, "meb200_quantize_e4m3")) == 3          # the features: every call
    with torch.no_grad():
        w.mul_(2)                                                  # modified in place
    B._conv_forward(torch.randn(10, 32), w, _Map(), fp8=True)
    assert len(_named(stub, "meb200_conv_pack_weights_e4m3")) == 2
    # the bf16 packing of the same tensor is a separate entry of the same cache
    saved = torch.backends.cuda.matmul.fp32_precision
    torch.backends.cuda.matmul.fp32_precision = "ieee"
    try:
        B._conv_forward(torch.randn(10, 32).bfloat16(), w, _Map())
        B._conv_forward(torch.randn(10, 32), w, _Map(), fp8=True)
    finally:
        torch.backends.cuda.matmul.fp32_precision = saved
    assert len(_named(stub, "meb200_conv_pack_weights_e4m3")) == 2
    assert len(_named(stub, "meb200_conv_pack_weights")) == 1


def test_without_fp8_the_call_is_unchanged(stub):
    with ME.fp8_inference():
        B._conv_forward(torch.randn(10, 32).bfloat16(), torch.randn(27, 32, 64), _Map())
    assert _named(stub, "meb200_conv_forward")
    assert not _named(stub, "meb200_quantize_e4m3") and not _named(stub, "meb200_conv_forward_fp8")


@pytest.mark.parametrize("affine", [True, False], ids=["affine", "no_affine"])
@pytest.mark.parametrize("bias", [False, True], ids=["no_bias", "bias"])
def test_folding_against_float64(stub, affine, bias):
    """fused_conv_bn_relu's epilogue on e4m3: scale = w_scale * bn_scale, shift = the batch norm's
    shift with the conv bias folded in.  y = fma(acc * a_scale, scale, shift) is the float64
    composition a_scale * w_scale * acc -> + bias -> eval batch norm within a few fp32 roundings."""
    from minkowskiengine_b200.normalization import _eval_scale_shift
    g = torch.Generator().manual_seed(5)
    C = 48
    bn = torch.nn.BatchNorm1d(C, eps=1e-3, affine=affine).eval()
    bn.running_mean.copy_(torch.randn(C, generator=g))
    bn.running_var.copy_(torch.rand(C, generator=g) * 4 + 0.01)
    if affine:
        with torch.no_grad():
            bn.weight.copy_(torch.randn(C, generator=g))
            bn.bias.copy_(torch.randn(C, generator=g))
    conv_bias = torch.randn(1, C, generator=g) if bias else None
    w = torch.randn(27, 32, C, generator=g)
    scale, shift = _eval_scale_shift(bn, conv_bias)
    B._conv_forward(torch.randn(10, 32), w, _Map(), epilogue=(scale, shift, None, False), fp8=True)
    (_, _, (e_scale, e_shift, _, _)), = _named(stub, "meb200_conv_forward_fp8")
    d = lambda t: t.detach().double()                                   # noqa: E731
    w_scale = d(w).abs().reshape(-1, C).max(0).values / 448
    invstd = 1 / torch.sqrt(d(bn.running_var) + bn.eps)
    s64 = invstd * (d(bn.weight) if affine else 1)
    b64 = d(bn.bias) if affine else torch.zeros(C, dtype=torch.float64)
    a_scale = 0.5                                                       # the stub's
    # e4m3 sums are integers times 2^-18 or so; take a spread of them
    acc = torch.randint(-2 ** 20, 2 ** 20, (200, C), generator=g).double() / 64
    deq = acc * a_scale * w_scale                                       # the dequantised conv
    want = (deq + (d(conv_bias) if bias else 0) - d(bn.running_mean)) * s64 + b64
    acc32 = (acc * a_scale).float()                                     # exact: power-of-two scale
    got = torch.addcmul(torch.from_numpy(e_shift).double(), acc32.double(),
                        torch.from_numpy(e_scale).double()).float().double()
    # roundings: w_scale (1), its product with the bn scale (1), the bn scale (<= 3), the fma (1),
    # and the shift's terms (as in test_conv_epilogue_cpu)
    mag = (deq * s64).abs() + (d(bn.running_mean) * s64).abs() + b64.abs()
    if bias:
        mag = mag + (d(conv_bias) * s64).abs()
    assert bool(((got - want).abs() <= 2 ** -20 * mag).all())


# ---- launch configuration at one byte per element -----------------------------------------------
SRC = r"""
#include <stdio.h>
#include <initializer_list>
#include "tc_config.h"
using namespace meb200::tc;
int main() {
  int bad = 0;
  const unsigned chans[] = {32, 64, 96, 128, 160, 192, 256, 384, 512};
  for (unsigned cr : chans) for (unsigned cc = 16; cc <= kMaxCols; cc += 16) {
    const unsigned w = fwd_stage_bytes(cr, 1);
    const unsigned smem = fwd_ring_bytes(w, cc);
    // an e4m3 row of cr channels: the stage width and ring of a bf16 row of cr / 2 channels
    const bool ok = (w == 128 || w == 64 || w == 32) && cr % w == 0 && smem <= kSmemLimit &&
                    (cr % 128 != 0 || w == 128) && w == fwd_stage_bytes(cr / 2, 2) &&
                    smem == fwd_smem_bytes(fwd_bk(cr / 2), cc);
    if (!ok) { printf("BAD cr=%u cc=%u width=%u smem=%u\n", cr, cc, w, smem); ++bad; }
  }
  for (unsigned cr : {8u, 16u, 24u, 40u, 48u, 80u})
    if (fwd_stage_bytes(cr, 1) != 0 && cr % 32 != 0) { printf("BAD: %u accepted\n", cr); ++bad; }
  if (fwd_stage_bytes(16, 1) != 0 || fwd_stage_bytes(48, 1) != 0) { printf("BAD partial k-step\n"); ++bad; }
  printf("bad=%d\n", bad);
  return bad != 0;
}
"""


def test_tc_config_one_byte_elements(tmp_path):
    src = tmp_path / "cfg.cpp"
    src.write_text(SRC)
    exe = tmp_path / "cfg"
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-O1", "-I",
                    os.path.join(ROOT, "minkowskiengine_b200", "csrc"), str(src), "-o", str(exe)],
                   check=True)
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-3000:]
    assert "bad=0" in r.stdout
