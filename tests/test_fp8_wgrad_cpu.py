"""fp8 weight gradient without a GPU (ME.fp8_training(weight_gradient=True)): the context's rules,
which layers it selects, the calls the autograd Functions make against a stub library (the wgrad
multiplies the very e4m3 bytes the forward multiplied and the e5m2 bytes the dgrad multiplied, the
output gradient is quantised once per backward, and the default context makes the calls it always
made), and the shared-memory footprint of k_wgrad_fp8 (csrc/tc_config.h) for every c_out on the
grid."""
import os
import subprocess
import threading

import pytest
import torch

import minkowskiengine_b200 as ME
from minkowskiengine_b200 import backend as B
from minkowskiengine_b200 import convolution as CV
from test_fp8_train_cpu import _TMap, _conv, _named, _Stub, _x

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- the context ---------------------------------------------------------------------------------
def test_default_is_off_and_innermost_decides():
    conv = _conv()
    assert not B.fp8_training_weight_gradient()
    with ME.fp8_training():
        assert not B.fp8_training_weight_gradient() and not CV._fp8_train_wgrad(conv)
        with ME.fp8_training(weight_gradient=True):
            assert B.fp8_training_weight_gradient() and CV._fp8_train_wgrad(conv)
            with ME.fp8_training():
                assert B.fp8_training_enabled() and not B.fp8_training_weight_gradient()
            assert B.fp8_training_weight_gradient()
        assert B.fp8_training_enabled() and not B.fp8_training_weight_gradient()
    assert not B.fp8_training_enabled() and not B.fp8_training_weight_gradient()


def test_weight_gradient_is_keyword_only():
    with pytest.raises(TypeError):
        with ME.fp8_training(True):
            pass
    assert not B.fp8_training_enabled()


def test_survives_exceptions():
    with ME.fp8_training():
        with pytest.raises(ValueError):
            with ME.fp8_training(weight_gradient=True):
                raise ValueError
        assert B.fp8_training_enabled() and not B.fp8_training_weight_gradient()
    assert not B.fp8_training_enabled()


def test_thread_local():
    seen = []
    with ME.fp8_training(weight_gradient=True):
        t = threading.Thread(target=lambda: seen.append(
            (B.fp8_training_enabled(), B.fp8_training_weight_gradient())))
        t.start()
        t.join()
        assert B.fp8_training_weight_gradient()
    assert seen == [(False, False)]


def test_nests_with_fp8_inference_and_calibration():
    conv = _conv()
    with ME.fp8_inference():
        with ME.fp8_training(weight_gradient=True):
            assert CV._fp8_train(conv, _x()) and CV._fp8_train_wgrad(conv)
            with torch.no_grad():
                assert CV._fp8(conv, _x()) and not CV._fp8_train(conv, _x())
        assert B.fp8_enabled() and not B.fp8_training_weight_gradient()
    calib = ME.Fp8Calibration(torch.nn.Sequential(conv))
    with calib.observe():
        with ME.fp8_training(weight_gradient=True):
            assert B.fp8_observer() is calib and CV._fp8_train_wgrad(conv)
        assert B.fp8_observer() is calib and not B.fp8_training_enabled()


# ---- the selection ---------------------------------------------------------------------------------
SHAPES = [(32, 32, 3), (32, 64, 3), (64, 96, 2), (96, 1024, 3), (1024, 1024, 1), (384, 256, 3),
          (32, 16, 3), (48, 64, 3), (32, 1040, 3), (3, 32, 5), (32, 32, 1)]


@pytest.mark.parametrize("c_in,c_out,ks", SHAPES, ids=lambda v: str(v))
@pytest.mark.parametrize("grad", [True, False], ids=["input_grad", "kernel_grad_only"])
def test_selects_the_layers_of_fp8_training(c_in, c_out, ks, grad):
    """The same layers as fp8_training() (convolution._fp8_train_rule); each of them also runs its
    weight gradient on fp8 (their K is at most 125 here)."""
    conv = _conv(c_in, c_out, kernel_size=ks)
    x = _x(c_in, grad=grad)
    with ME.fp8_training():
        plain = CV._fp8_train(conv, x)
    with ME.fp8_training(weight_gradient=True):
        assert CV._fp8_train(conv, x) == plain
        assert CV._fp8_train_wgrad(conv) == (B.fp8_supported(c_in, c_out) and
                                             B.fp8_supported(c_out, c_in))


@pytest.mark.parametrize("c_in,c_out,K,ok", [
    (32, 32, 1, True), (32, 32, 27, True), (1024, 1024, 1023, True), (32, 32, 1024, False),
    (32, 32, 1331, False), (32, 32, 0, False), (48, 32, 27, False), (32, 48, 27, False),
    (16, 32, 27, False), (32, 1056, 27, False), (1056, 32, 27, False)], ids=lambda v: str(v))
def test_wgrad_grid(c_in, c_out, K, ok):
    assert B.fp8_wgrad_supported(c_in, c_out, K) == ok


def test_more_than_1023_offsets_keep_the_feature_wgrad():
    """kernel_size 11 in 3-D has K = 1331, past the pair lists' limit: the layer is selected for
    the fp8 forward and dgrad, its weight gradient stays on the feature dtype."""
    conv = _conv(32, 32, kernel_size=11)
    with ME.fp8_training(weight_gradient=True):
        assert CV._fp8_train(conv, _x()) and not CV._fp8_train_wgrad(conv)


# ---- the calls, against a stub library --------------------------------------------------------------
class _PMap(_TMap):
    """_TMap with pair lists (and other row counts)."""

    def __init__(self, n_in=10, n_out=12):
        super().__init__()
        self.n_in, self.n_out = n_in, n_out
        self.pairs = (torch.zeros(64, dtype=torch.int32), torch.zeros(64, dtype=torch.int32),
                      torch.zeros(28, dtype=torch.int32), 1)

    def pair_lists(self):
        return self.pairs


class _Mgr:
    def __init__(self, km):
        self._manager = self
        self.km = km

    def _kernel_map(self, *a):
        return self.km

    def exists(self, key):
        return True

    def size(self, key):
        return self.km.n_out


@pytest.fixture
def stub(monkeypatch):
    from minkowskiengine_b200 import _lib
    real = _lib.load()
    calls = []
    monkeypatch.setattr(_lib, "load", lambda: _Stub(calls, real))
    monkeypatch.setattr(_lib, "current_stream", lambda: None)
    for name in ("_QUANT_WS", "_PACKED", "_PACK_TABLES"):
        monkeypatch.setattr(B, name, {})
    monkeypatch.setattr(B, "_check_feats", lambda *a, **k: None)

    def forward(in_feat, kernel, *a, fp8=False, act=None):   # the native forward past its checks
        return B._conv_forward(in_feat, kernel, a[-1]._kernel_map(), fp8=fp8, act=act)
    monkeypatch.setattr(B, "ConvolutionForwardGPU", forward)
    monkeypatch.setattr(B, "ConvolutionTransposeForwardGPU", forward)
    monkeypatch.setattr(B, "fp8_wgrad_supported", lambda c_in, c_out, K: bool(
        real.meb200_conv_wgrad_fp8_supported(c_in, c_out, K)))
    saved = torch.backends.cuda.matmul.fp32_precision
    torch.backends.cuda.matmul.fp32_precision = "ieee"
    yield calls
    torch.backends.cuda.matmul.fp32_precision = saved


def _step(cls, km, fp8_wgrad, dtype=torch.bfloat16, need_in=True, need_w=True):
    """One forward and backward through the autograd Function with the fp8 flag set."""
    x = torch.randn(10, 32).to(dtype).requires_grad_(need_in)
    k = torch.randn(27, 32, 64).requires_grad_(need_w)
    y = cls.apply(x, k, ME.KernelGenerator(3, dimension=3), None, object(), object(), _Mgr(km),
                  True, fp8_wgrad)
    g = torch.randn(y.shape).to(dtype)
    y.backward(g)
    return x, k, y


FUNCS = [CV.MinkowskiConvolutionFunction, CV.MinkowskiConvolutionTransposeFunction]
FIDS = ["conv", "transpose"]
DEFAULT_CALLS = ["meb200_conv_pack_weights_e4m3", "meb200_quantize_e4m3", "meb200_conv_forward_fp8",
                 "meb200_conv_pack_weights_e4m3_dgrad", "meb200_quantize_e5m2",
                 "meb200_conv_dgrad_fp8", "meb200_conv_backward"]


def _sequence(calls):
    return [c[0] for c in calls if not c[0].endswith(("_supported", "_bytes", "_uses_pairs"))]


@pytest.mark.parametrize("cls", FUNCS, ids=FIDS)
def test_default_context_makes_the_calls_it_made(stub, cls):
    """weight_gradient off: the e4m3 forward quantises its own input, the dgrad its own gradient,
    and the weight gradient is meb200_conv_backward's, as in fp8_training() before the option."""
    _step(cls, _PMap(), False)
    assert _sequence(stub) == DEFAULT_CALLS
    (_, a), = _named(stub, "meb200_conv_backward")
    assert a[5] is None and a[12] is not None          # the wgrad alone, in the feature dtype


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("cls", FUNCS, ids=FIDS)
def test_wgrad_multiplies_the_forward_and_dgrad_bytes(stub, cls, dtype):
    km = _PMap()
    x, k, y = _step(cls, km, True, dtype)
    assert y.dtype == dtype and x.grad.dtype == dtype and k.grad.dtype == torch.float32
    (_, qa), = _named(stub, "meb200_quantize_e4m3")
    (_, fa), = _named(stub, "meb200_conv_forward_fp8")
    (_, qg), = _named(stub, "meb200_quantize_e5m2")           # once per backward
    (_, da), = _named(stub, "meb200_conv_dgrad_fp8")
    (_, wa), = _named(stub, "meb200_conv_wgrad_fp8")
    assert qa[0] == x.data_ptr() and qa[1] == ME._lib.dtype_code(dtype)
    assert fa[0] == qa[4] and fa[1] == qa[5]                  # the forward's e4m3 bytes and scale
    assert wa[0] == qa[4] and wa[1] == qa[5]                  # ... are the wgrad's
    assert da[0] == qg[4] and da[1] == qg[5]                  # the dgrad's e5m2 bytes and scale
    assert wa[2] == qg[4] and wa[3] == qg[5]                  # ... are the wgrad's
    assert qg[1] == ME._lib.dtype_code(dtype) and qg[2:4] == (12, 64)
    pin, pout, seg, nch = km.pair_lists()
    assert wa[4:7] == (32, 27, 64)
    assert wa[7:12] == (pin.data_ptr(), pout.data_ptr(), seg.data_ptr(), nch, 12)
    assert not _named(stub, "meb200_conv_backward")
    assert _sequence(stub) == ["meb200_quantize_e4m3", "meb200_conv_pack_weights_e4m3",
                               "meb200_conv_forward_fp8", "meb200_quantize_e5m2",
                               "meb200_conv_pack_weights_e4m3_dgrad", "meb200_conv_dgrad_fp8",
                               "meb200_conv_wgrad_fp8"]


def test_input_needing_no_gradient_quantises_for_the_wgrad_alone(stub):
    _step(CV.MinkowskiConvolutionFunction, _PMap(), True, need_in=False)
    assert len(_named(stub, "meb200_quantize_e5m2")) == 1
    assert not _named(stub, "meb200_conv_dgrad_fp8")
    assert not _named(stub, "meb200_conv_pack_weights_e4m3_dgrad")
    (_, qg), = _named(stub, "meb200_quantize_e5m2")
    (_, wa), = _named(stub, "meb200_conv_wgrad_fp8")
    assert wa[2] == qg[4] and wa[3] == qg[5]


def test_kernel_needing_no_gradient_runs_no_wgrad(stub):
    _step(CV.MinkowskiConvolutionFunction, _PMap(), True, need_w=False)
    assert len(_named(stub, "meb200_quantize_e5m2")) == 1
    assert not _named(stub, "meb200_conv_wgrad_fp8") and not _named(stub, "meb200_conv_backward")


class _WsStub(_Stub):
    def __getattr__(self, name):
        if name == "meb200_conv_wgrad_fp8_workspace_bytes":
            return lambda *a: (self.calls.append((name, a)), 4096)[1]
        return super().__getattr__(name)


def test_workspace_is_the_library_query(stub, monkeypatch):
    """The host sizes the workspace by meb200_conv_wgrad_fp8_workspace_bytes and hands it over."""
    from minkowskiengine_b200 import _lib
    monkeypatch.setattr(_lib, "load", lambda: _WsStub(stub, None))
    gw = B._conv_wgrad_fp8((torch.zeros(10, 32, dtype=torch.uint8), torch.ones(2)),
                           (torch.zeros(12, 64, dtype=torch.uint8), torch.ones(2)),
                           torch.randn(27, 32, 64), _PMap())
    assert gw.shape == (27, 32, 64) and gw.dtype == torch.float32
    (_, ws), = _named(stub, "meb200_conv_wgrad_fp8_workspace_bytes")
    (_, wa), = _named(stub, "meb200_conv_wgrad_fp8")
    assert ws == (12, 32, 64, 27)
    assert wa[12] is not None and wa[13] is not None and wa[14] == 4096


@pytest.mark.parametrize("n_in,n_out", [(10, 0), (0, 12)], ids=["no_output_rows", "no_input_rows"])
def test_empty_maps_give_zero_without_a_launch(stub, n_in, n_out):
    act = (torch.zeros(n_in, 32, dtype=torch.uint8), torch.ones(2))
    gi, gw = B._conv_backward_fp8w(act, torch.bfloat16, torch.zeros(n_out, 64).bfloat16(),
                                   torch.randn(27, 32, 64), _PMap(n_in, n_out))
    assert gi.shape == (n_in, 32) and gi.dtype == torch.bfloat16 and not gi.any()
    assert gw.shape == (27, 32, 64) and gw.dtype == torch.float32 and not gw.any()
    assert not [c for c in stub if c[0].startswith(("meb200_quant", "meb200_conv"))]


# ---- the shared-memory footprint ---------------------------------------------------------------------
SRC = r"""
#include <stdio.h>
#include "tc_config.h"
using namespace meb200::tc;
int main() {
  int bad = 0;
  for (unsigned co = 32; co <= 1024; co += 32) {
    const unsigned cols = wgrad_fp8_cols(co), smem = wgrad_fp8_smem_bytes(cols);
    const bool ok = (cols == 32 || cols == 64 || cols == 96 || cols == 128) && co % cols == 0 &&
                    cols <= kWgFp8MaxCols && (co > kWgFp8MaxCols || cols == co) &&
                    smem <= kSmemLimit && co / cols <= 32;
    if (!ok) { printf("FP8 WG BAD co=%u cols=%u smem=%u\n", co, cols, smem); ++bad; }
    printf("fp8 wg %u : cols=%u smem=%u\n", co, cols, smem);
  }
  if (kWgFp8Sbo % 16 != 0 || (kWgFp8Sbo / 4) % 32 != 4) { printf("SBO BAD\n"); ++bad; }
  printf("bad=%d\n", bad);
  return bad != 0;
}
"""


def test_wgrad_fp8_footprint(tmp_path):
    """Every c_out on the grid gets a column tile of 32, 64, 96 or 128 dividing it (the whole
    c_out up to 128) whose ring and two transposed tiles fit in 227 KB, and the group stride of a
    transposed tile is a multiple of 16 bytes that is 4 words off a multiple of 32 banks."""
    src = tmp_path / "cfg.cpp"
    src.write_text(SRC)
    exe = tmp_path / "cfg"
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-O1", "-I",
                    os.path.join(ROOT, "minkowskiengine_b200", "csrc"), str(src), "-o", str(exe)],
                   check=True)
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-3000:]
    assert "bad=0" in r.stdout
