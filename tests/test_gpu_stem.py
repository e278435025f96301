"""Stem layers (c_in <= 4) against a float64 restatement on random neighbour tables, element by
element (tests/helpers.py).

`k_conv_small_cin_fwd` / `k_conv_small_cin_wgrad` (csrc/conv_simt.cu) run a kernel that is not an
fp32 master: every c_in, one and two 32-channel slabs, ragged slabs (scalar-load path), fp32 /
bf16 / fp16 features, K = 125 (the MinkUNet stem, k = 5) and row counts around the 256-entry scan
window and the 32-hit consume rounds.  An fp32 master kernel in bf16 / fp16 takes the stem mode of
the wgmma kernels instead: virtual channels 4 k + c, padded to 16 ceil(K / 16) offsets.
Reference semantics: src/convolution_kernel.hpp:33-144."""
import pytest
import torch

from helpers import TC_ACC, _pairs, assert_one_rounding, ref_conv, ref_wgrad
from test_gpu_tc import _random_table

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("cin,cout,n_in,n_out,K,density", [
    (3, 32, 5000, 5000, 125, 0.16),      # MinkUNet stem shape
    (3, 32, 900, 257, 27, 0.5),          # one row past a scan window
    (1, 64, 700, 1023, 27, 0.3),         # two full slabs
    (2, 48, 700, 2048, 8, 0.9),          # second slab ragged (16 channels)
    (4, 20, 3000, 4097, 27, 0.05),       # ragged single slab, sparse hits (carried remainders)
    (3, 32, 100, 31, 27, 1.0),           # fewer rows than one consume round
])
def test_stem_forward_and_wgrad(ME, cuda, dtype, cin, cout, n_in, n_out, K, density):
    from minkowskiengine_b200 import _lib, backend
    g = torch.Generator().manual_seed(cin * 100 + cout + K)
    feats = (torch.rand(n_in, cin, generator=g) - 0.5).to(dtype).to(cuda)
    w = ((torch.rand(K, cin, cout, generator=g) - 0.5) / (cin ** 0.5)).to(dtype).to(cuda)
    gout = (torch.rand(n_out, cout, generator=g) - 0.5).to(dtype).to(cuda)
    nbr = _random_table(K, n_out, n_in, density, seed=K + n_out, device=cuda)
    km = backend._KernelMap(nbr, torch.full((K, n_in), -1, dtype=torch.int32, device=cuda))
    ref, A = ref_conv(feats, w, _pairs(nbr), n_out)
    n0 = _lib.tc_launch_count()
    out = backend._conv_forward(feats, w, km)
    assert _lib.tc_launch_count() == n0, "a non-master stem kernel ran on the tensor cores"
    assert out.dtype == dtype and out.shape == (n_out, cout)
    assert_one_rounding(out, ref, A, "small-cin forward")
    assert torch.equal(out, backend._conv_forward(feats, w, km))
    if dtype != torch.float32:
        out32 = backend._conv_forward(feats, w, km, out_dtype=torch.float32)
        assert_one_rounding(out32, ref, A, "small-cin forward, fp32 output")
    # an fp32 copy of the kernel is a master: bf16 / fp16 with c_out % 16 == 0 take the stem mode
    wm = w.float()
    tc = backend._is_stem(wm, dtype)
    n0 = _lib.tc_launch_count()
    _, gw = backend._conv_backward(feats, gout, wm, km, need_in=False, need_w=True)
    assert (_lib.tc_launch_count() > n0) == tc
    _, gw2 = backend._conv_backward(feats, gout, wm, km, need_in=False, need_w=True)
    gref, gA = ref_wgrad(feats, gout, _pairs(nbr))
    assert gw.shape == gref.shape
    assert_one_rounding(gw, gref, gA, "stem wgrad", TC_ACC if tc else 1.0)
    assert torch.equal(gw, gw2), "stem wgrad differs run to run"


def _stem_tc_case(cuda, dtype, cin, cout, n_in, n_out, K, density, seed):
    """The layer through the tensor-core stem mode (fp32 master weights): forward in the feature
    dtype and in fp32, and the wgrad, each against float64 and repeated bitwise."""
    from minkowskiengine_b200 import backend, _lib
    lib = _lib.load()
    g = torch.Generator().manual_seed(seed)
    feats = (torch.rand(n_in, cin, generator=g) - 0.5).to(dtype).to(cuda)
    w = ((torch.rand(K, cin, cout, generator=g) - 0.5) / (cin ** 0.5)).to(dtype).float().to(cuda)
    gout = (torch.rand(n_out, cout, generator=g) - 0.5).to(dtype).to(cuda)
    nbr = _random_table(K, n_out, n_in, density, seed=K + n_out, device=cuda)
    km = backend._KernelMap(nbr, torch.full((K, n_in), -1, dtype=torch.int32, device=cuda))
    assert backend._is_stem(w, dtype)
    ref, A = ref_conv(feats, w, _pairs(nbr), n_out)
    n0 = lib.meb200_tc_launch_count()
    out = backend._conv_forward(feats, w, km)
    out32 = backend._conv_forward(feats, w, km, out_dtype=torch.float32)
    assert lib.meb200_tc_launch_count() == n0 + 2, "the stem forward did not take the tensor-core path"
    assert out.dtype == dtype and out.shape == (n_out, cout)
    assert_one_rounding(out32, ref, A, "stem forward, fp32 output", TC_ACC)
    assert_one_rounding(out, ref, A, "stem forward", TC_ACC)
    assert torch.equal(out, backend._conv_forward(feats, w, km)), "stem forward differs run to run"
    n0 = lib.meb200_tc_launch_count()
    gi, gw = backend._conv_backward(feats, gout, w, km, need_in=False, need_w=True)
    assert lib.meb200_tc_launch_count() == n0 + 1, "the stem wgrad did not take the tensor-core path"
    _, gw2 = backend._conv_backward(feats, gout, w, km, need_in=False, need_w=True)
    gref, gA = ref_wgrad(feats, gout, _pairs(nbr))
    assert gi is None and gw.shape == gref.shape
    assert_one_rounding(gw, gref, gA, "stem wgrad", TC_ACC)
    assert torch.equal(gw, gw2), "stem wgrad differs run to run"


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("cin,cout,n_in,n_out,K,density", [
    (3, 32, 5000, 5000, 125, 0.16),      # MinkUNet stem shape: 8 stages of 16 offsets per tile
    (3, 32, 900, 257, 27, 0.5),          # K not a multiple of 16: padded offsets
    (1, 64, 700, 1023, 27, 0.3),
    (2, 48, 700, 2048, 8, 0.9),          # half a virtual m-tile (K = 8 -> 64 virtual channels)
    (4, 16, 3000, 4097, 27, 0.05),       # unpadded rows, sparse hits
    (3, 32, 100, 31, 27, 1.0),           # less than one wgrad stage of rows
    (3, 128, 300, 1, 125, 0.5),          # one output row
    (3, 96, 40000, 40001, 125, 0.2),     # many CTAs, ragged last tile / stage
])
def test_stem_tensor_core_path(ME, cuda, dtype, cin, cout, n_in, n_out, K, density):
    _stem_tc_case(cuda, dtype, cin, cout, n_in, n_out, K, density, seed=cin * 100 + cout + K + 1)


# Around the padding of the virtual channels to 16 ceil(K / 16) offsets (K = 1, 15, 16, 17; 27 and
# 125 as in networks), every c_in, and output widths from one 16-column instruction to the 256
# columns conv_stem_tc_supported accepts at every K.
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("K,cin,cout", [
    (1, 1, 16), (1, 4, 256),
    (15, 2, 48), (15, 3, 112),
    (16, 3, 112), (16, 4, 16),
    (17, 4, 256), (17, 1, 48),
    (27, 1, 112), (27, 2, 256),
    (125, 4, 256), (125, 2, 16), (125, 1, 48),
])
def test_stem_tensor_core_padding_and_widths(ME, cuda, dtype, K, cin, cout):
    _stem_tc_case(cuda, dtype, cin, cout, 3000, 2500, K, 0.4, seed=K * 1000 + cin * 300 + cout)
