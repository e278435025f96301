"""Stem layers (c_in <= 4, c_out <= 64: `k_conv_small_cin_fwd` / `k_conv_small_cin_wgrad`,
csrc/conv_simt.cu) against an fp32 torch restatement on random neighbour tables: every c_in,
one and two 32-channel slabs, ragged slabs (scalar-load path), fp32 / bf16 / fp16 features,
K = 125 (the MinkUNet stem, k = 5) and row counts around the 256-entry scan window and the
32-hit consume rounds.  Reference semantics: src/convolution_kernel.hpp:33-144."""
import pytest
import torch

from test_gpu_tc import _random_table, _torch_ref_forward

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
    from minkowskiengine_b200 import backend
    torch.backends.cuda.matmul.allow_tf32 = False
    g = torch.Generator().manual_seed(cin * 100 + cout + K)
    feats = (torch.rand(n_in, cin, generator=g) - 0.5).to(dtype).to(cuda)
    w = ((torch.rand(K, cin, cout, generator=g) - 0.5) / (cin ** 0.5)).to(dtype).to(cuda)
    gout = (torch.rand(n_out, cout, generator=g) - 0.5).to(dtype).to(cuda)
    nbr = _random_table(K, n_out, n_in, density, seed=K + n_out, device=cuda)
    km = backend._KernelMap(nbr, torch.full((K, n_in), -1, dtype=torch.int32, device=cuda))
    ref = _torch_ref_forward(feats, w, nbr)
    scale = ref.abs().max().item()
    out = backend._conv_forward(feats, w, km)
    assert out.dtype == dtype and out.shape == (n_out, cout)
    tol = 2e-6 if dtype == torch.float32 else 6e-3          # fp32 sums; one output rounding
    assert (out.float() - ref).abs().max().item() / scale < tol
    if dtype != torch.float32:
        out32 = backend._conv_forward(feats, w, km, out_dtype=torch.float32)
        assert (out32 - ref).abs().max().item() / scale < 2e-6
    _, gw = backend._conv_backward(feats, gout, w.float(), km, need_in=False, need_w=True)
    gref = torch.zeros(K, cin, cout, dtype=torch.float32, device=cuda)
    f32, g32 = feats.float(), gout.float()
    for k in range(K):
        idx = nbr[k].long()
        gref[k] = (f32[idx.clamp(min=0)] * (idx >= 0).unsqueeze(1)).t() @ g32
    assert gw.shape == gref.shape
    assert (gw.float() - gref).abs().max().item() / gref.abs().max().item() < 2e-5


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("cin,cout,n_in,n_out,K,density", [
    (3, 32, 5000, 5000, 125, 0.16),      # MinkUNet stem shape: 8 stages of 16 offsets per tile
    (3, 32, 900, 257, 27, 0.5),          # K not a multiple of 16: padded offsets
    (1, 64, 700, 1023, 27, 0.3),
    (2, 48, 700, 2048, 8, 0.9),          # half a virtual m-tile (K = 8 -> 64 virtual channels)
    (4, 16, 3000, 4097, 27, 0.05),       # unpadded rows, sparse hits
    (3, 32, 100, 31, 27, 1.0),           # less than one wgrad stage of rows
    (3, 128, 300, 1, 125, 0.5),          # one output row, widest output the K = 125 stem takes
    (3, 96, 40000, 40001, 125, 0.2),     # many CTAs, ragged last tile / stage
])
def test_stem_tensor_core_path(ME, cuda, dtype, cin, cout, n_in, n_out, K, density):
    """The same layers through the tensor-core stem path (fp32 master weights: the wgmma
    kernels' stem mode forward and wgrad) — must have launched tensor-core kernels."""
    from minkowskiengine_b200 import backend, _lib
    lib = _lib.load()
    torch.backends.cuda.matmul.allow_tf32 = False
    g = torch.Generator().manual_seed(cin * 100 + cout + K + 1)
    feats = (torch.rand(n_in, cin, generator=g) - 0.5).to(dtype).to(cuda)
    w = ((torch.rand(K, cin, cout, generator=g) - 0.5) / (cin ** 0.5)).to(dtype).float().to(cuda)
    gout = (torch.rand(n_out, cout, generator=g) - 0.5).to(dtype).to(cuda)
    nbr = _random_table(K, n_out, n_in, density, seed=K + n_out, device=cuda)
    km = backend._KernelMap(nbr, torch.full((K, n_in), -1, dtype=torch.int32, device=cuda))
    assert backend._is_stem(w, dtype)
    ref = _torch_ref_forward(feats, w.to(dtype), nbr)
    scale = ref.abs().max().item()
    n0 = lib.meb200_tc_launch_count()
    out = backend._conv_forward(feats, w, km)
    out32 = backend._conv_forward(feats, w, km, out_dtype=torch.float32)
    assert lib.meb200_tc_launch_count() == n0 + 2, "the stem forward did not take the tensor-core path"
    assert out.dtype == dtype and out.shape == (n_out, cout)
    assert (out32 - ref).abs().max().item() / scale < 1e-5
    assert (out.float() - ref).abs().max().item() / scale < 6e-3
    n0 = lib.meb200_tc_launch_count()
    gi, gw = backend._conv_backward(feats, gout, w, km, need_in=False, need_w=True)
    assert lib.meb200_tc_launch_count() == n0 + 1, "the stem wgrad did not take the tensor-core path"
    gref = torch.zeros(K, cin, cout, dtype=torch.float32, device=cuda)
    f32, g32 = feats.float(), gout.float()
    for k in range(K):
        idx = nbr[k].long()
        gref[k] = (f32[idx.clamp(min=0)] * (idx >= 0).unsqueeze(1)).t() @ g32
    assert gi is None and gw.shape == gref.shape
    assert (gw.float() - gref).abs().max().item() / gref.abs().max().item() < 2e-5
