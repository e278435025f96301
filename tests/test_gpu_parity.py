"""GPU parity: the CUDA path (through the package's public API -> C-ABI) against the oracle.

Integer / index work (coordinate maps, kernel maps, max-pool indices) must be BIT-EXACT after
canonicalising row order by coordinate; features must agree within 1e-3 relative (north_star
tolerance) — in fp32 the observed error is ~1e-6 and the pooling tests assert 1e-5.  Convolution
features and gradients are held element by element to the bound of the CUDA-core kernels,
|y - ref| <= 2^-20 A (tests/helpers.py), A the oracle's same reduction over |x|, |w| and |g|.
"""
import numpy as np
import pytest
import torch

from helpers import (assert_one_rounding, kmap_lists, oracle_conv_layer, random_cloud, rel_err,
                     unique_cloud)
from oracle import oracle_np as O

pytestmark = pytest.mark.gpu

TOL_F32 = 1e-5          # fp32 CUDA path vs float64-accumulating oracle
TOL_NORTH_STAR = 1e-3   # BASELINE.json north_star: "within 1e-3 rel fp32"


@pytest.mark.parametrize("n,extent,D,batches,neg", [
    (1000, 32, 3, 1, False),      # BASELINE cfg0 shape
    (5000, 12, 3, 3, True),       # many duplicates, negative coordinates
    (20000, 40, 4, 2, True),      # 4-D
    (300, 1000, 2, 1, True),      # 2-D, no duplicates likely
    (1, 5, 3, 1, False),
])
def test_insert_and_map_matches_oracle(ME, cuda, n, extent, D, batches, neg):
    coords = random_cloud(n, extent, seed=n, D=D, batches=batches, allow_negative=neg)
    feats = torch.arange(n, dtype=torch.float32).unsqueeze(1)
    x = ME.SparseTensor(feats, coords, device=cuda)
    ui, inv = O.insert_and_map(coords.numpy())
    # first-occurrence order is deterministic and must match the CPU reference exactly
    assert x.C.cpu().numpy().tolist() == coords.numpy()[ui].tolist()
    assert x.F.cpu().numpy()[:, 0].tolist() == ui.astype(np.float32).tolist()
    assert x.unique_index.cpu().numpy().tolist() == ui.tolist()
    assert x.inverse_mapping.cpu().numpy().tolist() == inv.tolist()
    # reconstruct: unique[inverse] == input
    assert torch.equal(x.C.cpu()[x.inverse_mapping.cpu()], coords)


def test_empty_and_single(ME, cuda):
    mgr = ME.CoordinateManager(D=3)
    key, (ui, inv) = mgr.insert_and_map(torch.zeros((0, 4), dtype=torch.int32, device=cuda))
    assert mgr.size(key) == 0 and len(ui) == 0


@pytest.mark.parametrize("stride", [2, 4, 3])
def test_stride_matches_oracle(ME, cuda, stride):
    coords = unique_cloud(4000, 30, seed=7, allow_negative=True)
    mgr = ME.CoordinateManager(D=3)
    key, _ = mgr.insert_and_map(coords.to(cuda))
    skey = mgr.stride(key, stride)
    assert skey.get_tensor_stride() == [stride] * 3
    got = O.unique_rows(mgr.get_coordinates(skey).cpu().numpy())
    exp, _ = O.stride_map_coords(coords.numpy(), [1, 1, 1], [stride] * 3)
    assert got.shape == exp.shape and (got == exp).all()
    assert mgr.size(skey) == len(exp)          # no duplicate rows survived
    # second request returns the same key without creating a map
    assert mgr.stride(key, stride) == skey


def _gpu_layer(ME, cuda, coords, feats, conv):
    x = ME.SparseTensor(feats, coords, device=cuda, requires_grad=True)
    y = conv(x)
    return x, y


def _centred(shape, g):
    return torch.rand(shape, generator=g) - 0.5


def _one_rounding(got, ref, A, what):
    """assert_one_rounding of a GPU fp32 result against float64 oracle arrays."""
    assert_one_rounding(got.detach().cpu(), torch.from_numpy(ref), torch.from_numpy(A), what)


def _check_conv(x_F, y_F, gy, x_grad, w_grad, w, im, om, what):
    """Forward, input gradient and weight gradient of one layer (kernel w, maps im / om) against
    the oracle, given the layer's own input x_F and output gradient gy (numpy float32)."""
    aw = np.abs(w)
    _one_rounding(y_F, O.conv_forward(x_F, w, im, om, len(y_F)),
                  O.conv_forward(np.abs(x_F), aw, im, om, len(y_F)), f"{what} forward")
    gi, gw = O.conv_backward(x_F, gy, w, im, om)
    gi_A, gw_A = O.conv_backward(np.abs(x_F), np.abs(gy), aw, im, om)
    _one_rounding(x_grad, gi, gi_A, f"{what} dgrad")
    _one_rounding(w_grad, gw, gw_A, f"{what} wgrad")


@pytest.mark.parametrize("ks,stride,dil,D,cin,cout,n,extent", [
    (3, 1, 1, 3, 16, 16, 1000, 32),     # BASELINE cfg0
    (3, 2, 1, 3, 8, 24, 3000, 20),
    (2, 2, 1, 3, 5, 7, 3000, 20),
    (5, 1, 1, 3, 3, 32, 1500, 14),
    (3, 1, 2, 3, 4, 4, 2000, 16),
    (3, 1, 1, 4, 6, 10, 3000, 9),       # 4-D, K = 81
    (1, 2, 1, 3, 8, 8, 2000, 16),       # k=1 s=2 (ResNet downsample)
    (3, 1, 1, 2, 70, 130, 800, 24),     # channel counts past one tile
])
def test_convolution_forward_backward(ME, cuda, ks, stride, dil, D, cin, cout, n, extent):
    coords = unique_cloud(n, extent, seed=ks * 100 + stride, D=D, allow_negative=True)
    g = torch.Generator().manual_seed(1)
    feats = _centred((len(coords), cin), g)
    conv = ME.MinkowskiConvolution(cin, cout, kernel_size=ks, stride=stride, dilation=dil,
                                   dimension=D).to(cuda)
    x, y = _gpu_layer(ME, cuda, coords, feats, conv)
    K = ks ** D
    # ---- kernel map: bit-exact as a set of (k, in coordinate, out coordinate) --------
    kd = x.coordinate_manager.kernel_map(x.coordinate_map_key, y.coordinate_map_key,
                                         stride=stride, kernel_size=ks, dilation=dil)
    im_g, om_g = kmap_lists(kd, K)
    in_c, out_c = x.C.cpu().numpy(), y.C.cpu().numpy()
    out_or, im, om = oracle_conv_layer(in_c, [1] * D, ks, stride, dil)
    assert (O.unique_rows(out_c) == out_or).all() and len(out_c) == len(out_or)
    im2, om2 = O.kernel_map(in_c, out_c, O.region_offsets(O.HYPER_CUBE, [ks] * D, [dil] * D, [1] * D))
    t_gpu = O.kernel_map_triples(in_c, out_c, im_g, om_g)
    t_or = O.kernel_map_triples(in_c, out_c, im2, om2)
    assert t_gpu.shape == t_or.shape and (t_gpu == t_or).all()
    # ---- features --------------------------------------------------------------------
    gout = _centred(y.F.shape, g)
    y.F.backward(gout.to(cuda))
    _check_conv(x.F.detach().cpu().numpy(), y.F, gout.numpy(), x.F.grad, conv.kernel.grad,
                conv.kernel.detach().cpu().numpy(), im2, om2, "conv")


def test_transposed_convolution_unet_pair(ME, cuda):
    """conv k2 s2 down then conv-transpose k2 s2 up lands on the encoder's coordinate map
    (reference: coordinate_map_manager.cpp:450-465, 763-774) and matches the oracle.  Each layer
    is checked on its own input and output gradient as the GPU computed them (y.F, y.F.grad), so
    that the first layer's rounding is not charged to the second."""
    D, cin, cmid, cout = 3, 6, 10, 4
    coords = unique_cloud(3000, 18, seed=3, allow_negative=True)
    g = torch.Generator().manual_seed(2)
    feats = _centred((len(coords), cin), g)
    down = ME.MinkowskiConvolution(cin, cmid, kernel_size=2, stride=2, dimension=D).to(cuda)
    up = ME.MinkowskiConvolutionTranspose(cmid, cout, kernel_size=2, stride=2, dimension=D).to(cuda)
    x = ME.SparseTensor(feats, coords, device=cuda, requires_grad=True)
    y = down(x)
    y.F.retain_grad()
    z = up(y)
    assert z.coordinate_map_key == x.coordinate_map_key      # ME.cat(z, x) must be legal
    ME.cat(z, x)
    in_c, mid_c = x.C.cpu().numpy(), y.C.cpu().numpy()
    im, om = O.kernel_map(in_c, mid_c, O.region_offsets(O.HYPER_CUBE, [2] * D, [1] * D, [1] * D))
    # transposed: offsets in OUTPUT (fine) stride units, iterate coarse rows
    imt, omt = O.transposed_kernel_map(mid_c, in_c, O.region_offsets(O.HYPER_CUBE, [2] * D, [1] * D, [1] * D))
    kd = x.coordinate_manager.kernel_map(y.coordinate_map_key, z.coordinate_map_key, stride=2,
                                         kernel_size=2, is_transpose=True)
    im_g, om_g = kmap_lists(kd, 8)
    assert (O.kernel_map_triples(mid_c, in_c, im_g, om_g) ==
            O.kernel_map_triples(mid_c, in_c, imt, omt)).all()
    gout = _centred(z.F.shape, g)
    z.F.backward(gout.to(cuda))
    _check_conv(y.F.detach().cpu().numpy(), z.F, gout.numpy(), y.F.grad, up.kernel.grad,
                up.kernel.detach().cpu().numpy(), imt, omt, "transpose")
    _check_conv(x.F.detach().cpu().numpy(), y.F, y.F.grad.cpu().numpy(), x.F.grad,
                down.kernel.grad, down.kernel.detach().cpu().numpy(), im, om, "conv")


def test_generative_transpose_creates_coordinates(ME, cuda):
    D = 2
    coords = unique_cloud(200, 10, seed=5, D=D)
    coords[:, 1:] *= 2
    feats = torch.rand(len(coords), 3)
    x = ME.SparseTensor(feats, coords, tensor_stride=2, device=cuda)
    up = ME.MinkowskiGenerativeConvolutionTranspose(3, 5, kernel_size=2, stride=2, dimension=D).to(cuda)
    z = up(x)
    offs = O.region_offsets(O.HYPER_CUBE, [2] * D, [1] * D, [1] * D)
    cand = (coords.numpy()[:, None, :] + np.concatenate([np.zeros((4, 1), np.int32), offs], 1)[None]).reshape(-1, D + 1)
    exp = O.unique_rows(cand)
    got = O.unique_rows(z.C.cpu().numpy())
    assert z.tensor_stride == [1] * D and got.shape == exp.shape and (got == exp).all()


@pytest.mark.parametrize("mode,ks,stride", [
    ("avg", 2, 2), ("sum", 2, 2), ("max", 2, 2), ("max", 3, 2), ("avg", 3, 2), ("sum", 3, 1),
    ("max", 3, 3),
])
def test_local_pooling(ME, cuda, mode, ks, stride):
    D, C = 3, 6
    coords = unique_cloud(2500, 15, seed=11, allow_negative=True)
    g = torch.Generator().manual_seed(4)
    feats = torch.randn(len(coords), C, generator=g)
    layer = {"avg": ME.MinkowskiAvgPooling, "sum": ME.MinkowskiSumPooling,
             "max": ME.MinkowskiMaxPooling}[mode](kernel_size=ks, stride=stride, dimension=D)
    omode = {"avg": O.POOL_AVG, "sum": O.POOL_SUM, "max": O.POOL_MAX}[mode]
    x = ME.SparseTensor(feats, coords, device=cuda, requires_grad=True)
    y = layer(x)
    in_c, out_c = x.C.cpu().numpy(), y.C.cpu().numpy()
    if ks == stride:   # the reference takes the stride-map shortcut (coordinate_map_manager.cpp:722-729)
        im, om = O.stride_map(in_c, out_c, [stride] * D)
        kd = x.coordinate_manager.kernel_map(x.coordinate_map_key, y.coordinate_map_key,
                                             stride=stride, kernel_size=ks, is_pool=True)
        assert list(kd.keys()) == [0]
        got = np.stack(sorted(map(tuple, kd[0].cpu().numpy().T.tolist())))
        exp = np.stack(sorted(zip(im[0].tolist(), om[0].tolist())))
        assert (got == exp).all()
    else:
        im, om = O.kernel_map(in_c, out_c, O.region_offsets(O.HYPER_CUBE, [ks] * D, [1] * D, [1] * D))
    out_ref, aux = O.pool_forward(feats.numpy(), im, om, len(out_c), omode)
    assert rel_err(y.F.detach().cpu().numpy(), out_ref) < TOL_F32
    gout = torch.rand(y.F.shape, generator=g)
    y.F.backward(gout.to(cuda))
    gi_ref = O.pool_backward(gout.numpy(), len(in_c), im, om, omode, aux)
    assert rel_err(x.F.grad.cpu().numpy(), gi_ref) < TOL_F32


@pytest.mark.parametrize("ks,D", [(3, 3), (5, 3), (3, 4)])
def test_hyper_cross_convolution(ME, cuda, ks, D):
    """RegionType.HYPER_CROSS (kernel_region.hpp:217-243: centre + one arm per axis) through the
    public API on the GPU: kernel map bit-exact, features/gradients vs the oracle."""
    coords = unique_cloud(2500, 12, seed=40 + ks + D, D=D, allow_negative=True)
    g = torch.Generator().manual_seed(3)
    cin, cout = 6, 10
    feats = _centred((len(coords), cin), g)
    kgen = ME.KernelGenerator(kernel_size=ks, stride=1, dilation=1,
                              region_type=ME.RegionType.HYPER_CROSS, dimension=D)
    K = 1 + D * (ks - 1)
    assert kgen.kernel_volume == K
    conv = ME.MinkowskiConvolution(cin, cout, kernel_generator=kgen, dimension=D).to(cuda)
    assert tuple(conv.kernel.shape) == (K, cin, cout)
    x, y = _gpu_layer(ME, cuda, coords, feats, conv)
    kd = x.coordinate_manager.kernel_map(x.coordinate_map_key, y.coordinate_map_key,
                                         kernel_size=ks, region_type=ME.RegionType.HYPER_CROSS)
    im_g, om_g = kmap_lists(kd, K)
    in_c = x.C.cpu().numpy()
    im, om = O.kernel_map(in_c, in_c, O.region_offsets(O.HYPER_CROSS, [ks] * D, [1] * D, [1] * D))
    t_gpu = O.kernel_map_triples(in_c, in_c, im_g, om_g)
    t_or = O.kernel_map_triples(in_c, in_c, im, om)
    assert t_gpu.shape == t_or.shape and (t_gpu == t_or).all()
    gout = _centred(y.F.shape, g)
    y.F.backward(gout.to(cuda))
    _check_conv(x.F.detach().cpu().numpy(), y.F, gout.numpy(), x.F.grad, conv.kernel.grad,
                conv.kernel.detach().cpu().numpy(), im, om, "hyper-cross conv")
