"""Tile orders of neighbour tables (meb200_kernel_map): rows stably sorted by neighbour mask, the
table copied into slot order and one offset mask per 128-row tile.  The forward / dgrad kernel run
on an order must give exactly the bits it gives without one: a row's sum does not depend on its
tile-mates, and a skipped stage would only have added zero products to it."""
import numpy as np
import pytest
import torch

from helpers import unique_cloud

pytestmark = pytest.mark.gpu


def _check_order(nbr, order):
    """order == the tile order of the k-major table nbr, recomputed on the host."""
    K, n = nbr.shape
    nbr, order = nbr.cpu().numpy(), order.cpu().numpy()
    assert order.shape == ((K + 1) * n + (n + 127) // 128,)
    mask = ((nbr >= 0).astype(np.int64) << np.arange(K)[:, None]).sum(0)
    slot_row = order[K * n:(K + 1) * n]
    assert (np.sort(slot_row) == np.arange(n)).all(), "slot -> row is not a permutation"
    assert (slot_row == np.argsort(mask, kind="stable")).all(), "not a stable sort by mask"
    tiles = order[(K + 1) * n:].view(np.uint32).astype(np.int64)
    want = np.zeros(len(tiles), dtype=np.int64)
    np.bitwise_or.at(want, np.arange(n) // 128, mask[slot_row])
    assert (tiles == want).all(), "tile mask is not the OR of its rows' masks"
    assert (order[:K * n].reshape(K, n) == nbr[:, slot_row]).all(), "slot-order table"


def _maps(ME, coords, cuda, ks, stride, transpose):
    x = ME.SparseTensor(torch.zeros(len(coords), 1), coords, device=cuda)
    mgr = x.coordinate_manager
    key = x.coordinate_map_key
    other = key if stride == 1 else mgr.stride(key, stride)
    ik, ok = (other, key) if transpose else (key, other)
    return mgr._manager._kernel_map(ik, ok, [ks] * 3, [stride] * 3, [1] * 3,
                                    ME.RegionType.HYPER_CUBE, torch.IntTensor(), transpose, False)


def _apart_maps(cuda, n_x, n_y, seed):
    """Two maps of one cloud each, the second shifted so that only part of it meets the first:
    many rows without any neighbour (whole empty tiles) and a ragged last tile."""
    from minkowskiengine_b200 import backend
    a = unique_cloud(n_x, 40, seed=seed)
    b = unique_cloud(n_y, 40, seed=seed + 1)
    b[: len(b) // 2, 1] += 1000
    mx, _, _ = backend._CoordinateMap.build(a.int().to(cuda), (1, 1, 1))
    my, _, _ = backend._CoordinateMap.build(b.int().to(cuda), (1, 1, 1))
    return mx, my


def _probe(cuda, ks, n_x, n_y, seed):
    from minkowskiengine_b200 import backend
    mx, my = _apart_maps(cuda, n_x, n_y, seed)
    offs = backend._device_offsets(backend.RegionType.HYPER_CUBE, [ks] * 3, [1] * 3, (1, 1, 1),
                                   None, cuda)
    out_nbr, in_nbr, out_order, in_order = backend.CoordinateMapManagerGPU_c10._probe(
        mx, my, offs, orders=True)
    return out_nbr, in_nbr, out_order, in_order


@pytest.mark.parametrize("ks,stride,transpose", [(3, 1, False), (2, 2, False), (2, 2, True),
                                                 (3, 2, False), (3, 2, True)])
def test_order_of_manager_maps(ME, cuda, ks, stride, transpose):
    coords = unique_cloud(9000, 30, seed=ks + 3 * stride, batches=2)
    km = _maps(ME, coords, cuda, ks, stride, transpose)
    assert km.out_order is not None and km.in_order is not None
    _check_order(km.out_nbr, km.out_order)
    _check_order(km.in_nbr, km.in_order)


@pytest.mark.parametrize("ks", [3, 2])
def test_order_with_empty_rows_and_tiles(ME, cuda, ks):
    out_nbr, in_nbr, out_order, in_order = _probe(cuda, ks, 5000, 7001, seed=ks)
    assert int(((out_nbr >= 0).sum(0) == 0).sum()) >= 256 or int(((in_nbr >= 0).sum(0) == 0).sum()) >= 256
    _check_order(out_nbr, out_order)
    _check_order(in_nbr, in_order)
    tiles = in_order[(in_nbr.shape[0] + 1) * in_nbr.shape[1]:]
    assert int((tiles == 0).sum()) >= 1, "no empty tile"


def test_no_order_for_pooling_or_large_kernels(ME, cuda):
    coords = unique_cloud(3000, 20, seed=4)
    x = ME.SparseTensor(torch.zeros(len(coords), 1), coords, device=cuda)
    m = x.coordinate_manager._manager
    km = m._kernel_map(x.coordinate_map_key, x.coordinate_map_key, [3] * 3, [1] * 3, [1] * 3,
                       ME.RegionType.HYPER_CUBE, torch.IntTensor(), False, True)
    assert km.out_order is None and km.in_order is None
    km = m._kernel_map(x.coordinate_map_key, x.coordinate_map_key, [5] * 3, [1] * 3, [1] * 3,
                       ME.RegionType.HYPER_CUBE, torch.IntTensor(), False, False)
    assert km.out_order is None and km.in_order is None


def _same_bits(km, plain, cin, cout, dtype, cuda, seed):
    from minkowskiengine_b200 import _lib, backend
    g = torch.Generator().manual_seed(seed)
    feats = (torch.rand(km.n_in, cin, generator=g) - 0.5).to(dtype).to(cuda)
    gout = (torch.rand(km.n_out, cout, generator=g) - 0.5).to(dtype).to(cuda)
    w = ((torch.rand(km.K, cin, cout, generator=g) - 0.5) / cin ** 0.5).to(cuda)
    n0 = _lib.tc_launch_count()
    for out_dtype in (None, torch.float32):
        a = backend._conv_forward(feats, w, km, out_dtype=out_dtype)
        b = backend._conv_forward(feats, w, plain, out_dtype=out_dtype)
        assert torch.equal(a, b), f"forward ({out_dtype}) differs with the tile order"
    a, _ = backend._conv_backward(feats, gout, w, km, need_in=True, need_w=False)
    b, _ = backend._conv_backward(feats, gout, w, plain, need_in=True, need_w=False)
    assert torch.equal(a, b), "dgrad differs with the tile order"
    assert _lib.tc_launch_count() > n0, "did not take the tensor-core path"


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("ks,stride,transpose,cin,cout", [
    (3, 1, False, 32, 32), (2, 2, False, 64, 96), (2, 2, True, 96, 64),
    (3, 1, False, 320, 288),        # more than 256 columns: two launches share the order
])
def test_bitwise_equal_on_manager_maps(ME, cuda, dtype, ks, stride, transpose, cin, cout):
    from minkowskiengine_b200 import backend
    coords = unique_cloud(12000, 32, seed=7 * ks + stride, batches=2)
    km = _maps(ME, coords, cuda, ks, stride, transpose)
    assert km.out_order is not None and km.in_order is not None
    plain = backend._KernelMap(km.out_nbr, km.in_nbr)
    _same_bits(km, plain, cin, cout, dtype, cuda, seed=cin + cout)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("ks,cin,cout", [(3, 64, 64), (2, 32, 272)])
def test_bitwise_equal_with_empty_rows_and_tiles(ME, cuda, dtype, ks, cin, cout):
    from minkowskiengine_b200 import backend
    out_nbr, in_nbr, out_order, in_order = _probe(cuda, ks, 5000, 7001, seed=ks + 10)
    km = backend._KernelMap(out_nbr, in_nbr, orders=(out_order, in_order))
    plain = backend._KernelMap(out_nbr, in_nbr)
    _same_bits(km, plain, cin, cout, dtype, cuda, seed=ks)


def test_empty_side_still_gets_its_order(ME, cuda):
    """An empty x map (a layer whose input was pruned to nothing, onto an existing output map):
    y_nbr is all -1 and its order must still be written — the identity with empty tile masks —
    since the dgrad, and the forward of the swapped (transposed) view, read it over the y rows."""
    from minkowskiengine_b200 import backend
    mx, my = _apart_maps(cuda, 10, 3000, seed=21)
    mx, _, _ = backend._CoordinateMap.build(mx.coords[:0], (1, 1, 1))
    offs = backend._device_offsets(backend.RegionType.HYPER_CUBE, [3] * 3, [1] * 3, (1, 1, 1),
                                   None, cuda)
    out_nbr, in_nbr, out_order, in_order = backend.CoordinateMapManagerGPU_c10._probe(
        mx, my, offs, orders=True)
    assert out_nbr.shape[1] == 0 and in_nbr.shape[1] == my.size
    assert bool((in_nbr == -1).all())
    _check_order(in_nbr, in_order)
    km = backend._KernelMap(out_nbr, in_nbr, orders=(out_order, in_order))
    plain = backend._KernelMap(out_nbr, in_nbr)
    for a, b in ((km, plain), (km.swapped(), plain.swapped())):
        assert a.out_order is not None and a.in_order is not None
        _same_bits(a, b, 64, 32, torch.bfloat16, cuda, seed=3)
    w = torch.rand(27, 64, 32, device=cuda)
    y = backend._conv_forward(torch.zeros(0, 64, dtype=torch.bfloat16, device=cuda), w, km.swapped())
    assert y.shape == (my.size, 32) and not bool(y.any())


@pytest.mark.parametrize("transpose", [False, True])
def test_kernel_reads_the_tile_masks(ME, cuda, transpose):
    """With every tile mask cleared the ordered forward and dgrad run no stage: all-zero outputs.
    (Shows the order is what the kernel walks, not just an argument it receives.)"""
    from minkowskiengine_b200 import backend
    coords = unique_cloud(6000, 24, seed=8)
    km = _maps(ME, coords, cuda, 2, 2, transpose)

    def cleared(order, nbr):
        K, n = nbr.shape
        o = order.clone()
        o[(K + 1) * n:] = 0
        return o

    empty = backend._KernelMap(km.out_nbr, km.in_nbr, orders=(cleared(km.out_order, km.out_nbr),
                                                              cleared(km.in_order, km.in_nbr)))
    g = torch.Generator().manual_seed(1)
    feats = (torch.rand(km.n_in, 32, generator=g) + 0.5).bfloat16().to(cuda)
    gout = (torch.rand(km.n_out, 64, generator=g) + 0.5).bfloat16().to(cuda)
    w = (torch.rand(km.K, 32, 64, generator=g) + 0.5).to(cuda)
    assert bool(backend._conv_forward(feats, w, km).any())
    assert not bool(backend._conv_forward(feats, w, empty).any())
    gi, _ = backend._conv_backward(feats, gout, w, km, need_in=True, need_w=False)
    gi0, _ = backend._conv_backward(feats, gout, w, empty, need_in=True, need_w=False)
    assert bool(gi.any()) and not bool(gi0.any())
