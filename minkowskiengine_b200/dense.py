"""Sparse tensors <-> dense torch tensors (reference: SparseTensor.dense
MinkowskiSparseTensor.py:460-557; dense_coordinates, to_sparse, to_sparse_all,
MinkowskiToDenseTensor MinkowskiOps.py:246-457).  Rows -> dense and dense -> rows are one kernel
each of csrc/dense.cu, each the other's backward; a dense tensor is handed over by its strides, so
any axis order and any view is read or written where it lies."""
import ctypes

import torch
from torch.autograd import Function

from . import _lib
from . import backend as _C
from .common import MinkowskiModuleBase

_MAX_NCOLS = 8


class _DenseDesc(ctypes.Structure):      # == meb200_dense_desc (include/meb200.h)
    _fields_ = [("ncols", ctypes.c_uint32), ("channels", ctypes.c_uint32),
                ("shape", ctypes.c_uint32 * _MAX_NCOLS), ("stride", ctypes.c_int64 * _MAX_NCOLS),
                ("channel_stride", ctypes.c_int64), ("origin", ctypes.c_int32 * _MAX_NCOLS),
                ("step", ctypes.c_int32 * _MAX_NCOLS)]


def _describe(dense, ch_dim, origin=None, step=None):
    """Descriptor of a dense tensor whose axis 0 is the batch and axis `ch_dim` the channels; cell i
    of spatial axis j holds coordinate origin[j] + i * step[j] (default 0 and 1)."""
    _C._assert(dense.is_cuda, "minkowskiengine_b200 runs on CUDA tensors only (no CPU backend, no "
               "fallback)")
    axes = [a for a in range(dense.dim()) if a != ch_dim]
    D = len(axes) - 1
    _C._assert(1 <= D < _MAX_NCOLS, "a dense tensor needs 1 to", _MAX_NCOLS - 1, "spatial axes")
    d = _DenseDesc()
    d.ncols, d.channels = D + 1, dense.size(ch_dim)
    d.channel_stride = dense.stride(ch_dim)
    for j, a in enumerate(axes):
        d.shape[j], d.stride[j] = dense.size(a), dense.stride(a)
        d.origin[j] = 0 if j == 0 or origin is None else int(origin[j - 1])
        d.step[j] = 1 if j == 0 or step is None else int(step[j - 1])
    return d


def rows_to_dense(feats, cmap, dense, ch_dim=1, origin=None, step=None):
    """Fills every element of `dense`: the feature row of the voxel of map `cmap` on a cell, zero
    where there is none (meb200_dense_from_rows)."""
    feats = feats.contiguous()
    _C._assert(feats.dim() == 2 and feats.size(0) == cmap.size, "Invalid in_feat size",
               tuple(feats.shape), "for a map of", cmap.size, "rows")
    _C._assert(feats.dtype == dense.dtype and feats.device == dense.device,
               "features and dense tensor differ in dtype or device")
    d = _describe(dense, ch_dim, origin, step)
    _C._assert(d.channels == feats.size(1), "dense tensor has", d.channels, "channels, features",
               feats.size(1))
    _lib.check(_lib.load().meb200_dense_from_rows(
        _lib.ptr(feats), _lib.dtype_code(feats.dtype), cmap.size, _lib.ptr(cmap.coords),
        _lib.ptr(cmap.table), cmap.capacity, ctypes.byref(d), _lib.ptr(dense),
        _lib.current_stream()))
    return dense


def dense_to_rows(dense, coords, ch_dim=1, origin=None, step=None):
    """[n, C] rows: the cell of `dense` on every int32 coordinate row, zero for a row outside it
    (meb200_dense_to_rows)."""
    d = _describe(dense, ch_dim, origin, step)
    _C._assert(coords.dtype == torch.int32 and coords.is_contiguous() and coords.dim() == 2
               and coords.size(1) == d.ncols and coords.device == dense.device,
               "coordinates must be contiguous int32 [n,", d.ncols, "] on the dense tensor's device")
    out = torch.empty((coords.size(0), d.channels), dtype=dense.dtype, device=dense.device)
    _lib.check(_lib.load().meb200_dense_to_rows(
        _lib.ptr(dense), _lib.dtype_code(dense.dtype), ctypes.byref(d), _lib.ptr(coords),
        coords.size(0), _lib.ptr(out), _lib.current_stream()))
    return out


def nonzero_coordinates(dense, ch_dim=1):
    """int32 [M, D+1] indices of the cells of `dense` with a non-zero channel, in row-major
    (batch, X1..XD) order (meb200_dense_nonzero_*).  One host read: M."""
    d = _describe(dense, ch_dim)
    lib = _lib.load()
    cells = 1
    for j in range(d.ncols):
        cells *= d.shape[j]
    scratch = torch.empty(int(lib.meb200_dense_nonzero_scratch_bytes(cells)), dtype=torch.uint8,
                          device=dense.device)
    m = ctypes.c_uint32(0)
    _lib.check(lib.meb200_dense_nonzero_count(
        _lib.ptr(dense), _lib.dtype_code(dense.dtype), ctypes.byref(d), _lib.ptr(scratch),
        ctypes.byref(m), _lib.current_stream()))
    coords = torch.empty((int(m.value), d.ncols), dtype=torch.int32, device=dense.device)
    if m.value:
        _lib.check(lib.meb200_dense_nonzero_coords(ctypes.byref(d), _lib.ptr(scratch),
                                                   _lib.ptr(coords), _lib.current_stream()))
    return coords


class MinkowskiToDenseFunction(Function):
    """Features of the map `key` -> a contiguous dense tensor of `shape` ([B, C, X1..XD]) whose
    cell i holds coordinate min_coordinate + i * step, step = the tensor stride when
    `contract_stride` else 1.  Voxels outside the volume are cropped (their gradient is zero)."""

    @staticmethod
    def forward(ctx, feats, key, manager, min_coordinate, shape, contract_stride):
        cmap = manager._manager._get(key)
        ctx.cmap, ctx.origin = cmap, list(min_coordinate)
        ctx.step = list(cmap.tensor_stride) if contract_stride else None
        dense = torch.empty(list(shape), dtype=feats.dtype, device=feats.device)
        return rows_to_dense(feats, cmap, dense, 1, ctx.origin, ctx.step)

    @staticmethod
    def backward(ctx, grad_dense):
        return (dense_to_rows(grad_dense, ctx.cmap.coords, 1, ctx.origin, ctx.step),
                None, None, None, None, None)


class MinkowskiDenseToRowsFunction(Function):
    """[n, C] = the cells of dense tensor `x` (batch axis 0, channel axis `ch_dim`) on the distinct
    int32 coordinate rows `coordinates`.  The backward scatters through a table built over the rows
    there, so a forward pass alone pays for none."""

    @staticmethod
    def forward(ctx, x, ch_dim, coordinates):
        ctx.ch_dim, ctx.coordinates = ch_dim, coordinates
        ctx.x_shape, ctx.x_stride = x.shape, x.stride()
        return dense_to_rows(x, coordinates, ch_dim)

    @staticmethod
    def backward(ctx, grad_rows):
        cmap = _C._distinct_map(ctx.coordinates, [1] * (ctx.coordinates.size(1) - 1))
        # laid out as x is when x is dense in memory (channel-last stays channel-last)
        grad = torch.empty_strided(ctx.x_shape, ctx.x_stride, dtype=grad_rows.dtype,
                                   device=grad_rows.device)
        if grad.untyped_storage().nbytes() != grad.numel() * grad.element_size():
            grad = torch.empty(ctx.x_shape, dtype=grad_rows.dtype, device=grad_rows.device)
        return rows_to_dense(grad_rows, cmap, grad, ctx.ch_dim), None, None


def sparse_to_dense(x, shape=None, min_coordinate=None, contract_stride=True):
    """SparseTensor.dense (its docstring is there)."""
    D, C, ts = x.D, x.F.size(1), x.tensor_stride
    if shape is not None:
        assert len(shape) == D + 2, "shape must be [batch, channels, X1..XD]"
        shape = [int(shape[0]), C] + [int(s) for s in shape[2:]]
    stride_out = torch.tensor(ts, dtype=torch.int32)
    if len(x) == 0:
        assert shape is not None, "shape is required to densify an empty tensor"
        return (torch.zeros(shape, dtype=x.dtype, device=x.device),
                torch.zeros(D, dtype=torch.int32, device=x.device), stride_out)
    if min_coordinate is None or shape is None:
        # the one host read: the extent of the coordinates
        lo, hi = torch.aminmax(x.C, dim=0)
        lo, hi = torch.stack([lo, hi]).tolist()
    if min_coordinate is None:
        origin = lo[1:]
        min_out = torch.tensor(origin, dtype=torch.int32, device=x.device)
    else:
        min_out = torch.as_tensor(min_coordinate, device=x.device).int().flatten()
        origin = torch.as_tensor(min_coordinate).flatten().tolist()
        if len(origin) == 1:
            origin = origin * D
        assert len(origin) == D, "min_coordinate must have one entry per spatial axis"
        assert all(o % s == 0 for o, s in zip(origin, ts)), \
            "The minimum coordinates must be divisible by the tensor stride."
    if shape is None:
        step = ts if contract_stride else [1] * D
        shape = [hi[0] + 1, C] + [(h - o) // s + 1 for h, o, s in zip(hi[1:], origin, step)]
    dense = MinkowskiToDenseFunction.apply(x.F, x.coordinate_map_key, x.coordinate_manager,
                                           origin, shape, contract_stride)
    return dense, min_out, stride_out


def dense_coordinates(shape, device=None):
    """int32 [B * prod(X), D+1] coordinates of every cell of a [B, C, X1..XD] tensor in row-major
    (meshgrid indexing="ij") order, built on `device`.  Cache it when the shape does not change."""
    spatial_dim = len(shape) - 2
    assert spatial_dim > 0, "Invalid shape. Shape must be batch x channel x spatial dimensions."
    axes = [torch.arange(s, dtype=torch.int32, device=device) for s in (shape[0], *shape[2:])]
    return torch.stack([g.reshape(-1) for g in torch.meshgrid(*axes, indexing="ij")], 1)


def to_sparse(x, format=None, coordinates=None, device=None):
    r"""Converts a batched dense tensor to a SparseTensor over its non-zero cells (a cell is kept
    when any channel is non-zero), rows in row-major cell order.  Differentiable in `x`.

    :attr:`format`: one letter per axis: 'B' first, one 'C', 'X' elsewhere ("BCXX" for BCHW images,
    "BXXXC" for channel-last volumes); "BCX...X" when None.  `x` is read where it lies, whatever the
    format or strides.

    :attr:`device`: device of the sparse tensor; `x` is moved there first.

    :attr:`coordinates` is accepted and unused, as in the reference.
    """
    from .sparse_tensor import SparseTensor
    assert x.ndim > 2, "Input has 0 spatial dimension."
    assert isinstance(x, torch.Tensor)
    if format is None:
        format = "BC" + "X" * (x.ndim - 2)
    assert x.ndim == len(format), f"Invalid format: {format}. len(format) != x.ndim"
    assert "B" in format and "B" == format[0] and format.count("B") == 1, \
        "The input must have the batch axis and the format must include 'B' indicating the batch axis."
    assert "C" in format and format.count("C") == 1, "The format must indicate the channel axis"
    if device is not None:
        x = x.to(device)
    ch_dim = format.find("C")
    coords = nonzero_coordinates(x.detach(), ch_dim)
    features = MinkowskiDenseToRowsFunction.apply(x, ch_dim, coords)
    return SparseTensor(features=features, coordinates=coords)


def to_sparse_all(dense_tensor, coordinates=None):
    r"""Converts a (differentiable) [B, C, X1..XD] dense tensor to a SparseTensor with a row for
    every cell; `coordinates` defaults to `dense_coordinates(dense_tensor.shape)`."""
    from .sparse_tensor import SparseTensor
    spatial_dim = dense_tensor.ndim - 2
    assert spatial_dim > 0, "Invalid shape. Shape must be batch x channel x spatial dimensions."
    if coordinates is None:
        coordinates = dense_coordinates(dense_tensor.shape, dense_tensor.device)
    feat_tensor = dense_tensor.permute(0, *(2 + i for i in range(spatial_dim)), 1)
    return SparseTensor(feat_tensor.reshape(-1, dense_tensor.size(1)), coordinates,
                        device=dense_tensor.device)


class MinkowskiToDenseTensor(MinkowskiModuleBase):
    r"""Converts a (differentiable) SparseTensor to a [B, C, X1..XD] torch tensor of `shape` (the
    extent of the coordinates when None); see `SparseTensor.dense`."""

    def __init__(self, shape=None):
        super().__init__()
        self.shape = shape

    def forward(self, input):
        return input.dense(shape=self.shape)[0]

    def __repr__(self):
        return self.__class__.__name__ + "()"
