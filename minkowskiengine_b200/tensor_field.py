"""`TensorField`: features on points with float coordinates, quantised to a `SparseTensor` with
`.sparse()` and mapped back with `SparseTensor.slice` (reference: MinkowskiTensorField.py).

The reductions between points and voxels run in csrc/field.cu: the points are grouped by voxel once
per (field, map) (`meb200_group_by_row`, cached by the manager) and every output row walks its
points in field order, so results are bit-identical run to run and bf16 / fp16 sums are
accumulated in fp32 and rounded once."""
import torch
from torch.autograd import Function

from . import _lib
from . import backend as _C
from .backend import CoordinateMapKey
from .common import convert_to_int_list
from .coordinate_manager import CoordinateManager
from .enums import CoordinateMapType
from .interpolation import interp_adjoint
from .sparse_tensor import (COORDINATE_KEY_DIFFERENT_ERROR, COORDINATE_MANAGER_DIFFERENT_ERROR,
                            SparseTensor, SparseTensorOperationMode, SparseTensorQuantizationMode,
                            Tensor, global_coordinate_manager, set_global_coordinate_manager,
                            sparse_tensor_operation_mode)

_Q = SparseTensorQuantizationMode
_MODES = {_Q.UNWEIGHTED_SUM: _lib.FIELD_SUM, _Q.UNWEIGHTED_AVERAGE: _lib.FIELD_AVG,
          _Q.MAX_POOL: _lib.FIELD_MAX, _Q.RANDOM_SUBSAMPLE: _lib.FIELD_SUBSAMPLE}
SPLAT_ERROR = ("SPLAT_LINEAR_INTERPOLATION is not a quantisation mode of TensorField or .sparse(), "
               "as in the reference: call TensorField.splat() to splat the points linearly onto "
               "their 2^D corners")


class MinkowskiFieldQuantizationFunction(Function):
    """Points -> voxels of one field-to-map relation (`backend._FieldToSparse`) in one of the four
    quantisation modes, with its backward."""

    @staticmethod
    def forward(ctx, feats, f2s, mode):
        feats = feats.contiguous()
        ctx.f2s, ctx.mode, ctx.argmax = f2s, mode, None
        if mode == _lib.FIELD_SUBSAMPLE:
            return _C.gather_rows(feats, f2s.first_points(), f2s.M)
        out, ctx.argmax = _C.field_reduce(feats, f2s.group(), f2s.M, mode)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        f2s, mode = ctx.f2s, ctx.mode
        g = grad_out.contiguous()
        if mode == _lib.FIELD_SUM:
            grad = _C.gather_rows(g, f2s.inverse, f2s.inverse.numel())
        elif mode == _lib.FIELD_AVG:
            grad = _C.field_expand(g, f2s.inverse, mode, start=f2s.group()[0])
        elif mode == _lib.FIELD_MAX:
            grad = _C.field_expand(g, f2s.inverse, mode, argmax=ctx.argmax)
        else:
            grad = _C.field_expand(g, f2s.inverse, mode, unique_index=f2s.first_points())
        return grad, None, None


class MinkowskiSliceFunction(Function):
    """Voxels -> points: out[i] = F[inverse[i]] (0 where a point has no voxel); the backward adds
    the gradients of the points of each voxel in field order."""

    @staticmethod
    def forward(ctx, feats, f2s):
        ctx.f2s = f2s
        return _C.gather_rows(feats, f2s.inverse, f2s.inverse.numel())

    @staticmethod
    def backward(ctx, grad_out):
        f2s = ctx.f2s
        grad, _ = _C.field_reduce(grad_out, f2s.group(), f2s.M, _lib.FIELD_SUM)
        return grad, None


class MinkowskiSplatFunction(Function):
    """Points -> the M rows of a splat map: out[r] = sum of w * F[q] over the (point q, corner) pairs
    of row r in pair order (the interpolation backward's reduction), fp32 accumulation, one
    rounding.  The backward is the interpolation forward with the same rows and weights."""

    @staticmethod
    def forward(ctx, feats, rec, M):
        rows, w, group = rec
        ctx.rec = rec
        return interp_adjoint(feats, rows, w, M, group)

    @staticmethod
    def backward(ctx, grad_out):
        rows, w, _ = ctx.rec
        return _C.interp_forward(grad_out.contiguous(), rows, w), None, None


def _new_manager(D, allocator_type, minkowski_algorithm):
    if sparse_tensor_operation_mode() == SparseTensorOperationMode.SHARE_COORDINATE_MANAGER:
        manager = global_coordinate_manager()
        if manager is None:
            manager = CoordinateManager(D=D, coordinate_map_type=CoordinateMapType.CUDA,
                                        allocator_type=allocator_type,
                                        minkowski_algorithm=minkowski_algorithm)
            set_global_coordinate_manager(manager)
        return manager
    return CoordinateManager(D=D, coordinate_map_type=CoordinateMapType.CUDA,
                             allocator_type=allocator_type, minkowski_algorithm=minkowski_algorithm)


class TensorField(Tensor):
    def __init__(self, features: torch.Tensor, coordinates: torch.Tensor = None, tensor_stride=1,
                 coordinate_field_map_key: CoordinateMapKey = None,
                 coordinate_manager: CoordinateManager = None,
                 quantization_mode: SparseTensorQuantizationMode = _Q.UNWEIGHTED_AVERAGE,
                 allocator_type=None, minkowski_algorithm=None, requires_grad=None, device=None):
        assert isinstance(features, torch.Tensor), "Features must be a torch.Tensor"
        assert features.ndim == 2, \
            f"The feature should be a matrix, The input feature is an order-{features.ndim} tensor."
        assert isinstance(quantization_mode, SparseTensorQuantizationMode)
        if quantization_mode == _Q.SPLAT_LINEAR_INTERPOLATION:
            raise NotImplementedError(SPLAT_ERROR)
        assert quantization_mode in _MODES, "invalid quantization mode"
        self.quantization_mode = quantization_mode
        if coordinates is not None:
            assert isinstance(coordinates, torch.Tensor)
        if coordinate_field_map_key is not None:
            assert isinstance(coordinate_field_map_key, CoordinateMapKey)
            assert coordinate_manager is not None, \
                "Must provide coordinate_manager if coordinate_field_map_key is provided"
            assert coordinates is None, \
                "Must not provide coordinates if coordinate_field_map_key is provided"
        if coordinate_manager is not None:
            assert isinstance(coordinate_manager, CoordinateManager)
        if coordinates is None and (coordinate_field_map_key is None or coordinate_manager is None):
            raise ValueError("Either coordinates or (coordinate_field_map_key, coordinate_manager) "
                             "pair must be provided.")
        if device is not None:
            features = features.to(device)
            if coordinates is not None:
                coordinates = coordinates.to(device)
        if not features.is_cuda or (coordinates is not None and not coordinates.is_cuda):
            raise RuntimeError(
                "minkowskiengine_b200 runs on CUDA tensors only: pass device='cuda' or CUDA "
                "coordinates/features (no CPU backend, no fallback).")
        _lib.dtype_code(features.dtype)   # fp32 / bf16 / fp16 only
        self._D = coordinates.size(1) - 1 if coordinates is not None else coordinate_manager.D
        if coordinate_manager is None:
            coordinate_manager = _new_manager(self._D, allocator_type, minkowski_algorithm)
        self._manager = coordinate_manager
        if coordinates is not None:
            assert features.shape[0] == coordinates.shape[0], \
                "The number of rows in features and coordinates must match."
            coordinates = coordinates.float().contiguous()
            coordinate_field_map_key = self._manager.insert_field(
                coordinates, convert_to_int_list(tensor_stride, self._D), "")
        else:
            assert coordinate_field_map_key.is_key_set(), \
                "The coordinate field map key must be valid."
        if requires_grad is not None:
            features.requires_grad_(requires_grad)
        self._F = features
        self._C = coordinates
        self.coordinate_field_map_key = coordinate_field_map_key
        self._batch_rows = None
        self._inverse_mapping = {}   # map key -> backend._FieldToSparse
        self._splat = {}             # splat map key -> (rows, weights, grouping by row)

    @property
    def coordinate_key(self):
        return self.coordinate_field_map_key

    @property
    def coordinate_map_key(self):
        return self.coordinate_field_map_key

    @property
    def coordinates(self):
        if self._C is None:
            self._C = self._manager.get_coordinate_field(self.coordinate_field_map_key)
        return self._C

    @property
    def _batchwise_row_indices(self):
        if self._batch_rows is None:
            b = _batch_index(self.C[:, 0])
            nb = int(b.max().item()) + 1 if b.numel() else 0
            self._batch_rows = [torch.nonzero(b == i).flatten() for i in range(nb)]
        return self._batch_rows

    def _like(self, feats):
        return TensorField(feats, coordinate_field_map_key=self.coordinate_field_map_key,
                           coordinate_manager=self._manager, quantization_mode=self.quantization_mode)

    def _binary(self, other, fn, op):
        if isinstance(other, TensorField):
            assert self._manager == other._manager, COORDINATE_MANAGER_DIFFERENT_ERROR
            assert self.coordinate_field_map_key == other.coordinate_field_map_key, \
                COORDINATE_KEY_DIFFERENT_ERROR
            return self._like(fn(self._F, other._F))
        assert isinstance(other, (torch.Tensor, int, float)), \
            "a TensorField combines with a TensorField on the same field key or a tensor"
        return self._like(fn(self._F, other))

    def _record(self, key):
        """The backend._FieldToSparse relation of this field and map `key`."""
        mgr = self._manager._manager
        fk = self.coordinate_field_map_key
        rec = self._inverse_mapping.get(key)
        if rec is not None:
            return rec
        if mgr.exists_field_to_sparse(fk, key):
            rec = mgr._field_sparse_record(fk, key)
        else:
            # a map this field did not make: the field's stride-1 map composed with the stride map
            # from it to `key` (reference: MinkowskiTensorField.py:408-450)
            one = [k for k in mgr.field_to_sparse_keys(fk)
                   if all(s == 1 for s in k.get_tensor_stride())]
            one_key = one[0] if one else mgr.field_to_sparse_insert_and_map(fk, [1] * self._D)[0]
            base = self._record(one_key)
            in_rows, out_rows = mgr.stride_map(one_key, key)
            _C._assert(in_rows.numel() == mgr.size(one_key),
                       "the map", key, "is not a strided map of the field's voxels")
            # a point the stride-1 map lacks (-1) has no row at `key` either
            inv = torch.where(base.inverse >= 0, out_rows[base.inverse.clamp(min=0)],
                              base.inverse)
            rec = _C._FieldToSparse(inv, mgr.size(key))
        self._inverse_mapping[key] = rec
        return rec

    def inverse_mapping(self, sparse_tensor_map_key: CoordinateMapKey):
        """int64 [N]: the row of map `sparse_tensor_map_key` that holds each point."""
        return self._record(sparse_tensor_map_key).inverse

    def sparse(self, tensor_stride=1, coordinate_map_key: CoordinateMapKey = None,
               quantization_mode: SparseTensorQuantizationMode = None):
        """Quantises the field to a SparseTensor: onto a new map at `tensor_stride` (cached per field
        and stride), or onto the existing map `coordinate_map_key`."""
        mode = self.quantization_mode if quantization_mode is None else quantization_mode
        if mode == _Q.SPLAT_LINEAR_INTERPOLATION:
            raise NotImplementedError(SPLAT_ERROR)
        assert mode in _MODES, "invalid quantization mode"
        mgr = self._manager
        if coordinate_map_key is None:
            key, (_, inv) = mgr.field_to_sparse_insert_and_map(
                self.coordinate_field_map_key, convert_to_int_list(tensor_stride, self._D))
            rec = self._record(key)
            if len(inv) == 0:
                # no two points share a voxel: the rows are the points, in order
                return SparseTensor(self._F, coordinate_map_key=key, coordinate_manager=mgr)
        else:
            key = coordinate_map_key
            mgr.field_to_sparse_map(self.coordinate_field_map_key, key)
            rec = self._record(key)
        assert rec.M > 0, f"Invalid out coordinate map key. Found {rec.M} elements."
        feats = MinkowskiFieldQuantizationFunction.apply(self._F, rec, _MODES[mode])
        return SparseTensor(feats, coordinate_map_key=key, coordinate_manager=mgr)

    def splat(self):
        """Linear splatting, the adjoint of multilinear interpolation (reference:
        MinkowskiTensorField.py:381-406): every point adds w * F to each of its 2^D corners
        floor(x) + {0,1}^D, w = prod_j (1 - |x_j - c_j|), on a new map at tensor stride 1 (rows
        in order of first occurrence; a corner of weight 0 is a row too).  Use
        `y.interpolate(field)` to bring a network's output back to the points."""
        mgr = self._manager._manager
        key = mgr.splat_insert_and_map(self.coordinate_field_map_key)
        M = mgr.size(key)
        rows, w = mgr._interp_map(key, self.C.float().contiguous())
        rec = (rows, w, _C.group_by_row(rows.view(-1), M))
        self._splat[key] = rec
        feats = MinkowskiSplatFunction.apply(self._F, rec, M)
        return SparseTensor(feats, coordinate_map_key=key, coordinate_manager=self._manager)

    def __repr__(self):
        return (self.__class__.__name__ + "(\n  coordinates=" + str(self.C) + "\n  features="
                + str(self.F) + "\n  coordinate_field_map_key=" + str(self.coordinate_field_map_key)
                + "\n  coordinate_manager=" + str(self._manager) + "  spatial dimension="
                + str(self._D) + ")")


def same_kind(input, feats):
    """`feats` on the coordinates of `input`, as a tensor of its kind: a TensorField on its field key
    (for the point-wise layers of a point network) or a SparseTensor on its map."""
    if isinstance(input, TensorField):
        return input._like(feats)
    return SparseTensor(feats, coordinate_map_key=input.coordinate_map_key,
                        coordinate_manager=input.coordinate_manager)


def _batch_index(b):
    """Batch index of float batch coordinates, rounded half away from zero as the quantisation's
    lroundf rounds (torch.round rounds half to even)."""
    t = torch.trunc(b)
    return (t + torch.sign(b) * ((b - t).abs() >= 0.5)).long()


def _slice(sparse, X):
    """(features on the points of X, TensorField constructor arguments, the field-to-map
    relation) of SparseTensor.slice."""
    assert X.quantization_mode in (_Q.RANDOM_SUBSAMPLE, _Q.UNWEIGHTED_AVERAGE), \
        "slice only available for sparse tensors with quantization RANDOM_SUBSAMPLE or " \
        "UNWEIGHTED_AVERAGE"
    if isinstance(X, TensorField):
        assert X.coordinate_manager == sparse.coordinate_manager, \
            COORDINATE_MANAGER_DIFFERENT_ERROR
        rec = X._record(sparse.coordinate_map_key)
        feats = MinkowskiSliceFunction.apply(sparse.F, rec)
        return feats, rec, dict(coordinate_field_map_key=X.coordinate_field_map_key,
                           coordinate_manager=X.coordinate_manager,
                           quantization_mode=X.quantization_mode)
    if isinstance(X, SparseTensor):
        assert X.coordinate_map_key == sparse.coordinate_map_key, \
            "Slice can only be applied on the same coordinates (coordinate_map_key)"
        inv = X.inverse_mapping
        rec = _C._FieldToSparse(inv, len(sparse))
        feats = MinkowskiSliceFunction.apply(sparse.F, rec)
        # a byte copy of the int32 rows through the feature gather
        coords = _C.gather_rows(sparse.C.view(torch.float32), inv, inv.numel())
        coords = coords.view(torch.int32).float()
        return feats, rec, dict(coordinates=coords, coordinate_manager=sparse.coordinate_manager,
                           quantization_mode=sparse.quantization_mode)
    raise ValueError("Invalid input. The input must be an instance of TensorField or SparseTensor.")


def slice_sparse(sparse, X):
    feats, _, kw = _slice(sparse, X)
    return TensorField(feats, **kw)


def cat_slice_sparse(sparse, X):
    feats, rec, kw = _slice(sparse, X)
    if isinstance(X, SparseTensor):
        # X's features are per voxel: they reach the points through the same inverse map
        own = MinkowskiSliceFunction.apply(X.F, rec)
    else:
        own = X.F
    return TensorField(torch.cat((feats, own), dim=1), **kw)
