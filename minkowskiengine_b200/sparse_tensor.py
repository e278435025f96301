"""`SparseTensor`: COO features + a coordinate-map key inside a `CoordinateManager`
(reference: MinkowskiSparseTensor.py:48-345, MinkowskiTensor.py:125-604)."""
import copy
import warnings
from enum import Enum

import torch

from ._lib import UNION_ADD as _UNION_ADD, UNION_DIV as _UNION_DIV, UNION_MUL as _UNION_MUL, \
    UNION_SUB as _UNION_SUB
from .backend import CoordinateMapKey
from .common import convert_to_int_list
from .coordinate_manager import CoordinateManager
from .enums import CoordinateMapType, GPUMemoryAllocatorType, MinkowskiAlgorithm


class SparseTensorOperationMode(Enum):
    SEPARATE_COORDINATE_MANAGER = 0
    SHARE_COORDINATE_MANAGER = 1


class SparseTensorQuantizationMode(Enum):
    RANDOM_SUBSAMPLE = 0
    UNWEIGHTED_AVERAGE = 1
    UNWEIGHTED_SUM = 2
    NO_QUANTIZATION = 3
    MAX_POOL = 4
    SPLAT_LINEAR_INTERPOLATION = 5


_sparse_tensor_operation_mode = SparseTensorOperationMode.SEPARATE_COORDINATE_MANAGER
_global_coordinate_manager = None

COORDINATE_MANAGER_DIFFERENT_ERROR = (
    "SparseTensors must share the same coordinate manager for this operation.")
COORDINATE_KEY_DIFFERENT_ERROR = "SparseTensors must have the same coordinate_map_key."


def set_sparse_tensor_operation_mode(operation_mode: SparseTensorOperationMode):
    assert isinstance(operation_mode, SparseTensorOperationMode)
    global _sparse_tensor_operation_mode
    _sparse_tensor_operation_mode = operation_mode


def sparse_tensor_operation_mode() -> SparseTensorOperationMode:
    return copy.deepcopy(_sparse_tensor_operation_mode)


def global_coordinate_manager():
    return _global_coordinate_manager


def set_global_coordinate_manager(coordinate_manager):
    global _global_coordinate_manager
    _global_coordinate_manager = coordinate_manager


def clear_global_coordinate_manager():
    global _global_coordinate_manager
    _global_coordinate_manager = None


class Tensor:
    """Shared behaviour of sparse tensors (reference: MinkowskiTensor.py:125-604)."""

    @property
    def coordinate_manager(self):
        return self._manager

    @property
    def tensor_stride(self):
        return self.coordinate_map_key.get_tensor_stride()

    @property
    def C(self):
        return self.coordinates

    @property
    def coordinates(self):
        if self._C is None:
            self._C = self._manager.get_coordinates(self.coordinate_map_key)
        return self._C

    @property
    def F(self):
        return self._F

    @property
    def features(self):
        return self._F

    @property
    def D(self):
        return self._D

    @property
    def dimension(self):
        return self._D

    @property
    def requires_grad(self):
        return self._F.requires_grad

    def requires_grad_(self, requires_grad: bool = True):
        self._F.requires_grad_(requires_grad)

    @property
    def dtype(self):
        return self._F.dtype

    @property
    def device(self):
        return self._F.device

    @property
    def shape(self):
        return self._F.shape

    def size(self):
        return self._F.size()

    def __len__(self):
        return len(self._F)

    def float(self):
        self._F = self._F.float()
        return self

    def double(self):
        self._F = self._F.double()
        return self

    def get_device(self):
        return self._F.get_device()

    def _like(self, feats):
        return self.__class__(feats, coordinate_map_key=self.coordinate_map_key,
                              coordinate_manager=self._manager)

    def _binary(self, other, fn, op):
        if isinstance(other, Tensor):
            assert self._manager == other._manager, COORDINATE_MANAGER_DIFFERENT_ERROR
            if self.coordinate_map_key != other.coordinate_map_key:
                return self._binary_union(other, op)
            return self._like(fn(self._F, other._F))
        return self._like(fn(self._F, other))

    def _binary_union(self, other, op):
        """op over the union of the two coordinate maps (reference: MinkowskiTensor.py:522-540):
        rows only in self keep self's features, rows only in other give op(0, other), rows in both
        op(self, other).  Rows: self's in order, then other's new rows in order.  Mixed dtypes are
        computed in their promoted dtype and the result has self's dtype, as in the reference."""
        from .union import MinkowskiBinaryFunction
        out_key = CoordinateMapKey(self.coordinate_map_key.get_coordinate_size())
        dt = torch.promote_types(self._F.dtype, other._F.dtype)
        out = MinkowskiBinaryFunction.apply(op, [self.coordinate_map_key, other.coordinate_map_key],
                                            out_key, self._manager, self._F.to(dt), other._F.to(dt))
        return self.__class__(out.to(self._F.dtype), coordinate_map_key=out_key,
                              coordinate_manager=self._manager)

    def __add__(self, other):
        return self._binary(other, lambda a, b: a + b, _UNION_ADD)

    __radd__ = __add__

    def __sub__(self, other):
        return self._binary(other, lambda a, b: a - b, _UNION_SUB)

    def __mul__(self, other):
        return self._binary(other, lambda a, b: a * b, _UNION_MUL)

    __rmul__ = __mul__

    def __truediv__(self, other):
        return self._binary(other, lambda a, b: a / b, _UNION_DIV)

    def __neg__(self):
        return self._like(-self._F)

    def __iadd__(self, other):
        """In-place add; both operands must live on the same coordinate map
        (reference: MinkowskiTensor.py:483-494)."""
        if isinstance(other, Tensor):
            assert self._manager == other._manager, COORDINATE_MANAGER_DIFFERENT_ERROR
            assert self.coordinate_map_key == other.coordinate_map_key, \
                COORDINATE_KEY_DIFFERENT_ERROR
            self._F += other._F
        else:
            self._F += other
        return self

    def __isub__(self, other):
        if isinstance(other, Tensor):
            assert self._manager == other._manager, COORDINATE_MANAGER_DIFFERENT_ERROR
            assert self.coordinate_map_key == other.coordinate_map_key, \
                COORDINATE_KEY_DIFFERENT_ERROR
            self._F -= other._F
        else:
            self._F -= other
        return self

    def detach(self):
        return self._like(self._F.detach())

    # -- batch decomposition (torch index ops on the batch column) --------------------
    @property
    def _batchwise_row_indices(self):
        if self._batch_rows is None:
            b = self.C[:, 0]
            nb = int(b.max().item()) + 1 if b.numel() else 0
            self._batch_rows = [torch.nonzero(b == i).flatten() for i in range(nb)]
        return self._batch_rows

    @property
    def decomposition_permutations(self):
        return self._batchwise_row_indices

    @property
    def decomposed_coordinates(self):
        return [self.C[r, 1:] for r in self._batchwise_row_indices]

    @property
    def decomposed_features(self):
        return [self._F[r] for r in self._batchwise_row_indices]

    @property
    def decomposed_coordinates_and_features(self):
        rows = self._batchwise_row_indices
        return [self.C[r, 1:] for r in rows], [self._F[r] for r in rows]

    def coordinates_at(self, batch_index):
        return self.C[self._batchwise_row_indices[batch_index], 1:]

    def features_at(self, batch_index):
        return self._F[self._batchwise_row_indices[batch_index]]

    def __repr__(self):
        return (self.__class__.__name__ + "(\n  coordinates=" + str(self.C) + "\n  features="
                + str(self.F) + "\n  coordinate_map_key=" + str(self.coordinate_map_key)
                + "\n  coordinate_manager=" + str(self._manager) + "  spatial dimension="
                + str(self._D) + ")")


class SparseTensor(Tensor):
    def __init__(self, features: torch.Tensor, coordinates: torch.Tensor = None,
                 tensor_stride=1, coordinate_map_key: CoordinateMapKey = None,
                 coordinate_manager: CoordinateManager = None,
                 quantization_mode: SparseTensorQuantizationMode =
                 SparseTensorQuantizationMode.RANDOM_SUBSAMPLE,
                 allocator_type: GPUMemoryAllocatorType = None,
                 minkowski_algorithm: MinkowskiAlgorithm = None, requires_grad=None,
                 device=None):
        assert isinstance(features, torch.Tensor), "Features must be a torch.Tensor"
        assert features.ndim == 2, \
            f"The feature should be a matrix, The input feature is an order-{features.ndim} tensor."
        assert isinstance(quantization_mode, SparseTensorQuantizationMode)
        self.quantization_mode = quantization_mode
        if coordinates is not None:
            assert isinstance(coordinates, torch.Tensor)
        if coordinate_map_key is not None:
            assert isinstance(coordinate_map_key, CoordinateMapKey)
            assert coordinate_manager is not None, \
                "Must provide coordinate_manager if coordinate_map_key is provided"
            assert coordinates is None, \
                "Must not provide coordinates if coordinate_map_key is provided"
        if coordinate_manager is not None:
            assert isinstance(coordinate_manager, CoordinateManager)
        if coordinates is None and (coordinate_map_key is None or coordinate_manager is None):
            raise ValueError("Either coordinates or (coordinate_map_key, coordinate_manager) "
                             "pair must be provided.")

        if device is not None:
            features = features.to(device)
            if coordinates is not None:
                coordinates = coordinates.to(device)

        self._D = coordinates.size(1) - 1 if coordinates is not None else coordinate_manager.D
        self._inverse_mapping = None
        self._num_input_rows = features.shape[0]
        self.unique_index = None
        if coordinate_manager is None:
            if not coordinates.is_cuda:
                raise RuntimeError(
                    "minkowskiengine_b200 runs on CUDA tensors only: pass device='cuda' or CUDA "
                    "coordinates/features (no CPU backend, no fallback).")
            if sparse_tensor_operation_mode() == SparseTensorOperationMode.SHARE_COORDINATE_MANAGER:
                coordinate_manager = global_coordinate_manager()
                if coordinate_manager is None:
                    coordinate_manager = CoordinateManager(
                        D=self._D, coordinate_map_type=CoordinateMapType.CUDA,
                        allocator_type=allocator_type, minkowski_algorithm=minkowski_algorithm)
                    set_global_coordinate_manager(coordinate_manager)
            else:
                coordinate_manager = CoordinateManager(
                    D=self._D, coordinate_map_type=CoordinateMapType.CUDA,
                    allocator_type=allocator_type, minkowski_algorithm=minkowski_algorithm)
        self._manager = coordinate_manager

        if coordinates is not None:
            assert features.shape[0] == coordinates.shape[0], \
                "The number of rows in features and coordinates must match."
            assert features.is_cuda == coordinates.is_cuda, \
                "Features and coordinates must have the same backend."
            coordinate_map_key = CoordinateMapKey(convert_to_int_list(tensor_stride, self._D), "")
            coordinates, features, coordinate_map_key = self.initialize_coordinates(
                coordinates, features, coordinate_map_key)
        else:
            assert coordinate_map_key.is_key_set(), "The coordinate key must be valid."

        if requires_grad is not None:
            features.requires_grad_(requires_grad)

        self._F = features
        self._C = coordinates
        self.coordinate_map_key = coordinate_map_key
        self._batch_rows = None

    @property
    def coordinate_key(self):
        return self.coordinate_map_key

    @property
    def inverse_mapping(self):
        if self._inverse_mapping is None:
            self._inverse_mapping = torch.arange(self._num_input_rows, dtype=torch.int64,
                                                 device=self._F.device)
        return self._inverse_mapping

    def initialize_coordinates(self, coordinates, features, coordinate_map_key):
        """reference: MinkowskiSparseTensor.py:293-345"""
        if coordinates.dtype != torch.int32:
            warnings.warn("coordinates implicitly converted to torch.IntTensor. To remove this "
                          "warning, use `.int()` to convert the coords into an torch.IntTensor")
            coordinates = torch.floor(coordinates).int()
        coordinates = coordinates.contiguous()
        coordinate_map_key, (unique_index, inverse_mapping) = self._manager.insert_and_map(
            coordinates, *coordinate_map_key.get_key())
        self._num_input_rows = coordinates.shape[0]
        self.unique_index = unique_index
        if len(inverse_mapping) == 0:
            # no duplicate coordinates: rows are kept as given
            self._inverse_mapping = None
            return coordinates, features, coordinate_map_key
        coordinates = self._manager.get_coordinates(coordinate_map_key)
        self._inverse_mapping = inverse_mapping
        mode = self.quantization_mode
        if mode in (SparseTensorQuantizationMode.UNWEIGHTED_SUM,
                    SparseTensorQuantizationMode.UNWEIGHTED_AVERAGE):
            m = len(unique_index)
            acc = torch.zeros((m, features.shape[1]), dtype=features.dtype,
                              device=features.device)
            acc.index_add_(0, inverse_mapping, features)
            if mode == SparseTensorQuantizationMode.UNWEIGHTED_AVERAGE:
                cnt = torch.zeros(m, dtype=features.dtype, device=features.device)
                cnt.index_add_(0, inverse_mapping, torch.ones_like(features[:, 0]))
                acc = acc / cnt.unsqueeze(1)
            features = acc
        elif mode == SparseTensorQuantizationMode.RANDOM_SUBSAMPLE:
            features = features[unique_index]
        return coordinates, features, coordinate_map_key

    # -- tensor fields (reference: MinkowskiSparseTensor.py:559-718) -----------------------
    def slice(self, X):
        """Features of this tensor on the points of X (a TensorField or the SparseTensor whose
        quantisation made this map), as a TensorField in X's point order."""
        from .tensor_field import slice_sparse
        return slice_sparse(self, X)

    def cat_slice(self, X):
        """slice(X) with X's own features concatenated after this tensor's."""
        from .tensor_field import cat_slice_sparse
        return cat_slice_sparse(self, X)

    def interpolate(self, X):
        """Features interpolated multilinearly at the points of TensorField X."""
        from .tensor_field import TensorField
        assert isinstance(X, TensorField)
        return TensorField(self.features_at_coordinates(X.C),
                           coordinate_field_map_key=X.coordinate_field_map_key,
                           coordinate_manager=X.coordinate_manager)

    def features_at_coordinates(self, query_coordinates: torch.Tensor):
        """[N, C] features interpolated at float32 / float64 points [N, D+1] (rows of zeros where no
        corner of a point is in the map)."""
        from .interpolation import MinkowskiInterpolationFunction
        return MinkowskiInterpolationFunction.apply(self._F, query_coordinates,
                                                    self.coordinate_map_key, self._manager)[0]

    def dense(self, shape=None, min_coordinate=None, contract_stride=True):
        """Dense [B, C, X1..XD] tensor (reference: MinkowskiSparseTensor.py:347-448)."""
        ts = torch.tensor(self.tensor_stride, device=self.device, dtype=torch.int64)
        coords = self.C.long()
        b = coords[:, 0]
        xyz = coords[:, 1:]
        if min_coordinate is None:
            min_coordinate = xyz.min(0).values if len(xyz) else torch.zeros_like(ts)
        else:
            min_coordinate = torch.as_tensor(min_coordinate, device=self.device).long().flatten()
        xyz = xyz - min_coordinate
        if contract_stride:
            xyz = xyz // ts
        nb = int(b.max().item()) + 1 if len(b) else 0
        spatial = (xyz.max(0).values + 1).tolist() if len(xyz) else [0] * self._D
        if shape is not None:
            nb, spatial = shape[0], list(shape[2:])
        dense = torch.zeros([nb, self._F.size(1)] + spatial, dtype=self.dtype, device=self.device)
        idx = (b,) + tuple(xyz[:, i] for i in range(self._D))
        dense.permute(0, *range(2, 2 + self._D), 1)[idx] = self._F
        return dense, min_coordinate.int(), torch.tensor(self.tensor_stride, dtype=torch.int32)


def _get_coordinate_map_key(input: SparseTensor, coordinates=None, tensor_stride=1,
                            expand_coordinates: bool = False):
    """reference: MinkowskiSparseTensor.py:754-783"""
    if coordinates is not None and not expand_coordinates:
        assert isinstance(coordinates, (CoordinateMapKey, torch.Tensor, SparseTensor))
        if isinstance(coordinates, torch.Tensor):
            assert coordinates.ndim == 2
            key = CoordinateMapKey(convert_to_int_list(tensor_stride, coordinates.size(1) - 1), "")
            key, _ = input._manager.insert_and_map(coordinates.contiguous(), *key.get_key())
        elif isinstance(coordinates, SparseTensor):
            key = coordinates.coordinate_map_key
        else:
            key = coordinates
        return key
    return CoordinateMapKey(input.coordinate_map_key.get_coordinate_size())
