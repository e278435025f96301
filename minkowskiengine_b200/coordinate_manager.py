"""`CoordinateManager`: the Python face of the coordinate-map manager
(reference: MinkowskiCoordinateManager.py:107-440)."""
import os
import warnings
from collections.abc import Sequence
from typing import Tuple, Union

import numpy as np
import torch

from . import backend as _C
from .backend import CoordinateMapKey
from .common import convert_to_int_list
from .enums import (CoordinateMapType, GPUMemoryAllocatorType, MinkowskiAlgorithm, RegionType)

CPU_COUNT = os.cpu_count() or 1

_allocator_type = GPUMemoryAllocatorType.PYTORCH
_coordinate_map_type = CoordinateMapType.CUDA
_minkowski_algorithm = MinkowskiAlgorithm.DEFAULT


def set_coordinate_map_type(coordinate_map_type: CoordinateMapType):
    global _coordinate_map_type
    _coordinate_map_type = coordinate_map_type


def set_gpu_allocator(backend: GPUMemoryAllocatorType):
    """Accepted for API parity (MinkowskiCoordinateManager.py:63-89); all device memory
    here comes from torch's caching allocator."""
    assert isinstance(backend, GPUMemoryAllocatorType)
    global _allocator_type
    _allocator_type = backend


def set_memory_manager_backend(backend: GPUMemoryAllocatorType):
    warnings.warn("`set_memory_manager_backend` has been deprecated. Use `set_gpu_allocator`.",
                  DeprecationWarning)
    set_gpu_allocator(backend)


class CoordsManager:
    def __init__(*args, **kwargs):
        raise DeprecationWarning(
            "`CoordsManager` has been deprecated. Use `CoordinateManager` instead.")


class CoordinateManager:
    def __init__(self, D: int = 0, num_threads: int = -1,
                 coordinate_map_type: CoordinateMapType = None,
                 allocator_type: GPUMemoryAllocatorType = None,
                 minkowski_algorithm: MinkowskiAlgorithm = None):
        if D < 1:
            raise ValueError(f"Invalid rank D > 0, D = {D}.")
        if num_threads < 0:
            num_threads = min(CPU_COUNT, 20)
        coordinate_map_type = coordinate_map_type or _coordinate_map_type
        allocator_type = allocator_type or _allocator_type
        minkowski_algorithm = minkowski_algorithm or _minkowski_algorithm
        if coordinate_map_type == CoordinateMapType.CPU:
            raise RuntimeError(
                "minkowskiengine_b200 provides the CUDA coordinate manager only "
                "(CoordinateMapManagerGPU_*); CPU tensors are not supported and there is no "
                "fallback path. Move coordinates and features to a CUDA device.")
        postfix = "GPU" + ("_default" if allocator_type == GPUMemoryAllocatorType.CUDA else "_c10")
        self.D = D
        self.minkowski_algorithm = minkowski_algorithm
        self._CoordinateManagerClass = getattr(_C, "CoordinateMapManager" + postfix)
        self._manager = self._CoordinateManagerClass(minkowski_algorithm, num_threads)

    def insert_and_map(self, coordinates: torch.Tensor,
                       tensor_stride: Union[int, Sequence, np.ndarray] = 1,
                       string_id: str = "") -> Tuple[CoordinateMapKey, Tuple[torch.Tensor, torch.Tensor]]:
        tensor_stride = convert_to_int_list(tensor_stride, self.D)
        return self._manager.insert_and_map(coordinates, tensor_stride, string_id)

    def stride(self, coordinate_map_key: CoordinateMapKey,
               stride: Union[int, Sequence, np.ndarray, torch.Tensor],
               string_id: str = "") -> CoordinateMapKey:
        stride = convert_to_int_list(stride, self.D)
        return self._manager.stride(coordinate_map_key, stride, string_id)

    def size(self, coordinate_map_key: CoordinateMapKey) -> int:
        return self._manager.size(coordinate_map_key)

    def _get_coordinate_map_key(self, key_or_tensor_strides) -> CoordinateMapKey:
        assert isinstance(key_or_tensor_strides,
                          (CoordinateMapKey, Sequence, np.ndarray, torch.Tensor, int)), \
            f"The input must be either a CoordinateMapKey or a tensor_stride: {key_or_tensor_strides}"
        if isinstance(key_or_tensor_strides, CoordinateMapKey):
            return key_or_tensor_strides
        tensor_strides = convert_to_int_list(key_or_tensor_strides, self.D)
        keys = self._manager.get_coordinate_map_keys(tensor_strides)
        assert len(keys) > 0
        return keys[0]

    def get_coordinates(self, coords_key_or_tensor_strides) -> torch.Tensor:
        key = self._get_coordinate_map_key(coords_key_or_tensor_strides)
        return self._manager.get_coordinates(key)

    def get_unique_coordinate_map_key(self, tensor_stride: Union[int, list]) -> CoordinateMapKey:
        ts = convert_to_int_list(tensor_stride, self.D)
        k = self._manager.get_random_string_id(ts, "")
        return CoordinateMapKey(list(k[0]), k[1])

    def get_kernel_map(self, in_key, out_key, stride=1, kernel_size=3, dilation=1,
                       region_type=RegionType.HYPER_CUBE, region_offset=None,
                       is_transpose=False, is_pool=False) -> dict:
        warnings.warn("`get_kernel_map` will be deprecated. Please use `kernel_map` instead.")
        return self.kernel_map(in_key, out_key, stride, kernel_size, dilation, region_type,
                               region_offset, is_transpose, is_pool)

    def kernel_map(self, in_key, out_key, stride=1, kernel_size=3, dilation=1,
                   region_type=RegionType.HYPER_CUBE, region_offset=None, is_transpose=False,
                   is_pool=False) -> dict:
        """dict{kernel_index: IntTensor[2, n_k]} — row 0 input rows, row 1 output rows."""
        if isinstance(kernel_size, torch.Tensor):
            assert (kernel_size > 0).all(), f"Invalid kernel size: {kernel_size}"
            if (kernel_size == 1).all():
                region_type = RegionType.HYPER_CUBE
        elif isinstance(kernel_size, int):
            assert kernel_size > 0, f"Invalid kernel size: {kernel_size}"
            if kernel_size == 1:
                region_type = RegionType.HYPER_CUBE
        in_key = self._get_coordinate_map_key(in_key)
        out_key = self._get_coordinate_map_key(out_key)
        if region_offset is None:
            region_offset = torch.IntTensor()
        return self._manager.kernel_map(
            in_key, out_key, convert_to_int_list(kernel_size, self.D),
            convert_to_int_list(stride, self.D), convert_to_int_list(dilation, self.D),
            region_type, region_offset, is_transpose, is_pool)

    def origin(self) -> CoordinateMapKey:
        """Key of the origin map: one row (b, 0, ..., 0) per batch index, ascending
        (reference: MinkowskiCoordinateManager.py:270)."""
        return self._manager.origin()

    def origin_map(self, key: CoordinateMapKey):
        """(batch_indices int64 [B], [row indices of batch index b, b = 0..max batch index])
        (reference: MinkowskiCoordinateManager.py:423)."""
        return self._manager.origin_map(key)

    def origin_map_size(self) -> int:
        """Number of clouds B (rows of the origin map)."""
        return self._manager.origin_map_size()

    def union_map(self, in_keys: list, out_key):
        """Sets `out_key` to the union of the maps `in_keys` (rows of the first map in order, then
        the new rows of each following map in order; cached per ordered tuple of keys) and returns,
        per input, int64 [2, n_i]: (input rows, union rows)
        (reference: MinkowskiCoordinateManager.py:432)."""
        return self._manager.union_map(in_keys, out_key)

    def stride_map(self, in_key: CoordinateMapKey, stride_key: CoordinateMapKey):
        return self._manager.stride_map(in_key, stride_key)

    # -- tensor fields (reference: MinkowskiCoordinateManager.py, coordinate_map_manager.cpp:145-343)
    def insert_field(self, coordinates: torch.Tensor, tensor_stride=1,
                     string_id: str = "") -> CoordinateMapKey:
        """Registers float32 point coordinates [N, D+1] and returns the field key."""
        return self._manager.insert_field(coordinates, convert_to_int_list(tensor_stride, self.D),
                                          string_id)

    def get_coordinate_field(self, field_key: CoordinateMapKey) -> torch.Tensor:
        return self._manager.get_coordinate_field(field_key)

    def field_to_sparse_insert_and_map(self, field_key: CoordinateMapKey, tensor_stride=1,
                                       string_id: str = ""):
        """Quantises the field at `tensor_stride` into a coordinate map -> (map key, (unique_index,
        inverse_mapping)); quantising the same field at the same stride again returns the same
        map.  Raises ValueError for non-finite coordinates."""
        return self._manager.field_to_sparse_insert_and_map(
            field_key, convert_to_int_list(tensor_stride, self.D), string_id)

    def field_to_sparse_map(self, field_key: CoordinateMapKey, sparse_key: CoordinateMapKey):
        """(inverse_mapping int64 [N], unique_index int64 [M]) of the field's points in an existing
        map (-1 where the map lacks a point's voxel / a row has no point)."""
        return self._manager.field_to_sparse_map(field_key, sparse_key)

    def exists_field_to_sparse(self, field_key: CoordinateMapKey, sparse_key: CoordinateMapKey):
        return self._manager.exists_field_to_sparse(field_key, sparse_key)

    def get_field_to_sparse_map(self, field_key: CoordinateMapKey, sparse_key: CoordinateMapKey):
        """(unique_index, inverse_mapping) of a field-to-map relation made before."""
        return self._manager.get_field_to_sparse_map(field_key, sparse_key)

    def field_to_sparse_keys(self, field_key: CoordinateMapKey):
        return self._manager.field_to_sparse_keys(field_key)

    def interpolation_map_weight(self, key: CoordinateMapKey, samples: torch.Tensor):
        """[in rows, out rows, weights] of the multilinear interpolation of the map's rows at the
        float sample points (every present corner, ordered by sample, then corner)."""
        return self._manager.interpolation_map_weight(key, samples)

    def __repr__(self):
        return (self._CoordinateManagerClass.__name__ + "(\n" + str(self._manager)
                + f"\talgorithm={self.minkowski_algorithm}\n  )\n")
