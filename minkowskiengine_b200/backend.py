"""Host-side mirror of the reference's native boundary `MinkowskiEngineBackend._C`
(pybind/extern.hpp:515-838) for the sparse-convolution hot path.

Same names, argument order and side effects as the reference's `...GPU` functions and
`CoordinateMapManagerGPU_c10`, but the bodies are thin: they validate, keep the manager's
bookkeeping (key naming / reuse / kernel-map cache — coordinate_map_manager.cpp:353-466,
662-823) and hand device pointers to the C-ABI library (include/meb200.h).  All device
work happens in libmeb200.so on torch's current CUDA stream; the only host<->device
synchronisation is the unique-row count read when a NEW coordinate map is created.
"""
import ctypes
import os
import random
import string
import weakref

import torch

from . import _lib
from .enums import MinkowskiAlgorithm, PoolingMode, RegionType
from .kernel_generator import region_offsets

ERROR_MAP_NOT_FOUND = "CoordinateMap not found"  # reference: src/errors.hpp:33


def _assert(cond, *msg):
    """Reference ASSERT semantics (src/utils.hpp:141-150): RuntimeError with the message."""
    if not cond:
        raise RuntimeError(" ".join(str(m) for m in msg))


def is_cuda_available():
    return torch.cuda.is_available()


def cuda_version():
    return int(torch.version.cuda.replace(".", "")) * 10 if torch.version.cuda else 0


def cudart_version():
    return int(_lib.load().meb200_cudart_version())


def get_gpu_memory_info():
    return torch.cuda.mem_get_info()


# ----------------------------------------------------------------------------------------
class CoordinateMapKey:
    """(tensor_stride, string_id) handle of a coordinate map
    (reference: src/coordinate_map_key.hpp:44-157, pybind/extern.hpp:744-763)."""

    __slots__ = ("_coordinate_size", "_tensor_stride", "_string_id", "_set", "_tup")

    def __init__(self, *args):
        if len(args) == 1 and isinstance(args[0], int):
            self._coordinate_size = args[0]
            self._tensor_stride, self._string_id, self._set = None, "", False
            self._tup = None
        elif len(args) == 2:
            ts = [int(v) for v in args[0]]
            self._coordinate_size = len(ts) + 1
            self._tensor_stride, self._string_id, self._set = ts, str(args[1]), True
            self._tup = (tuple(ts), self._string_id)     # hashable form, built once
        else:
            raise TypeError("CoordinateMapKey(coordinate_size:int) or "
                            "CoordinateMapKey(tensor_stride:list, string_id:str)")

    def is_key_set(self):
        return self._set

    def get_coordinate_size(self):
        return self._coordinate_size

    def get_dimension(self):
        return self._coordinate_size

    def get_key(self):
        _assert(self._set, "CoordinateMapKey: Key Not Set")
        return (list(self._tensor_stride), self._string_id)

    def set_key(self, *args):
        if len(args) == 1:
            ts, sid = args[0]
        else:
            ts, sid = args
        ts = [int(v) for v in ts]
        _assert(len(ts) + 1 == self._coordinate_size, "Invalid tensor stride size", ts,
                "for coordinate size", self._coordinate_size)
        self._tensor_stride, self._string_id, self._set = ts, str(sid), True
        self._tup = (tuple(ts), self._string_id)

    def get_tensor_stride(self):
        _assert(self._set, "CoordinateMapKey: Key Not Set")
        return list(self._tensor_stride)

    def _tuple(self):
        return self._tup

    def __eq__(self, other):
        if not isinstance(other, CoordinateMapKey):
            return NotImplemented
        if not (self._set and other._set):
            return False
        return self._coordinate_size == other._coordinate_size and self._tuple() == other._tuple()

    def __hash__(self):
        return hash(self._tuple()) if self._set else hash(self._coordinate_size)

    def __repr__(self):
        if not self._set:
            return f"coordinate map key: unset (coordinate size {self._coordinate_size})"
        s = "coordinate map key:" + "[" + ", ".join(str(v) for v in self._tensor_stride) + "]"
        return s + (":" + self._string_id if self._string_id else "")


# ----------------------------------------------------------------------------------------
class _CoordinateMap:
    """Device-resident coordinate map: unique int32 rows + open-addressing row-index table
    (replaces CoordinateMapGPU, src/coordinate_map_gpu.cuh:61-317)."""

    __slots__ = ("coords", "table", "capacity", "tensor_stride")

    def __init__(self, coords, table, capacity, tensor_stride):
        self.coords, self.table, self.capacity = coords, table, capacity
        self.tensor_stride = tuple(tensor_stride)

    @property
    def size(self):
        return self.coords.shape[0]

    @property
    def ncols(self):
        return self.coords.shape[1]

    @staticmethod
    def build(candidates, tensor_stride, valid=None):
        """Deduplicating insert of candidate rows -> (map, unique_index, inverse_map)."""
        lib = _lib.load()
        n, ncols = candidates.shape
        dev = candidates.device
        cap = int(lib.meb200_hash_capacity(n))
        table = torch.empty(cap, dtype=torch.int32, device=dev)
        uniq = torch.empty((n, ncols), dtype=torch.int32, device=dev)
        uidx = torch.empty(n, dtype=torch.int64, device=dev)
        inv = torch.empty(n, dtype=torch.int64, device=dev)
        scratch = torch.empty(int(lib.meb200_insert_scratch_bytes(n)), dtype=torch.uint8,
                              device=dev)
        m = ctypes.c_uint32(0)
        _lib.check(lib.meb200_insert_and_map(
            _lib.ptr(candidates), _lib.ptr(valid), n, ncols, _lib.ptr(table), cap,
            _lib.ptr(uniq), _lib.ptr(uidx), _lib.ptr(inv), _lib.ptr(scratch),
            ctypes.byref(m), _lib.current_stream()))
        m = int(m.value)
        cmap = _CoordinateMap(uniq[:m], table, cap, tensor_stride)
        return cmap, uidx[:m], inv


class _PendingLevel:
    """One level of a stride pyramid whose kernels are enqueued but whose size has not been read
    yet (see CoordinateMapManagerGPU_c10._prefetch_pyramid)."""

    __slots__ = ("parent_key", "tensor_stride", "uniq", "inverse", "count_dev", "count_host",
                 "event")


# kernel strides requested along the stride chain below the first inserted map of the previous
# coordinate manager, per coordinate width: the prediction for the next manager's pyramid
_PYRAMID_HINT = {}
# ... and the kernel maps it was asked for, in order (keys + kernel geometry, no tensors)
_KMAP_HINT = {}
_PAIR_HINT = set()      # kernel-map cache keys whose pair lists (wgrad) were asked for
_PREFETCH = os.environ.get("MEB200_MAP_PREFETCH", "1") not in ("", "0")


class _KernelMap:
    """k-major neighbour tables of one (in map, out map, kernel) triple.

    out_nbr[k, o] = input row reached from output row o through offset k (or -1)
    in_nbr [k, i] = output row that input row i feeds through offset k (or -1)
    Replaces gpu_kernel_map's three flat arrays + host offset table (src/kernel_map.cuh:48-429);
    `swapped()` is the reference's swap_in_out (kernel_map.cuh:191-241)."""

    __slots__ = ("out_nbr", "_in_nbr", "_in_thunk", "_n_in", "stride_pairs", "_n_pairs", "_pairs",
                 "_pair_src", "_hint_key")
    PAIR_STAGE = 64   # pairs per pipeline stage of the wgrad kernel (k_wgrad_wg)
    # table rows per chunk of the pair lists (multiple of 2048): one chunk's rows of both feature
    # matrices stay L2-resident while the wgrad walks its K offsets
    PAIR_CHUNK_ROWS = int(os.environ.get("MEB200_PAIR_CHUNK_ROWS", "262144"))

    def __init__(self, out_nbr, in_nbr, stride_pairs=None, n_in=None, in_thunk=None):
        # in_nbr may be None with (n_in, in_thunk): the reverse table of a large kernel (the
        # K = 125 stem: 400 MB at 800k rows) is only built if somebody asks for it — dgrad or a
        # transposed layer; the stem of a network needs neither
        self.out_nbr, self._in_nbr, self._in_thunk = out_nbr, in_nbr, in_thunk
        self._n_in = in_nbr.shape[1] if in_nbr is not None else int(n_in)
        self.stride_pairs = stride_pairs  # (in_rows, out_rows) when built as a stride map
        self._n_pairs = None
        self._pairs = None      # (pairs_in, pairs_out, seg_start) once built
        self._pair_src = None   # the map this one is the swapped view of
        self._hint_key = None   # the manager's cache key (prediction of the next manager's needs)

    def pair_lists(self):
        """(pairs_in, pairs_out, seg_start, n_chunks): compacted (input row, output row) lists in
        (row chunk, offset) order, every segment padded to PAIR_STAGE entries
        (meb200_kernel_map_pairs) — the reference's own kernel-map representation, chunked so
        that a consumer keeps one chunk's feature rows L2-resident across the offsets.  Built on
        first use; a swapped view shares its source's lists with the two sides exchanged."""
        if self._pairs is None:
            if self._hint_key is not None:
                _PAIR_HINT.add(self._hint_key)
            if self._pair_src is not None:
                pin, pout, seg, nch = self._pair_src.pair_lists()
                self._pairs = (pout, pin, seg, nch)
                return self._pairs
            lib = _lib.load()
            K, n = self.out_nbr.shape
            dev = self.out_nbr.device
            chunk_rows = self.PAIR_CHUNK_ROWS
            while K * int(lib.meb200_pair_list_chunks(n, chunk_rows)) > 2047:
                chunk_rows *= 2
            nch = int(lib.meb200_pair_list_chunks(n, chunk_rows))
            cap = int(lib.meb200_pair_list_capacity(K, n, self.PAIR_STAGE, chunk_rows))
            pairs = torch.empty((2, cap), dtype=torch.int32, device=dev)
            seg = torch.empty(nch * K + 1, dtype=torch.int32, device=dev)
            scratch = torch.empty(int(lib.meb200_pair_list_scratch_bytes(K, n, chunk_rows)),
                                  dtype=torch.uint8, device=dev)
            _lib.check(lib.meb200_kernel_map_pairs(
                _lib.ptr(self.out_nbr), K, n, self.PAIR_STAGE, chunk_rows, _lib.ptr(pairs[0]),
                _lib.ptr(pairs[1]), _lib.ptr(seg), _lib.ptr(scratch), _lib.current_stream()))
            self._pairs = (pairs[0], pairs[1], seg, nch)   # other side = input rows, row = output rows
        return self._pairs

    @property
    def n_pairs(self):
        """Number of (in, out) pairs; costs one reduction + host read, cached (profiling only)."""
        if self._n_pairs is None:
            self._n_pairs = int((self.out_nbr >= 0).sum().item())
        return self._n_pairs

    @property
    def K(self):
        return self.out_nbr.shape[0]

    @property
    def n_out(self):
        return self.out_nbr.shape[1]

    @property
    def n_in(self):
        return self._n_in

    @property
    def in_nbr(self):
        if self._in_nbr is None:
            self._in_nbr = self._in_thunk()
            self._in_thunk = None
        return self._in_nbr

    def swapped(self):
        sp = None if self.stride_pairs is None else (self.stride_pairs[1], self.stride_pairs[0])
        km = _KernelMap(self.in_nbr, self.out_nbr, sp)
        km._n_pairs = self._n_pairs
        km._pair_src = self
        return km

    def to_dict(self):
        """{k: IntTensor[2, n_k]} as kernel_map_th returns (coordinate_map_manager.cpp:1395-1414);
        pairs within an offset are ordered by output row (the reference order is unspecified)."""
        if self.stride_pairs is not None:
            i, o = self.stride_pairs
            return {0: torch.stack([i.int(), o.int()])} if i.numel() else {}
        out = {}
        hit = self.out_nbr >= 0
        counts = hit.sum(dim=1).tolist()
        for k, c in enumerate(counts):
            if c > 0:
                o = torch.nonzero(hit[k]).flatten()
                out[k] = torch.stack([self.out_nbr[k, o], o.int()])
        return out


_OFFSET_CACHE = {}


def _device_offsets(region_type, kernel_size, dilation, tensor_stride, custom, device):
    """[K, D] int32 offset table on `device` (cached: a network reuses a handful)."""
    ckey = (region_type, tuple(kernel_size), tuple(dilation), tuple(tensor_stride),
            None if custom is None or custom.numel() == 0 else tuple(map(tuple, custom.tolist())),
            str(device))
    t = _OFFSET_CACHE.get(ckey)
    if t is None:
        offs = region_offsets(region_type, list(kernel_size), list(dilation),
                              list(tensor_stride), custom)
        t = torch.tensor(offs, dtype=torch.int32).reshape(len(offs), len(kernel_size)).to(device)
        _OFFSET_CACHE[ckey] = t
    return t


class CoordinateMapManagerGPU_c10:
    """Owner of coordinate maps and kernel maps on one device
    (reference: CoordinateMapManager, src/coordinate_map_manager.hpp:130-565)."""

    def __init__(self, algorithm=MinkowskiAlgorithm.DEFAULT, num_threads=-1):
        self.algorithm = algorithm
        self.num_threads = num_threads  # accepted for signature parity; unused on GPU
        self._maps = {}         # (tuple tensor_stride, str id) -> _CoordinateMap
        self._kernel_maps = {}  # 8-tuple (types.hpp:183-192) -> _KernelMap
        self._parents = {}      # out key -> (in key, int64 row of every in row in out map)
        self._pending = {}      # out key -> _PendingLevel (enqueued, size not yet read)
        self._chain_tip = None  # last map of the stride chain below the first inserted map
        self._chain = []        # kernel strides requested along that chain
        self._km_seen = set()   # kernel-map cache keys the caller has asked for
        self._km_requests = []  # ... in order: the prediction for the next manager
        self._replaying = False
        self._hint_ncols = None
        _lib.load()             # fail at construction if the native library is missing

    # -- keys ------------------------------------------------------------------------
    @staticmethod
    def _k(key):
        if isinstance(key, CoordinateMapKey):
            _assert(key._set, "CoordinateMapKey: Key Not Set")
            return key._tup
        return (tuple(key[0]), key[1])

    def exists(self, key):
        return self._k(key) in self._maps

    def _get(self, key, what=""):
        k = self._k(key)
        _assert(k in self._maps, what, ERROR_MAP_NOT_FOUND)
        return self._maps[k]

    def get_random_string_id(self, tensor_stride, string_id=""):
        ts = tuple(int(v) for v in tensor_stride)
        while True:
            r = "".join(random.choices(string.ascii_letters + string.digits, k=5))
            key = (ts, (string_id + "-" + r) if string_id else r)
            if key not in self._maps:
                return key

    def get_coordinate_map_keys(self, tensor_stride):
        ts = tuple(int(v) for v in tensor_stride)
        return [CoordinateMapKey(list(k[0]), k[1]) for k in self._maps if k[0] == ts]

    def size(self, key):
        return self._get(key).size

    def get_coordinates(self, key):
        return self._get(key).coords

    # -- map creation ----------------------------------------------------------------
    def insert_and_map(self, coordinates, tensor_stride, string_id=""):
        """reference: coordinate_map_manager.cpp:353-399"""
        _assert(coordinates.dim() == 2, "coordinates must be 2-dimensional")
        _assert(coordinates.dtype == torch.int32, "coordinates must be an IntTensor")
        _assert(coordinates.is_contiguous(), "coordinates must be contiguous")
        _assert(coordinates.is_cuda,
                "coordinates must be a CUDA tensor: minkowskiengine_b200 implements the GPU "
                "coordinate manager only (no CPU backend, no fallback)")
        ts = [int(v) for v in tensor_stride]
        _assert(coordinates.size(1) - 1 == len(ts),
                "The coordinate dimension (coordinate_size - 1):", coordinates.size(1) - 1,
                " must match the size of tensor stride:", ts)
        key = (tuple(ts), string_id)
        if key in self._maps:
            key = self.get_random_string_id(ts, string_id)
        cmap, unique_index, inverse_map = _CoordinateMap.build(coordinates, ts)
        first = not self._maps
        self._maps[key] = cmap
        if first:
            self._chain_tip = key
            self._hint_ncols = cmap.ncols
            self._prefetch_pyramid(key, cmap)
            self._prefetch_kernel_maps(cmap.ncols)
        if cmap.size == coordinates.size(0):
            # no duplicates: the reference GPU path returns an empty inverse map here
            # (coordinate_map_manager.cu:94-112) and Python substitutes arange
            inverse_map = inverse_map[:0]
        return CoordinateMapKey(list(key[0]), key[1]), (unique_index, inverse_map)

    def _stride(self, in_key, kernel_stride, string_id=""):
        """reference: coordinate_map_manager.cpp:406-429 -> (out key tuple, created?)"""
        in_key = self._k(in_key)
        _assert(in_key in self._maps, ERROR_MAP_NOT_FOUND)
        _assert(len(kernel_stride) == len(in_key[0]), "stride size mismatch.")
        out_ts = tuple(t * int(s) for t, s in zip(in_key[0], kernel_stride))
        out_key = (out_ts, string_id if string_id else in_key[1])
        if in_key == self._chain_tip and out_key != in_key and not self._replaying:
            # remember the pyramid for the next manager
            self._chain_tip = out_key
            self._chain.append(tuple(int(s) for s in kernel_stride))
            _PYRAMID_HINT[len(in_key[0]) + 1] = tuple(self._chain)
        if out_key in self._maps:
            return out_key, False
        if self._take_pending(in_key, out_key):
            return out_key, True
        in_map = self._maps[in_key]
        lib = _lib.load()
        cand = torch.empty_like(in_map.coords)
        ts_arr = (ctypes.c_int32 * len(out_ts))(*out_ts)
        _lib.check(lib.meb200_stride_coords(_lib.ptr(in_map.coords), in_map.size, in_map.ncols,
                                            ts_arr, _lib.ptr(cand), _lib.current_stream()))
        out_map, _, inverse = _CoordinateMap.build(cand, out_ts)
        self._maps[out_key] = out_map
        self._parents[out_key] = (in_key, inverse)
        return out_key, True

    # A strided map is a function of the input coordinates alone, but creating it where the
    # network first asks for it costs a blocking read of its size with the whole forward pass
    # queued in front (the host's lead over the GPU is lost at every down-sampling layer, and the
    # coarse levels — 10-30 us kernels — then run launch bound).  So the pyramid the PREVIOUS
    # manager was asked for (_PYRAMID_HINT) is enqueued right behind the input map, on upper-bound
    # buffers with device-side row counts (meb200_insert_and_map_enqueue); its sizes reach the
    # host long before the layers that need them.  A wrong prediction is only wasted work: a
    # level that is never requested, or requested with another stride, is dropped.
    def _prefetch_pyramid(self, key, cmap):
        hint = _PYRAMID_HINT.get(cmap.ncols) if _PREFETCH else None
        if not hint or cmap.size == 0:
            return
        lib = _lib.load()
        dev = cmap.coords.device
        n, ncols = cmap.size, cmap.ncols
        stream = _lib.current_stream()
        cap = int(lib.meb200_hash_capacity(n))
        scratch_bytes = int(lib.meb200_insert_scratch_bytes(n))
        parent_key, parent_coords, parent_count = key, cmap.coords, None
        for ks in hint:
            if len(ks) != len(parent_key[0]):
                return
            out_ts = tuple(t * s for t, s in zip(parent_key[0], ks))
            out_key = (out_ts, parent_key[1])
            if out_key in self._maps or out_key in self._pending:
                return
            lv = _PendingLevel()
            lv.parent_key, lv.tensor_stride = parent_key, out_ts
            cand = torch.empty((n, ncols), dtype=torch.int32, device=dev)
            ts_arr = (ctypes.c_int32 * len(out_ts))(*out_ts)
            # rows past the parent's (device-side) count are whatever the buffer holds: they are
            # strided like the others and then ignored by the insert
            _lib.check(lib.meb200_stride_coords(_lib.ptr(parent_coords), n, ncols, ts_arr,
                                                _lib.ptr(cand), stream))
            table = torch.empty(cap, dtype=torch.int32, device=dev)
            lv.uniq = torch.empty((n, ncols), dtype=torch.int32, device=dev)
            uidx = torch.empty(n, dtype=torch.int64, device=dev)
            lv.inverse = torch.empty(n, dtype=torch.int64, device=dev)
            scratch = torch.empty(scratch_bytes, dtype=torch.uint8, device=dev)
            lv.count_dev = torch.empty(1, dtype=torch.int32, device=dev)
            _lib.check(lib.meb200_insert_and_map_enqueue(
                _lib.ptr(cand), None, _lib.ptr(parent_count), n, ncols, _lib.ptr(table), cap,
                _lib.ptr(lv.uniq), _lib.ptr(uidx), _lib.ptr(lv.inverse), _lib.ptr(scratch),
                _lib.ptr(lv.count_dev), stream))
            lv.count_host = torch.empty(1, dtype=torch.int32, pin_memory=True)
            lv.count_host.copy_(lv.count_dev, non_blocking=True)
            lv.event = torch.cuda.Event()
            lv.event.record()
            self._pending[out_key] = lv
            parent_key, parent_coords, parent_count = out_key, lv.uniq, lv.count_dev

    # The kernel maps are functions of the coordinate maps alone as well: the ones the previous
    # manager was asked for (_KMAP_HINT) are built right here, before the first layer runs.  The
    # GPU gets ~1.5 ms of table probing to chew on while the host enqueues the layers, instead of
    # meeting each map where the forward pass first needs it with nothing else queued (the coarse
    # levels of a U-Net are launch bound: 10-30 us kernels against ~50 us of host work per layer).
    def _materialize(self, key):
        if key in self._maps:
            return True
        lv = self._pending.get(key)
        return (lv is not None and self._materialize(lv.parent_key)
                and self._take_pending(lv.parent_key, key))

    def _prefetch_kernel_maps(self, ncols):
        hint = _KMAP_HINT.get(ncols) if _PREFETCH else None
        if not hint:
            return
        self._replaying = True
        try:
            for ik, ok, ksize, kstride, kdil, region, is_transpose, is_pool in hint:
                if self._materialize(ik) and self._materialize(ok):
                    km = self._kernel_map(ik, ok, ksize, kstride, kdil, region, None,
                                          is_transpose, is_pool)
                    if (ik, ok, ksize, kstride, kdil, region, is_transpose, is_pool) in _PAIR_HINT:
                        km.pair_lists()          # the backward pass will want them
        finally:
            self._replaying = False

    def _take_pending(self, in_key, out_key):
        """Turns the enqueued level `out_key` into a map if it was built from `in_key`."""
        lv = self._pending.pop(out_key, None)
        if lv is None or lv.parent_key != in_key:
            return False
        lib = _lib.load()
        lv.event.synchronize()          # normally long past: enqueued before the first layer
        m = int(lv.count_host.item())
        cap = int(lib.meb200_hash_capacity(m))
        table = torch.empty(cap, dtype=torch.int32, device=lv.uniq.device)
        coords = lv.uniq[:m]
        _lib.check(lib.meb200_map_build_table(_lib.ptr(coords), m, coords.shape[1],
                                              _lib.ptr(table), cap, _lib.current_stream()))
        self._maps[out_key] = _CoordinateMap(coords, table, cap, lv.tensor_stride)
        self._parents[out_key] = (in_key, lv.inverse[:self._maps[in_key].size])
        return True

    def stride(self, key, stride, string_id=""):
        out_key, _ = self._stride(key, [int(s) for s in stride], string_id)
        return CoordinateMapKey(list(out_key[0]), out_key[1])

    def _stride_region(self, in_key, region_type, kernel_size, dilation, custom_offsets,
                       region_tensor_stride, out_tensor_stride, is_transpose,
                       expand_coordinates):
        """reference: coordinate_map_manager.cpp:435-466 + coordinate_map_cpu.hpp:446-487"""
        in_key = self._k(in_key)
        _assert(in_key in self._maps, ERROR_MAP_NOT_FOUND)
        out_ts = tuple(int(v) for v in out_tensor_stride)
        out_key = (out_ts, "")
        exists = out_key in self._maps
        if exists and not expand_coordinates:
            return out_key, False
        in_map = self._maps[in_key]
        lib = _lib.load()
        offs = _device_offsets(region_type, kernel_size, dilation, region_tensor_stride,
                               custom_offsets, in_map.coords.device)
        K = offs.shape[0]
        n = in_map.size
        cand = torch.empty((n * K, in_map.ncols), dtype=torch.int32, device=in_map.coords.device)
        valid = torch.empty(n * K, dtype=torch.uint8, device=in_map.coords.device)
        ts_arr = (ctypes.c_int32 * len(out_ts))(*out_ts)
        _lib.check(lib.meb200_region_coords(
            _lib.ptr(in_map.coords), n, in_map.ncols, _lib.ptr(offs), K, ts_arr,
            0 if is_transpose else 1, _lib.ptr(cand), _lib.ptr(valid), _lib.current_stream()))
        out_map, _, _ = _CoordinateMap.build(cand, out_ts, valid)
        out_map.coords = out_map.coords.clone()  # drop the n*K candidate buffer
        if exists:
            out_key = self.get_random_string_id(out_ts, "")
        self._maps[out_key] = out_map
        return out_key, True

    # -- kernel maps -----------------------------------------------------------------
    LAZY_REVERSE_K = 64      # kernels this large get their reverse table on demand

    @staticmethod
    def _probe(x_map, y_map, offsets, need_y=True):
        """x-stationary probe: returns (x_nbr [K,nx], y_nbr [K,ny] or None).  (Static: the deferred
        reverse-table build below must not keep the manager alive through a reference cycle —
        a manager owns ~1.5 GB of tables on the bench clouds and should die with its tensors.)"""
        lib = _lib.load()
        K = offsets.shape[0]
        dev = x_map.coords.device
        x_nbr = torch.empty((K, x_map.size), dtype=torch.int32, device=dev)
        y_nbr = torch.full((K, y_map.size), -1, dtype=torch.int32, device=dev) if need_y else None

        def launch():
            _lib.check(lib.meb200_kernel_map(
                _lib.ptr(x_map.coords), x_map.size, _lib.ptr(y_map.coords), y_map.size,
                _lib.ptr(y_map.table), y_map.capacity, x_map.ncols, _lib.ptr(offsets), K,
                _lib.ptr(x_nbr), _lib.ptr(y_nbr), None, _lib.current_stream()))
        if _PROFILE is not None:
            # algorithmic bytes (SURVEY.md 8d): coordinate rows read once, one 4-byte table slot
            # + one coordinate row compared per probe, both neighbour tables written
            nc4 = x_map.ncols * 4
            probes = float(K) * x_map.size
            nbytes = x_map.size * nc4 + probes * (4 + nc4) + probes * 4 + \
                (float(K) * y_map.size * 4 if need_y else 0.0)
            _record("kernel_map", launch, probes, nbytes, always=True)
        else:
            launch()
        return x_nbr, y_nbr

    def _kernel_map(self, in_key, out_key, kernel_size, kernel_stride, kernel_dilation,
                    region_type, offset, is_transpose, is_pool):
        """reference: coordinate_map_manager.cpp:662-823 (cache key = types.hpp:183-192)"""
        ik, ok = self._k(in_key), self._k(out_key)
        ksize = tuple(int(v) for v in kernel_size)
        kstride = tuple(int(v) for v in kernel_stride)
        kdil = tuple(int(v) for v in kernel_dilation)
        _assert(len(ksize) == len(kstride) == len(kdil), "kernel size mismatch")
        cache_key = (ik, ok, ksize, kstride, kdil, region_type, bool(is_transpose), bool(is_pool))
        if not self._replaying and cache_key not in self._km_seen:
            self._km_seen.add(cache_key)
            if region_type != RegionType.CUSTOM and self._hint_ncols is not None:
                self._km_requests.append(cache_key)
                _KMAP_HINT[self._hint_ncols] = tuple(self._km_requests)
        km = self._kernel_maps.get(cache_key)
        if km is not None:
            return km
        _assert(ik in self._maps, "in_map", ERROR_MAP_NOT_FOUND)
        _assert(ok in self._maps, "out_map", ERROR_MAP_NOT_FOUND)
        in_map, out_map = self._maps[ik], self._maps[ok]
        _assert(len(ksize) + 1 == in_map.ncols, "kernel size mismatch")
        custom = offset if region_type == RegionType.CUSTOM else None
        dev = in_map.coords.device
        stride_map = is_pool and kstride == ksize
        if not is_transpose:
            if stride_map:
                # every input row -> its strided parent (coordinate_map_cpu.hpp:672-722);
                # the floor cell [u, u + k*ts_in) is probed with non-centred offsets
                offs = self._cell_offsets(ksize, in_map.tensor_stride, dev)
                out_nbr, in_nbr = self._probe(out_map, in_map, offs)
                km = _KernelMap(out_nbr, in_nbr, self._stride_pairs(ik, ok, in_map, out_map))
            else:
                offs = _device_offsets(region_type, ksize, kdil, in_map.tensor_stride, custom, dev)
                if offs.shape[0] >= self.LAZY_REVERSE_K:
                    out_nbr, _ = self._probe(out_map, in_map, offs, need_y=False)
                    probe = self._probe
                    km = _KernelMap(out_nbr, None, n_in=in_map.size,
                                    in_thunk=lambda: probe(out_map, in_map, offs)[1])
                else:
                    out_nbr, in_nbr = self._probe(out_map, in_map, offs)
                    km = _KernelMap(out_nbr, in_nbr)
        else:
            swapped_key = (ok, ik, ksize, kstride, kdil, region_type, False, bool(is_pool))
            fwd = self._kernel_maps.get(swapped_key)
            if fwd is None:
                # iterate the coarse input rows, probe the fine output map with offsets in
                # output-stride units (coordinate_map_manager.cpp:789-811), i.e. the forward
                # map of (out -> in); cached under the forward key as well
                if stride_map:
                    offs = self._cell_offsets(ksize, out_map.tensor_stride, dev)
                    a, b = self._probe(in_map, out_map, offs)
                    fwd = _KernelMap(a, b, self._stride_pairs(ok, ik, out_map, in_map))
                else:
                    offs = _device_offsets(region_type, ksize, kdil, out_map.tensor_stride,
                                           custom, dev)
                    a, b = self._probe(in_map, out_map, offs)
                    fwd = _KernelMap(a, b)
                fwd._hint_key = swapped_key
                self._kernel_maps[swapped_key] = fwd
            km = fwd.swapped()
        km._hint_key = cache_key
        self._kernel_maps[cache_key] = km
        return km

    @staticmethod
    def _cell_offsets(ksize, tensor_stride, dev):
        # offsets i * ts, i in [0, k): the members of one stride cell
        return _device_offsets(RegionType.CUSTOM, ksize, [1] * len(ksize), tensor_stride,
                               _cell_table(ksize), dev)

    def _stride_pairs(self, in_key, out_key, in_map, out_map):
        """(in_rows, out_rows) of the stride map as the API reports it."""
        par = self._parents.get(out_key)
        if par is not None and par[0] == in_key:
            inv = par[1]
        else:
            lib = _lib.load()
            cand = torch.empty_like(in_map.coords)
            ts = out_map.tensor_stride
            ts_arr = (ctypes.c_int32 * len(ts))(*ts)
            _lib.check(lib.meb200_stride_coords(_lib.ptr(in_map.coords), in_map.size,
                                                in_map.ncols, ts_arr, _lib.ptr(cand),
                                                _lib.current_stream()))
            res = torch.empty(in_map.size, dtype=torch.int32, device=cand.device)
            _lib.check(lib.meb200_map_find(_lib.ptr(out_map.coords), _lib.ptr(out_map.table),
                                           out_map.capacity, out_map.ncols, _lib.ptr(cand),
                                           in_map.size, _lib.ptr(res), _lib.current_stream()))
            inv = res.long()
        rows = torch.arange(in_map.size, dtype=torch.int64, device=inv.device)
        keep = inv >= 0
        return rows[keep], inv[keep]

    def kernel_map(self, in_key, out_key, kernel_size, kernel_stride, kernel_dilation,
                   region_type, offset, is_transpose, is_pool):
        """Python-facing dict form (kernel_map_th, coordinate_map_manager.cpp:1395-1414)."""
        return self._kernel_map(in_key, out_key, kernel_size, kernel_stride, kernel_dilation,
                                region_type, offset, is_transpose, is_pool).to_dict()

    def stride_map(self, in_key, out_key):
        ik, ok = self._k(in_key), self._k(out_key)
        in_map, out_map = self._get(ik), self._get(ok)
        return self._stride_pairs(ik, ok, in_map, out_map)

    def __repr__(self):
        lines = [f"\t{list(k[0])}{':' + k[1] if k[1] else ''}:\tCoordinateMapGPU:{m.size}x{m.ncols}"
                 for k, m in self._maps.items()]
        return "\n".join(lines + [f"\tkernel maps: {len(self._kernel_maps)}"]) + "\n"


def _cell_table(ksize):
    import itertools
    rows = []
    for idx in itertools.product(*[range(k) for k in reversed(ksize)]):
        rows.append(list(reversed(idx)))  # axis 0 fastest, like HYPER_CUBE
    return torch.tensor(rows, dtype=torch.int32)


CoordinateMapManagerGPU_default = CoordinateMapManagerGPU_c10


# ----------------------------------------------------------------------------------------
def _check_feats(in_feat, manager, in_key, name="in_feat"):
    _assert(in_feat.is_cuda, f"{name} must be CUDA (this backend has no CPU path)")
    _assert(in_feat.is_contiguous(), f"{name} must be contiguous")
    _assert(in_feat.dim() == 2, f"{name}.dim():", in_feat.dim())
    _assert(manager.exists(in_key), ERROR_MAP_NOT_FOUND)
    _assert(in_feat.size(0) == manager.size(in_key), "Invalid in_feat size", in_feat.size(0),
            "!=", manager.size(in_key))


def _workspace(n_in, n_out, c_in, c_out, K, code, device):
    nbytes = int(_lib.load().meb200_conv_workspace_bytes(n_in, n_out, c_in, c_out, K, code))
    if nbytes == 0:
        return None, 0
    return torch.empty(nbytes, dtype=torch.uint8, device=device), nbytes


def _wgrad_workspace(c_in, c_out, K, n_out, device):
    """Room for the row-split partial sums of a wgrad (added in a fixed order: deterministic)."""
    nbytes = int(_lib.load().meb200_conv_wgrad_workspace_bytes(c_in, c_out, K, n_out))
    if nbytes == 0:
        return None, 0
    return torch.empty(nbytes, dtype=torch.uint8, device=device), nbytes


# ---- live per-kernel timing for bench.py's roofline (CUDA events on the launch stream) ------
_PROFILE = None   # None, or {"conv_fwd_dgrad": [...], "conv_wgrad": [...], "kernel_map": [...]}


def _record(kind, fn, flops, nbytes, always=False):
    """Run fn() between two CUDA events on the current stream; keep the record if it launched
    a tensor-core kernel (the family the roofline is reported for) or `always`."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    tc0 = _lib.tc_launch_count()
    e0.record()
    out = fn()
    e1.record()
    if always or _lib.tc_launch_count() > tc0:
        _PROFILE[kind].append((e0, e1, flops, nbytes))
    return out


def profile_conv_kernels(step_fn, steps=2):
    """Runs `steps` extra steps with every convolution launch bracketed by CUDA events and
    returns, per kernel family, the summed device time and ALGORITHMIC work:
    flops = 2*P*Cin*Cout per launch, bytes = the compulsory traffic of SURVEY.md §8d."""
    global _PROFILE
    _PROFILE = {"conv_fwd_dgrad": [], "conv_wgrad": [], "kernel_map": []}
    try:
        for _ in range(steps):
            step_fn()
        torch.cuda.synchronize()
        res = {}
        for kind, recs in _PROFILE.items():
            res[kind] = {"ms": sum(a.elapsed_time(b) for a, b, _, _ in recs),
                         "flops": float(sum(r[2] for r in recs)),
                         "bytes": float(sum(r[3] for r in recs)),
                         "launches": len(recs), "steps": steps}
        return res
    finally:
        _PROFILE = None


def _conv_forward(in_feat, kernel, km, out_dtype=None):
    if _PROFILE is not None:
        esz = in_feat.element_size()
        K, c_in, c_out = kernel.shape
        P = km.n_pairs
        nbytes = km.n_in * c_in * esz + km.n_out * c_out * esz + K * c_in * c_out * esz + P * 8
        return _record("conv_fwd_dgrad", lambda: _conv_forward_impl(in_feat, kernel, km, out_dtype),
                       2.0 * P * c_in * c_out, nbytes)
    return _conv_forward_impl(in_feat, kernel, km, out_dtype)


# ---- packed weights: one cast + transpose per optimizer step, not per call -------------------
_PACKED = {}   # id(kernel tensor) -> (weakref, version, data_ptr, dtype, w_cast, w_t)
_ERR_UNSUPPORTED = -3


_PACK_BATCHED = os.environ.get("MEB200_PACK_BATCHED", "1") not in ("", "0")


class _PackJob(ctypes.Structure):      # == meb200_pack_job (include/meb200.h)
    _fields_ = [("w", ctypes.c_void_p), ("w_cast", ctypes.c_void_p), ("w_t", ctypes.c_void_p),
                ("w_cp", ctypes.c_void_p), ("w_tp", ctypes.c_void_p), ("K", ctypes.c_uint32),
                ("c_in", ctypes.c_uint32), ("c_out", ctypes.c_uint32),
                ("tile_begin", ctypes.c_uint32)]


class _PackTable:
    """Every fp32 convolution kernel of one (device, operand dtype) seen so far, with its packed
    buffers and a DEVICE job table: when the optimizer has stepped, the first layer that notices
    re-packs ALL of them with one launch (meb200_conv_pack_weights_batched) instead of every
    layer paying an allocation, a ctypes call and a launch on the forward pass (55 of them per
    MinkUNet34C step, ~1.2 ms of host time where the step is launch bound)."""

    def __init__(self, device, dtype):
        self.device, self.dtype = device, dtype
        self.entries = {}        # id(kernel) -> [weakref, data_ptr, (w_cast, w_t)]
        self.jobs_dev = None
        self.n_jobs = self.total_tiles = 0
        self.order = []          # ids in job order

    def add(self, kernel, packed):
        self.entries[id(kernel)] = [weakref.ref(kernel), kernel.data_ptr(), packed]
        self.jobs_dev = None     # table is stale

    def _rebuild(self):
        jobs, self.order, tile = [], [], 0
        for key, (ref, ptr, packed) in list(self.entries.items()):
            k = ref()
            if k is None or k.data_ptr() != ptr:      # gone or re-allocated: drop (re-added on use)
                del self.entries[key]
                continue
            K, c_in, c_out = k.shape
            w_cast, w_t = packed
            jobs.append(_PackJob(ptr, _lib.ptr(w_cast), _lib.ptr(w_t), None, None, K, c_in, c_out,
                                 tile))
            tile += K * ((c_in + 31) // 32) * ((c_out + 31) // 32)
            self.order.append(key)
        self.n_jobs, self.total_tiles = len(jobs), tile
        if jobs:
            raw = bytes((_PackJob * len(jobs))(*jobs))
            self.jobs_dev = torch.frombuffer(bytearray(raw), dtype=torch.uint8).to(self.device)
        else:
            self.jobs_dev = torch.empty(0, dtype=torch.uint8, device=self.device)

    def repack_all(self):
        """One launch over every registered kernel; refreshes their cache entries."""
        stale = self.jobs_dev is None
        if not stale:
            for key in self.order:             # a tensor died or moved since the table was built?
                ent = self.entries.get(key)
                k = ent[0]() if ent is not None else None
                if k is None or k.data_ptr() != ent[1]:
                    stale = True
                    break
        if stale:
            self._rebuild()
        lib = _lib.load()
        _lib.check(lib.meb200_conv_pack_weights_batched(
            _lib.ptr(self.jobs_dev), self.n_jobs, self.total_tiles, _lib.dtype_code(self.dtype),
            _lib.current_stream()))
        for key in self.order:
            ref, ptr, packed = self.entries[key]
            k = ref()
            _PACKED[key] = (ref, k._version, ptr, self.dtype, packed)


_PACK_TABLES = {}      # (device index, dtype) -> _PackTable


def _packed_weights(kernel, dtype):
    """(w_cast [K,Cin,Cout], w_t [K,Cout,Cin]) of an fp32 master weight in `dtype` (the operand-B
    layouts of dgrad and forward; the permuted copies the packing ABI can also emit are not read
    by any kernel and are not built), rebuilt only when the tensor was modified in place (its autograd version counter moved) or
    replaced."""
    key = id(kernel)
    ent = _PACKED.get(key)
    if ent is not None and ent[0]() is kernel and ent[1] == kernel._version \
            and ent[2] == kernel.data_ptr() and ent[3] == dtype:
        return ent[4]
    tbl = None
    if _PACK_BATCHED:
        tkey = (kernel.device.index, dtype)
        tbl = _PACK_TABLES.get(tkey)
        if tbl is None:
            tbl = _PACK_TABLES[tkey] = _PackTable(kernel.device, dtype)
        reg = tbl.entries.get(key)
        if reg is not None and reg[0]() is kernel and reg[1] == kernel.data_ptr():
            tbl.repack_all()               # a known kernel went stale: the optimizer stepped
            return _PACKED[key][4]
    lib = _lib.load()
    K, c_in, c_out = kernel.shape
    src = kernel.detach()
    buf = torch.empty((2, K * c_in * c_out), dtype=dtype, device=kernel.device)
    w_cast, w_t = buf[0].view(K, c_in, c_out), buf[1].view(K, c_out, c_in)
    _lib.check(lib.meb200_conv_pack_weights(
        _lib.ptr(src), K, c_in, c_out, _lib.dtype_code(dtype), _lib.ptr(w_cast), _lib.ptr(w_t),
        None, None, _lib.current_stream()))
    if len(_PACKED) > 4096:      # dead entries of discarded networks
        for k in [k for k, e in _PACKED.items() if e[0]() is None]:
            del _PACKED[k]
    packed = (w_cast, w_t)
    _PACKED[key] = (weakref.ref(kernel), kernel._version, kernel.data_ptr(), dtype, packed)
    if tbl is not None:
        tbl.add(kernel, packed)            # first sight of this kernel: packed alone, batched next time
    return packed


_STEM = os.environ.get("MEB200_STEM_TC", "1") not in ("", "0")


def _is_stem(kernel, feat_dtype):
    """Layers with <= 4 input channels (the stem of a network) on the bf16/fp16 path: run over
    virtual channels (offset, channel) by the stem kernels (include/meb200.h)."""
    if not (_STEM and kernel.dim() == 3 and kernel.shape[1] <= 4 and _can_pack(kernel, feat_dtype)):
        return False
    return bool(_lib.load().meb200_conv_stem_supported(_lib.dtype_code(feat_dtype), kernel.shape[0],
                                                       kernel.shape[2]))


def _stem_weights(kernel, dtype):
    """Packed weights of the stem's virtual K = 1 layer, [c_out, V] (cached like _packed_weights)."""
    key = (id(kernel), "stem")
    ent = _PACKED.get(key)
    if ent is not None and ent[0]() is kernel and ent[1] == kernel._version \
            and ent[2] == kernel.data_ptr() and ent[3] == dtype:
        return ent[4]
    lib = _lib.load()
    K, c_in, c_out = kernel.shape
    V = int(lib.meb200_conv_stem_virtual_channels(K))
    wv = torch.zeros((V // 4, 4, c_out), dtype=torch.float32, device=kernel.device)
    wv[:K, :c_in] = kernel.detach()
    buf = torch.empty((2, V * c_out), dtype=dtype, device=kernel.device)
    _lib.check(lib.meb200_conv_pack_weights(
        _lib.ptr(wv), 1, V, c_out, _lib.dtype_code(dtype), _lib.ptr(buf[0]), _lib.ptr(buf[1]),
        None, None, _lib.current_stream()))
    w_v = buf[1].view(c_out, V)
    _PACKED[key] = (weakref.ref(kernel), kernel._version, kernel.data_ptr(), dtype, w_v)
    return w_v


def _pad4(feat):
    c = feat.shape[1]
    return feat.contiguous() if c == 4 else torch.nn.functional.pad(feat, (0, 4 - c))


def _can_pack(kernel, feat_dtype):
    return (kernel.dtype == torch.float32 and feat_dtype in (torch.bfloat16, torch.float16)
            and kernel.is_contiguous() and kernel.dim() == 3)


def _conv_forward_impl(in_feat, kernel, km, out_dtype=None):
    lib = _lib.load()
    code = _lib.dtype_code(in_feat.dtype)
    if _is_stem(kernel, in_feat.dtype):
        K, c_in, c_out = kernel.shape
        _assert(K == km.K, "kernel volume", K, "does not match the kernel map", km.K)
        out = torch.empty((km.n_out, c_out), dtype=out_dtype or in_feat.dtype,
                          device=in_feat.device)
        # (named, so that they outlive the argument list: a temporary freed before the call can
        # be handed by the allocator to the next temporary and overwritten before the kernel runs)
        in4, w_v = _pad4(in_feat), _stem_weights(kernel, in_feat.dtype)
        rc = lib.meb200_conv_stem_forward(
            _lib.ptr(in4), code, K, _lib.ptr(w_v), c_out, _lib.ptr(km.out_nbr), km.n_out,
            _lib.ptr(out), _lib.dtype_code(out.dtype), _lib.current_stream())
        if rc != _ERR_UNSUPPORTED:
            _lib.check(rc)
            return out
    if _can_pack(kernel, in_feat.dtype):
        K, c_in, c_out = kernel.shape
        _assert(K == km.K, "kernel volume", K, "does not match the kernel map", km.K)
        _, w_t = _packed_weights(kernel, in_feat.dtype)
        out = torch.empty((km.n_out, c_out), dtype=out_dtype or in_feat.dtype,
                          device=in_feat.device)
        rc = lib.meb200_conv_forward_packed(
            _lib.ptr(in_feat), code, km.n_in, c_in, _lib.ptr(w_t), None, K, c_out,
            _lib.ptr(km.out_nbr), km.n_out, _lib.ptr(out), _lib.dtype_code(out.dtype),
            _lib.current_stream())
        if rc != _ERR_UNSUPPORTED:
            _lib.check(rc)
            return out
    if kernel.dtype != in_feat.dtype:
        kernel = kernel.to(in_feat.dtype)
    kernel = kernel.contiguous()
    K, c_in, c_out = kernel.shape
    _assert(K == km.K, "kernel volume", K, "does not match the kernel map", km.K)
    n_out, n_in = km.n_out, km.n_in
    out = torch.empty((n_out, c_out), dtype=out_dtype or in_feat.dtype, device=in_feat.device)
    ws, ws_bytes = _workspace(n_in, n_out, c_in, c_out, K, code, in_feat.device)
    _lib.check(lib.meb200_conv_forward(
        _lib.ptr(in_feat), code, n_in, c_in, _lib.ptr(kernel), K, c_out, _lib.ptr(km.out_nbr),
        n_out, _lib.ptr(out), _lib.dtype_code(out.dtype), _lib.ptr(ws), ws_bytes,
        _lib.current_stream()))
    return out


def _conv_backward(in_feat, grad_out, kernel, km, need_in=True, need_w=True):
    if _PROFILE is not None:
        esz = in_feat.element_size()
        K, c_in, c_out = kernel.shape
        P = km.n_pairs
        flops = 2.0 * P * c_in * c_out
        gi = gw = None
        if need_in:   # dgrad alone: dOut in, dIn out, W, table
            nb = km.n_out * c_out * esz + km.n_in * c_in * esz + K * c_in * c_out * esz + P * 8
            gi, _ = _record("conv_fwd_dgrad", lambda: _conv_backward_impl(
                in_feat, grad_out, kernel, km, True, False), flops, nb)
        if need_w:    # wgrad alone: In and dOut in, dW (fp32) out, table
            nb = km.n_in * c_in * esz + km.n_out * c_out * esz + K * c_in * c_out * 4 + P * 8
            _, gw = _record("conv_wgrad", lambda: _conv_backward_impl(
                in_feat, grad_out, kernel, km, False, True), flops, nb)
        return gi, gw
    return _conv_backward_impl(in_feat, grad_out, kernel, km, need_in, need_w)


def _conv_backward_impl(in_feat, grad_out, kernel, km, need_in=True, need_w=True):
    lib = _lib.load()
    code = _lib.dtype_code(in_feat.dtype)
    if grad_out.dtype != in_feat.dtype:
        grad_out = grad_out.to(in_feat.dtype)
    grad_out = grad_out.contiguous()
    K, c_in, c_out = kernel.shape
    n_out, n_in = km.n_out, km.n_in
    grad_in = torch.empty((n_in, c_in), dtype=in_feat.dtype, device=in_feat.device) \
        if need_in else None
    grad_w = torch.empty((K, c_in, c_out), dtype=torch.float32, device=in_feat.device) \
        if need_w else None
    if need_w and not need_in and _is_stem(kernel, in_feat.dtype):
        # the stem's input needs no gradient (it is the network input): wgrad alone
        V = int(lib.meb200_conv_stem_virtual_channels(K))
        gwv = torch.empty((V // 4, 4, c_out), dtype=torch.float32, device=in_feat.device)
        in4 = _pad4(in_feat)
        ws, ws_bytes = _wgrad_workspace(V, c_out, 1, n_out, in_feat.device)
        rc = lib.meb200_conv_stem_wgrad(
            _lib.ptr(in4), _lib.ptr(grad_out), code, K, c_out, _lib.ptr(km.out_nbr),
            n_out, _lib.ptr(gwv), _lib.ptr(ws), ws_bytes, _lib.current_stream())
        if rc != _ERR_UNSUPPORTED:
            _lib.check(rc)
            return None, gwv[:K, :c_in].contiguous()
    if _can_pack(kernel, in_feat.dtype):
        w, _ = _packed_weights(kernel, in_feat.dtype)
        pin = pout = seg = None
        nch = 0
        if need_w and c_in % 8 == 0 and c_in >= 16 and K <= 1023:
            pin, pout, seg, nch = km.pair_lists()
        ws, ws_bytes = _wgrad_workspace(c_in, c_out, K, n_out, in_feat.device) if need_w \
            else (None, 0)
        rc = lib.meb200_conv_backward_packed(
            _lib.ptr(in_feat), _lib.ptr(grad_out), code, n_in, c_in, _lib.ptr(w), None,
            K, c_out, _lib.ptr(km.out_nbr), _lib.ptr(km.in_nbr) if need_in else None, n_out,
            _lib.ptr(grad_in), code, _lib.ptr(grad_w), _lib.ptr(pin), _lib.ptr(pout), _lib.ptr(seg), nch,
            _lib.ptr(ws), ws_bytes, _lib.current_stream())
        if rc != _ERR_UNSUPPORTED:
            _lib.check(rc)
            return grad_in, grad_w
    else:
        w = kernel if kernel.dtype == in_feat.dtype else kernel.to(in_feat.dtype)
        w = w.contiguous()
    ws, ws_bytes = _workspace(n_in, n_out, c_in, c_out, K, code, in_feat.device)
    _lib.check(lib.meb200_conv_backward(
        _lib.ptr(in_feat), _lib.ptr(grad_out), code, n_in, c_in, _lib.ptr(w), K, c_out,
        _lib.ptr(km.out_nbr), _lib.ptr(km.in_nbr) if need_in else None, n_out, _lib.ptr(grad_in),
        code, _lib.ptr(grad_w), _lib.ptr(ws), ws_bytes, _lib.current_stream()))
    if grad_w is not None and grad_w.dtype != kernel.dtype:
        grad_w = grad_w.to(kernel.dtype)
    return grad_in, grad_w


def ConvolutionForwardGPU(in_feat, kernel, kernel_size, kernel_stride, kernel_dilation,
                          region_type, offset, expand_coordinates, convolution_mode, in_key,
                          out_key, manager):
    """reference: ConvolutionForwardGPU src/convolution_gpu.cu:45-159 (CPU twin
    convolution_cpu.cpp:42-135).  Mutates `out_key` when it is unset."""
    _assert(kernel.dim() == 3, "kernel.dim():", kernel.dim())
    _assert(kernel.is_cuda, "kernel must be CUDA")
    _check_feats(in_feat, manager, in_key)
    _assert(in_feat.size(1) == kernel.size(1), "Input feature size and kernel size mismatch")
    if not out_key.is_key_set():
        if expand_coordinates:
            ik = manager._k(in_key)
            out_ts = [t * int(s) for t, s in zip(ik[0], kernel_stride)]
            ok, _ = manager._stride_region(in_key, region_type, kernel_size, kernel_dilation,
                                           offset, ik[0], out_ts, False, True)
        else:
            ok, _ = manager._stride(in_key, kernel_stride)
        out_key.set_key(list(ok[0]), ok[1])
    km = manager._kernel_map(in_key, out_key, kernel_size, kernel_stride, kernel_dilation,
                             region_type, offset, False, False)
    return _conv_forward(in_feat, kernel, km)


def ConvolutionBackwardGPU(in_feat, grad_out_feat, kernel, kernel_size, kernel_stride,
                           kernel_dilation, region_type, offset, convolution_mode, in_key,
                           out_key, manager, need_in=True, need_w=True):
    """reference: ConvolutionBackwardGPU src/convolution_gpu.cu:161-244"""
    _check_feats(in_feat, manager, in_key)
    _assert(manager.exists(out_key), ERROR_MAP_NOT_FOUND)
    _assert(grad_out_feat.size(0) == manager.size(out_key), "Invalid grad_out size")
    km = manager._kernel_map(in_key, out_key, kernel_size, kernel_stride, kernel_dilation,
                             region_type, offset, False, False)
    return _conv_backward(in_feat, grad_out_feat, kernel, km, need_in, need_w)


def ConvolutionTransposeForwardGPU(in_feat, kernel, kernel_size, kernel_stride,
                                   kernel_dilation, region_type, offset,
                                   generate_new_coordinates, convolution_mode, in_key, out_key,
                                   manager):
    """reference: src/convolution_transpose_gpu.cu (CPU twin convolution_transpose_cpu.cpp:42-125)"""
    _assert(kernel.dim() == 3, "kernel.dim():", kernel.dim())
    _check_feats(in_feat, manager, in_key)
    _assert(in_feat.size(1) == kernel.size(1), "Input feature size and kernel size mismatch")
    if not out_key.is_key_set():
        ik = manager._k(in_key)
        for t, s in zip(ik[0], kernel_stride):
            _assert(t % int(s) == 0, "Invalid up stride on tensor stride:", list(ik[0]),
                    "kernel stride:", list(kernel_stride))
        out_ts = [t // int(s) for t, s in zip(ik[0], kernel_stride)]
        ok, _ = manager._stride_region(in_key, region_type, kernel_size, kernel_dilation, offset,
                                       out_ts, out_ts, True, generate_new_coordinates)
        out_key.set_key(list(ok[0]), ok[1])
    km = manager._kernel_map(in_key, out_key, kernel_size, kernel_stride, kernel_dilation,
                             region_type, offset, True, False)
    return _conv_forward(in_feat, kernel, km)


def ConvolutionTransposeBackwardGPU(in_feat, grad_out_feat, kernel, kernel_size, kernel_stride,
                                    kernel_dilation, region_type, offset, convolution_mode,
                                    in_key, out_key, manager, need_in=True, need_w=True):
    _check_feats(in_feat, manager, in_key)
    _assert(manager.exists(out_key), ERROR_MAP_NOT_FOUND)
    km = manager._kernel_map(in_key, out_key, kernel_size, kernel_stride, kernel_dilation,
                             region_type, offset, True, False)
    return _conv_backward(in_feat, grad_out_feat, kernel, km, need_in, need_w)


_POOL_CODE = {PoolingMode.LOCAL_SUM_POOLING: _lib.POOL_SUM,
              PoolingMode.LOCAL_AVG_POOLING: _lib.POOL_AVG,
              PoolingMode.LOCAL_MAX_POOLING: _lib.POOL_MAX}


def LocalPoolingForwardGPU(in_feat, kernel_size, kernel_stride, kernel_dilation, region_type,
                           offset, pooling_mode, in_key, out_key, manager):
    """reference: LocalPoolingForwardGPU src/local_pooling_gpu.cu:46-137 (CPU twin
    local_pooling_cpu.cpp:43-120) -> (out_feat, num_nonzero | max_index)"""
    _check_feats(in_feat, manager, in_key)
    _assert(pooling_mode in _POOL_CODE, "Invalid pooling mode", pooling_mode)
    if not out_key.is_key_set():
        ok, _ = manager._stride(in_key, kernel_stride)
        out_key.set_key(list(ok[0]), ok[1])
    km = manager._kernel_map(in_key, out_key, kernel_size, kernel_stride, kernel_dilation,
                             region_type, offset, False, True)
    lib = _lib.load()
    C = in_feat.size(1)
    n_out = km.n_out
    out = torch.empty((n_out, C), dtype=in_feat.dtype, device=in_feat.device)
    mode = _POOL_CODE[pooling_mode]
    if mode == _lib.POOL_MAX:
        aux = torch.empty((n_out, C), dtype=torch.int32, device=in_feat.device)
    elif mode == _lib.POOL_AVG:
        aux = torch.empty(n_out, dtype=in_feat.dtype, device=in_feat.device)
    else:
        aux = torch.empty(0, dtype=in_feat.dtype, device=in_feat.device)
    _lib.check(lib.meb200_pool_forward(
        _lib.ptr(in_feat), _lib.dtype_code(in_feat.dtype), km.n_in, C, _lib.ptr(km.out_nbr),
        km.K, n_out, mode, _lib.ptr(out), _lib.ptr(aux) if aux.numel() else None,
        _lib.current_stream()))
    return out, aux


def LocalPoolingBackwardGPU(in_feat, grad_out_feat, num_nonzero, kernel_size, kernel_stride,
                            kernel_dilation, region_type, offset, pooling_mode, in_key, out_key,
                            manager):
    """reference: LocalPoolingBackwardGPU src/local_pooling_gpu.cu:139-220"""
    _check_feats(in_feat, manager, in_key)
    _assert(manager.exists(out_key), ERROR_MAP_NOT_FOUND)
    grad_out_feat = grad_out_feat.contiguous()
    _assert(in_feat.dtype == grad_out_feat.dtype, "type mismatch")
    km = manager._kernel_map(in_key, out_key, kernel_size, kernel_stride, kernel_dilation,
                             region_type, offset, False, True)
    lib = _lib.load()
    C = in_feat.size(1)
    mode = _POOL_CODE[pooling_mode]
    if mode == _lib.POOL_MAX:
        grad_in = torch.zeros_like(in_feat)
    else:
        grad_in = torch.empty_like(in_feat)
    _lib.check(lib.meb200_pool_backward(
        _lib.ptr(grad_out_feat), _lib.dtype_code(in_feat.dtype), km.n_in, C, _lib.ptr(km.in_nbr),
        km.K, km.n_out, mode, _lib.ptr(num_nonzero) if num_nonzero.numel() else None,
        _lib.ptr(grad_in), _lib.current_stream()))
    return grad_in
