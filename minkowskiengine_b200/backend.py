"""Host-side mirror of the reference's native boundary `MinkowskiEngineBackend._C`
(pybind/extern.hpp:515-838) for the sparse-convolution hot path.

Same names, argument order and side effects as the reference's `...GPU` functions and
`CoordinateMapManagerGPU_c10`, but the bodies are thin: they validate, keep the manager's
bookkeeping (key naming / reuse / kernel-map cache — coordinate_map_manager.cpp:353-466,
662-823) and hand device pointers to the C-ABI library (include/meb200.h).  All device
work happens in libmeb200.so on torch's current CUDA stream; the only host<->device
synchronisation is the unique-row count read when a NEW coordinate map is created.
"""
import contextlib
import ctypes
import os
import random
import string
import threading
import warnings
import weakref

import torch

from . import _lib
from .enums import BroadcastMode, MinkowskiAlgorithm, PoolingMode, RegionType
from .kernel_generator import region_offsets

ERROR_MAP_NOT_FOUND = "CoordinateMap not found"  # reference: src/errors.hpp:33
ERROR_FIELD_DOMAIN = "TensorField coordinates must be finite and quantise to int32 voxels"


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
        """Deduplicating insert of candidate rows (meb200_insert_and_map) -> (map, unique_index,
        inverse_map): rows numbered by first occurrence, -1 for a row that is not `valid`.  Zero
        candidates give a 0-row map over an empty table without a native call."""
        n, ncols = candidates.shape
        dev = candidates.device
        if n == 0:
            table = _new_table(0, dev).fill_(-1)
            empty = torch.empty(0, dtype=torch.int64, device=dev)
            return _CoordinateMap(candidates, table, table.numel(), tensor_stride), empty, empty
        table, uniq, uidx, inv, scratch = _insert_buffers(n, ncols, dev)
        m = ctypes.c_uint32(0)
        _lib.check(_lib.load().meb200_insert_and_map(
            _lib.ptr(candidates), _lib.ptr(valid), n, ncols, _lib.ptr(table), table.numel(),
            _lib.ptr(uniq), _lib.ptr(uidx), _lib.ptr(inv), _lib.ptr(scratch), ctypes.byref(m),
            _lib.current_stream()))
        m = int(m.value)
        return _CoordinateMap(uniq[:m], table, table.numel(), tensor_stride), uidx[:m], inv


def _c_ints(values):
    return (ctypes.c_int32 * len(values))(*values)


def _new_table(n, dev):
    """Uninitialised row-index table sized for n rows (meb200_hash_capacity slots)."""
    return torch.empty(int(_lib.load().meb200_hash_capacity(n)), dtype=torch.int32, device=dev)


def _insert_buffers(n, ncols, dev):
    """(table, unique rows, unique_index, inverse_map, scratch) of an insert of n candidate rows."""
    table = _new_table(n, dev)
    return (table, torch.empty((n, ncols), dtype=torch.int32, device=dev),
            torch.empty(n, dtype=torch.int64, device=dev),
            torch.empty(n, dtype=torch.int64, device=dev),
            torch.empty(int(_lib.load().meb200_insert_scratch_bytes(n)), dtype=torch.uint8,
                        device=dev))


def _distinct_map(coords, tensor_stride, table=None):
    """Map over rows known to be distinct (meb200_map_build_table), built into `table` when given
    (a power of two of at least twice the rows), else into a table sized for the rows."""
    if table is None:
        table = _new_table(coords.shape[0], coords.device)
    _lib.check(_lib.load().meb200_map_build_table(_lib.ptr(coords), coords.shape[0],
                                                  coords.shape[1], _lib.ptr(table), table.numel(),
                                                  _lib.current_stream()))
    return _CoordinateMap(coords, table, table.numel(), tensor_stride)


def _strided(coords, tensor_stride):
    """Candidate rows: every row of `coords` floored to `tensor_stride` (meb200_stride_coords)."""
    out = torch.empty_like(coords)
    _lib.check(_lib.load().meb200_stride_coords(_lib.ptr(coords), coords.shape[0], coords.shape[1],
                                                _c_ints(tensor_stride), _lib.ptr(out),
                                                _lib.current_stream()))
    return out


def _find_rows(cmap, query):
    """int64 row of every query row in map `cmap`, -1 where it has none (meb200_map_find)."""
    res = torch.empty(query.shape[0], dtype=torch.int32, device=query.device)
    _lib.check(_lib.load().meb200_map_find(_lib.ptr(cmap.coords), _lib.ptr(cmap.table),
                                           cmap.capacity, cmap.ncols, _lib.ptr(query),
                                           query.shape[0], _lib.ptr(res), _lib.current_stream()))
    return res.long()


_COORDINATE_DTYPE_ERROR = {torch.int32: "coordinates must be an IntTensor",
                           torch.float32: "field coordinates must be a FloatTensor"}


def _check_coordinates(coordinates, tensor_stride, dtype):
    """Checks the int32 coordinates of a map or the float32 points of a field handed to the
    manager -> the tensor stride as a list of ints."""
    _assert(coordinates.dim() == 2, "coordinates must be 2-dimensional")
    _assert(coordinates.dtype == dtype, _COORDINATE_DTYPE_ERROR[dtype])
    _assert(coordinates.is_contiguous(), "coordinates must be contiguous")
    _assert(coordinates.is_cuda,
            "coordinates must be a CUDA tensor: minkowskiengine_b200 implements the GPU "
            "coordinate manager only (no CPU backend, no fallback)")
    ts = [int(v) for v in tensor_stride]
    _assert(coordinates.size(1) - 1 == len(ts),
            "The coordinate dimension (coordinate_size - 1):", coordinates.size(1) - 1,
            " must match the size of tensor stride:", ts)
    return ts


# ---- map prediction (DESIGN.md §2) ---------------------------------------------------------------
# A strided map is a function of the input coordinates alone, but creating it where the network
# first asks for it costs a blocking read of its size with the whole forward pass queued in front
# (the host's lead over the GPU is lost at every down-sampling layer, and the coarse levels —
# 10-30 us kernels — then run launch bound).  So the pyramid the PREVIOUS manager of the same
# coordinate width was asked for is enqueued right behind the first inserted map, on upper-bound
# buffers with device-side row counts (meb200_insert_and_map_enqueue); its sizes reach the host
# long before the layers that need them.  The kernel maps are functions of the coordinate maps as
# well: the ones the previous manager was asked for are built right there, before the first layer
# runs.  The GPU gets ~1.5 ms of table probing to chew on while the host enqueues the layers,
# instead of meeting each map where the forward pass first needs it with nothing else queued.
# A wrong prediction is only wasted work: a level that is never requested, or requested with
# another stride, is dropped.
_PREFETCH = os.environ.get("MEB200_MAP_PREFETCH", "1") not in ("", "0")


class _Hint:
    """What the last manager of one coordinate width was asked for: the kernel strides along the
    stride chain below its first inserted map, its kernel maps in order (cache keys, no tensors)
    and the cache keys of those whose pair lists (wgrad) were built."""

    __slots__ = ("pyramid", "kernel_maps", "pairs")

    def __init__(self):
        self.pyramid, self.kernel_maps, self.pairs = (), (), set()


_HINTS = {}     # coordinate width -> _Hint


def _hint(ncols):
    return _HINTS.setdefault(ncols, _Hint())


class _PendingLevel:
    """One level of a stride pyramid whose kernels are enqueued but whose size has not been read
    yet (see _Prediction.start)."""

    __slots__ = ("parent_key", "tensor_stride", "uniq", "inverse", "count_dev", "count_host",
                 "event")


class _Prediction:
    """The map prediction of one manager: it records what the manager is asked for from its first
    inserted map on (into _HINTS), and builds what the previous manager was asked for behind that
    map.  The manager is passed in, not kept: a manager must die by reference counting alone."""

    __slots__ = ("ncols", "chain_tip", "chain", "seen", "requests", "replaying", "pending")

    def __init__(self):
        self.ncols = None       # width of the first inserted map, once there is one
        self.chain_tip = None   # last map of the stride chain below that map
        self.chain = []         # kernel strides requested along that chain
        self.seen = set()       # kernel-map cache keys the caller has asked for
        self.requests = []      # ... in order, from the first inserted map on
        self.replaying = False  # building predicted kernel maps, which are not requests
        self.pending = {}       # out key -> _PendingLevel (enqueued, size not yet read)

    def start(self, mgr, key, cmap):
        """`key` is the first map inserted into `mgr`."""
        self.ncols, self.chain_tip = cmap.ncols, key
        hint = _HINTS.get(cmap.ncols) if _PREFETCH else None
        if hint is not None:
            self._enqueue_pyramid(mgr, key, cmap, hint.pyramid)
            self._build_kernel_maps(mgr, hint)

    def stride_requested(self, in_key, out_key, kernel_stride):
        if in_key == self.chain_tip and out_key != in_key and not self.replaying:
            self.chain_tip = out_key
            self.chain.append(tuple(int(s) for s in kernel_stride))
            _hint(self.ncols).pyramid = tuple(self.chain)

    def kernel_map_requested(self, cache_key, region_type):
        if self.replaying or cache_key in self.seen:
            return
        self.seen.add(cache_key)
        if region_type != RegionType.CUSTOM and self.ncols is not None:
            self.requests.append(cache_key)
            _hint(self.ncols).kernel_maps = tuple(self.requests)

    def take(self, mgr, in_key, out_key):
        """Makes the enqueued level `out_key` a map of `mgr` if it was built from `in_key`."""
        lv = self.pending.pop(out_key, None)
        if lv is None or lv.parent_key != in_key:
            return False
        lv.event.synchronize()          # normally long past: enqueued before the first layer
        m = int(lv.count_host.item())
        mgr._maps[out_key] = _distinct_map(lv.uniq[:m], lv.tensor_stride)
        mgr._parents[out_key] = (in_key, lv.inverse[:mgr._maps[in_key].size])
        return True

    def _enqueue_pyramid(self, mgr, key, cmap, strides):
        if not strides or cmap.size == 0:
            return
        n, ncols, dev = cmap.size, cmap.ncols, cmap.coords.device
        parent_key, parent_coords, parent_count = key, cmap.coords, None
        for ks in strides:
            if len(ks) != len(parent_key[0]):
                return
            out_ts = tuple(t * s for t, s in zip(parent_key[0], ks))
            out_key = (out_ts, parent_key[1])
            if out_key in mgr._maps or out_key in self.pending:
                return
            # rows past the parent's (device-side) count are whatever the buffer holds: they are
            # strided like the others and then ignored by the insert
            cand = _strided(parent_coords, out_ts)
            table, uniq, uidx, inverse, scratch = _insert_buffers(n, ncols, dev)
            lv = _PendingLevel()
            lv.parent_key, lv.tensor_stride, lv.uniq, lv.inverse = parent_key, out_ts, uniq, inverse
            lv.count_dev = torch.empty(1, dtype=torch.int32, device=dev)
            _lib.check(_lib.load().meb200_insert_and_map_enqueue(
                _lib.ptr(cand), None, _lib.ptr(parent_count), n, ncols, _lib.ptr(table),
                table.numel(), _lib.ptr(uniq), _lib.ptr(uidx), _lib.ptr(inverse), _lib.ptr(scratch),
                _lib.ptr(lv.count_dev), _lib.current_stream()))
            lv.count_host = torch.empty(1, dtype=torch.int32, pin_memory=True)
            lv.count_host.copy_(lv.count_dev, non_blocking=True)
            lv.event = torch.cuda.Event()
            lv.event.record()
            self.pending[out_key] = lv
            parent_key, parent_coords, parent_count = out_key, uniq, lv.count_dev

    def _materialize(self, mgr, key):
        if key in mgr._maps:
            return True
        lv = self.pending.get(key)
        return (lv is not None and self._materialize(mgr, lv.parent_key)
                and self.take(mgr, lv.parent_key, key))

    def _build_kernel_maps(self, mgr, hint):
        self.replaying = True
        try:
            for ck in hint.kernel_maps:
                ik, ok, ksize, kstride, kdil, region, is_transpose, is_pool = ck
                if self._materialize(mgr, ik) and self._materialize(mgr, ok):
                    km = mgr._kernel_map(ik, ok, ksize, kstride, kdil, region, None, is_transpose,
                                         is_pool)
                    if ck in hint.pairs:
                        km.pair_lists()          # the backward pass will want them
        finally:
            self.replaying = False


class _KernelMap:
    """k-major neighbour tables of one (in map, out map, kernel) triple.

    out_nbr[k, o] = input row reached from output row o through offset k (or -1)
    in_nbr [k, i] = output row that input row i feeds through offset k (or -1)
    Replaces gpu_kernel_map's three flat arrays + host offset table (src/kernel_map.cuh:48-429);
    `swapped()` is the reference's swap_in_out (kernel_map.cuh:191-241)."""

    __slots__ = ("out_nbr", "_in_nbr", "_in_thunk", "_n_in", "stride_pairs", "_n_pairs", "_pairs",
                 "_pair_src", "_hint_key", "out_order", "in_order")
    PAIR_STAGE = 64   # pairs per pipeline stage of the wgrad kernel (k_wgrad_wg)
    # table rows per chunk of the pair lists (multiple of 2048): one chunk's rows of both feature
    # matrices stay L2-resident while the wgrad walks its K offsets
    PAIR_CHUNK_ROWS = 262144

    def __init__(self, out_nbr, in_nbr, stride_pairs=None, n_in=None, in_thunk=None, orders=None):
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
        # tile orders of out_nbr / in_nbr (meb200_kernel_map, include/meb200.h) or None: the
        # forward reads the first, the dgrad the second
        self.out_order, self.in_order = orders if orders is not None else (None, None)

    def pair_lists(self):
        """(pairs_in, pairs_out, seg_start, n_chunks): compacted (input row, output row) lists in
        (row chunk, offset) order, every segment padded to PAIR_STAGE entries
        (meb200_kernel_map_pairs) — the reference's own kernel-map representation, chunked so
        that a consumer keeps one chunk's feature rows L2-resident across the offsets.  Built on
        first use; a swapped view shares its source's lists with the two sides exchanged."""
        if self._pairs is None:
            if self._hint_key is not None:     # (its in map's key gives the width)
                _hint(len(self._hint_key[0][0]) + 1).pairs.add(self._hint_key)
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
        km = _KernelMap(self.in_nbr, self.out_nbr, sp, orders=(self.in_order, self.out_order))
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


MAX_ORDER_K = 32     # tile orders are built for convolution tables of 2..32 offsets


def tile_order_words(K, n):
    """int32 words of the tile order of a [K, n] table (include/meb200.h, meb200_kernel_map)."""
    return (K + 1) * n + (n + 127) // 128


def tile_order_scratch_bytes(n):
    """Scratch bytes meb200_kernel_map needs to build the tile orders of tables of up to n rows."""
    return 4 * (2 * n + 256 * ((n + 2047) // 2048) + 256)


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
        self._prediction = _Prediction()
        self._inserted = []     # keys of the maps made by insert_and_map, in order
        self._origin_covers = 0  # ... how many of them the origin map was built from
        self._groupings = {}    # map key -> _OriginGrouping
        # field key -> _OriginGrouping of its points: apart from _groupings, because a field key and
        # a map key may be the same tuple
        self._field_groupings = {}
        self._origin_fields = set()  # field keys the origin map was built from
        self._prunes = {}       # (in key, out key) -> (unique_index, inverse_map) of a pruned map
        self._unions = {}       # tuple of input keys -> _UnionMap
        self._fields = {}       # field key -> float32 [N, D+1] point coordinates
        self._field_maps = {}   # (field key, map key) -> _FieldToSparse
        self._field_quant = {}  # (field key, tensor stride, string id) -> map key it quantised to
        self._field_valid = set()  # field keys whose coordinates a quantisation has checked
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

    def _free_key(self, tensor_stride, string_id, taken):
        """(tensor stride, string_id), with a random suffix when `taken` holds that key."""
        key = (tuple(tensor_stride), string_id)
        while key in taken:
            key = (key[0], self.get_random_string_id(key[0], string_id)[1])
        return key

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
        ts = _check_coordinates(coordinates, tensor_stride, torch.int32)
        key = self._free_key(ts, string_id, self._maps)
        cmap, unique_index, inverse_map = _CoordinateMap.build(coordinates, ts)
        self._add_inserted(key, cmap)
        if cmap.size == coordinates.size(0):
            # no duplicates: the reference GPU path returns an empty inverse map here
            # (coordinate_map_manager.cu:94-112) and Python substitutes arange
            inverse_map = inverse_map[:0]
        return CoordinateMapKey(list(key[0]), key[1]), (unique_index, inverse_map)

    def _add_inserted(self, key, cmap):
        """Registers a map made from input coordinates (insert_and_map, or the quantisation of a
        tensor field): the first one starts the predicted pyramid and kernel maps, and every one
        counts towards the origin map."""
        first = not self._inserted   # (an origin map built from fields may exist already)
        self._maps[key] = cmap
        self._inserted.append(key)
        if first:
            self._prediction.start(self, key, cmap)

    def _stride(self, in_key, kernel_stride, string_id=""):
        """reference: coordinate_map_manager.cpp:406-429 -> (out key tuple, created?)"""
        in_key = self._k(in_key)
        _assert(in_key in self._maps, ERROR_MAP_NOT_FOUND)
        _assert(len(kernel_stride) == len(in_key[0]), "stride size mismatch.")
        out_ts = tuple(t * int(s) for t, s in zip(in_key[0], kernel_stride))
        out_key = (out_ts, string_id if string_id else in_key[1])
        self._prediction.stride_requested(in_key, out_key, kernel_stride)
        if out_key in self._maps:
            return out_key, False
        if self._prediction.take(self, in_key, out_key):
            return out_key, True
        out_map, _, inverse = _CoordinateMap.build(_strided(self._maps[in_key].coords, out_ts),
                                                   out_ts)
        self._maps[out_key] = out_map
        self._parents[out_key] = (in_key, inverse)
        return out_key, True

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
        _lib.check(lib.meb200_region_coords(
            _lib.ptr(in_map.coords), n, in_map.ncols, _lib.ptr(offs), K, _c_ints(out_ts),
            0 if is_transpose else 1, _lib.ptr(cand), _lib.ptr(valid), _lib.current_stream()))
        out_map, _, _ = _CoordinateMap.build(cand, out_ts, valid)
        out_map.coords = out_map.coords.clone()  # drop the n*K candidate buffer
        out_key = self._free_key(out_ts, "", self._maps)
        self._maps[out_key] = out_map
        return out_key, True

    # -- kernel maps -----------------------------------------------------------------
    LAZY_REVERSE_K = 64      # kernels this large get their reverse table on demand

    @staticmethod
    def _probe(x_map, y_map, offsets, need_y=True, orders=False):
        """x-stationary probe: returns (x_nbr [K,nx], y_nbr [K,ny] or None), and with `orders` (and
        y) also the tile orders of both tables, (x_order, y_order) or (None, None) where K is
        outside 2..MAX_ORDER_K.  (Static: the deferred reverse-table build below must not keep the
        manager alive through a reference cycle — a manager owns ~1.5 GB of tables on the bench
        clouds and should die with its tensors.)"""
        lib = _lib.load()
        K = offsets.shape[0]
        dev = x_map.coords.device
        x_nbr = torch.empty((K, x_map.size), dtype=torch.int32, device=dev)
        y_nbr = torch.full((K, y_map.size), -1, dtype=torch.int32, device=dev) if need_y else None
        x_order = y_order = scratch = None
        if orders and need_y and 2 <= K <= MAX_ORDER_K:
            x_order = torch.empty(tile_order_words(K, x_map.size), dtype=torch.int32, device=dev)
            y_order = torch.empty(tile_order_words(K, y_map.size), dtype=torch.int32, device=dev)
            scratch = torch.empty(tile_order_scratch_bytes(max(x_map.size, y_map.size)),
                                  dtype=torch.uint8, device=dev)

        def launch():
            _lib.check(lib.meb200_kernel_map(
                _lib.ptr(x_map.coords), x_map.size, _lib.ptr(y_map.coords), y_map.size,
                _lib.ptr(y_map.table), y_map.capacity, x_map.ncols, _lib.ptr(offsets), K,
                _lib.ptr(x_nbr), _lib.ptr(y_nbr), None, _lib.ptr(x_order), _lib.ptr(y_order),
                _lib.ptr(scratch), _lib.current_stream()))
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
        if orders:
            return x_nbr, y_nbr, x_order, y_order
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
        self._prediction.kernel_map_requested(cache_key, region_type)
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
                    out_nbr, in_nbr, *orders = self._probe(out_map, in_map, offs, orders=not is_pool)
                    km = _KernelMap(out_nbr, in_nbr, orders=orders or None)
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
                    a, b, *orders = self._probe(in_map, out_map, offs, orders=not is_pool)
                    fwd = _KernelMap(a, b, orders=orders or None)
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
            inv = _find_rows(out_map, _strided(in_map.coords, out_map.tensor_stride))
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

    # -- origin map and per-cloud grouping ---------------------------------------------
    def _origin_key(self, ncols):
        return (tuple([0] * (ncols - 1)), "")

    def _origin(self):
        """reference: coordinate_map_manager.cpp:474-508.  The origin map holds one row
        (b, 0, ..., 0) per batch index of the inserted maps, in ASCENDING batch order; built once
        (the one host read is its row count B) and cached under the key ([0]*D, "").  A manager
        that holds only tensor fields builds it from the batch columns of its fields (reference:
        origin_field, coordinate_map_manager.cpp), rounded with lroundf as the quantisation
        rounds them; a batch value that is not finite or outside int32 raises ValueError."""
        if self._inserted:
            ncols = self._maps[self._inserted[0]].ncols
        else:
            _assert(len(self._fields) > 0, "No coordinate map found")
            ncols = next(iter(self._fields.values())).size(1)
        key = self._origin_key(ncols)
        if key in self._maps:
            return key
        if self._inserted:
            batch = torch.cat([self._maps[k].coords[:, 0] for k in self._inserted])
            cand = torch.zeros((batch.numel(), ncols), dtype=torch.int32, device=batch.device)
            cand[:, 0] = batch
            cmap, _, _ = _CoordinateMap.build(cand, key[0])
        else:
            cmap = self._field_origin(key[0])
        # ascending batch index: rebuild the table over the sorted rows
        coords = cmap.coords[torch.argsort(cmap.coords[:, 0])].contiguous()
        self._maps[key] = _distinct_map(coords, key[0], cmap.table)
        self._origin_covers = len(self._inserted)
        return key

    def _field_origin(self, tensor_stride):
        """The rows (lroundf(b), 0, ..., 0) of every field's points, deduplicated
        (meb200_field_origin_insert: the validity of the batch column comes with the row count)."""
        fks = list(self._fields)
        field = torch.cat([self._fields[k] for k in fks]) if len(fks) > 1 else self._fields[fks[0]]
        n, ncols = field.shape
        ocoords = torch.empty((n, ncols), dtype=torch.int32, device=field.device)
        table, uniq, uidx, inv, scratch = _insert_buffers(n, ncols, field.device)
        m = ctypes.c_uint32(0)
        rc = _lib.load().meb200_field_origin_insert(
            _lib.ptr(field), n, ncols, _lib.ptr(ocoords), _lib.ptr(table), table.numel(),
            _lib.ptr(uniq), _lib.ptr(uidx), _lib.ptr(inv), _lib.ptr(scratch), ctypes.byref(m),
            _lib.current_stream())
        if rc == _lib.ERR_DOMAIN:
            raise ValueError(ERROR_FIELD_DOMAIN)
        _lib.check(rc)
        self._origin_fields.update(fks)
        return _CoordinateMap(uniq[:int(m.value)], table, table.numel(), tensor_stride)

    def origin_field(self):
        """reference: MinkowskiCoordinateManager.py:273.  The one origin map of the manager, which
        pooling a field and pooling a map share."""
        return self.origin()

    def origin(self):
        k = self._origin()
        return CoordinateMapKey(list(k[0]), k[1])

    def origin_map_size(self):
        return self._maps[self._origin()].size

    def _origin_grouping(self, in_key):
        """Rows of map `in_key` grouped by cloud (cached per map, like kernel maps)."""
        ik = self._k(in_key)
        grp = self._groupings.get(ik)
        if grp is not None:
            return grp
        _assert(ik in self._maps, ERROR_MAP_NOT_FOUND)
        okey = self._origin()
        omap, imap = self._maps[okey], self._maps[ik]
        _assert(imap.ncols == omap.ncols, "coordinate size mismatch")
        lib = _lib.load()
        n, B, dev = imap.size, omap.size, imap.coords.device
        grp = _OriginGrouping()
        grp.n, grp.B = n, B
        grp.row_seg = torch.empty(n, dtype=torch.int32, device=dev)
        grp.order = torch.empty(n, dtype=torch.int32, device=dev)
        starts = torch.empty((2, B + 1), dtype=torch.int32, device=dev)
        grp.seg_start, grp.tile_start = starts[0], starts[1]
        scratch = torch.empty(int(lib.meb200_origin_group_scratch_bytes(n, B)), dtype=torch.uint8,
                              device=dev)
        _lib.check(lib.meb200_origin_group(
            _lib.ptr(imap.coords), n, imap.ncols, _lib.ptr(omap.coords), _lib.ptr(omap.table),
            omap.capacity, B, _lib.ptr(grp.row_seg), _lib.ptr(grp.order), _lib.ptr(grp.seg_start),
            _lib.ptr(grp.tile_start), _lib.ptr(scratch), _lib.current_stream()))
        if len(self._inserted) > self._origin_covers:
            # a map inserted after the origin map was built may hold batch indices it lacks: the
            # one case that needs a host read (maps derived from covered ones share their batches)
            _assert(int(grp.seg_start[B].item()) == n,
                    "the coordinate map holds batch indices that are not in the origin map")
        self._groupings[ik] = grp
        return grp

    def _field_grouping(self, field_key):
        """Points of field `field_key` grouped by cloud (meb200_field_origin_group), cached per field.
        The first grouping reads back, in one read, whether the batch column is valid and whether
        every point found its cloud; a field the origin map was built from needs neither."""
        fk, field = self._field(field_key)
        grp = self._field_groupings.get(fk)
        if grp is not None:
            return grp
        okey = self._origin()
        omap = self._maps[okey]
        _assert(field.size(1) == omap.ncols, "coordinate size mismatch")
        lib = _lib.load()
        n, B, dev = field.size(0), omap.size, field.device
        grp = _OriginGrouping()
        grp.n, grp.B = n, B
        grp.row_seg = torch.empty(n, dtype=torch.int32, device=dev)
        grp.order = torch.empty(n, dtype=torch.int32, device=dev)
        starts = torch.empty((2, B + 1), dtype=torch.int32, device=dev)
        grp.seg_start, grp.tile_start = starts[0], starts[1]
        scratch = torch.empty(int(lib.meb200_origin_group_scratch_bytes(n, B)), dtype=torch.uint8,
                              device=dev)
        check = fk not in self._origin_fields
        bad = torch.empty(1, dtype=torch.int32, device=dev) \
            if check and fk not in self._field_valid else None
        _lib.check(lib.meb200_field_origin_group(
            _lib.ptr(field), n, field.size(1), _lib.ptr(omap.coords), _lib.ptr(omap.table),
            omap.capacity, B, _lib.ptr(grp.row_seg), _lib.ptr(grp.order), _lib.ptr(grp.seg_start),
            _lib.ptr(grp.tile_start), _lib.ptr(bad), _lib.ptr(scratch), _lib.current_stream()))
        if check:
            words = (grp.seg_start[B:] if bad is None else torch.cat([bad, grp.seg_start[B:]]))
            words = words.tolist()
            if bad is not None and words[0] != 0:
                raise ValueError(ERROR_FIELD_DOMAIN)
            _assert(words[-1] == n, "the tensor field holds batch indices that are not in the "
                    "origin map")
        self._field_groupings[fk] = grp
        return grp

    def _grouping(self, key, is_field=False):
        """Per-cloud grouping of the rows of map `key`, or of the points of field `key`."""
        return self._field_grouping(key) if is_field else self._origin_grouping(key)

    def _origin_rows(self, grp):
        """(batch_indices int64 [B], [row indices (int64) of batch index b for b in 0..max batch
        index]) of a grouping."""
        okey = self._origin()
        batch = self._maps[okey].coords[:, 0].long()
        starts = grp.seg_start.tolist()
        rows = [torch.empty(0, dtype=torch.int64, device=batch.device)
                for _ in range(int(batch.max().item()) + 1 if batch.numel() else 0)]
        order = grp.order.long()
        for s, b in enumerate(batch.tolist()):
            rows[b] = order[starts[s]:starts[s + 1]]
        return batch, rows

    def origin_map(self, key):
        """reference: origin_map_th, coordinate_map_manager.cpp:828-885 -> (batch_indices int64
        [B], [row indices (int64) of batch index b for b in 0..max batch index])."""
        return self._origin_rows(self._origin_grouping(key))

    def origin_field_map(self, field_key):
        """reference: origin_field_map_th -> origin_map's form for the points of a field."""
        return self._origin_rows(self._field_grouping(field_key))

    # -- pruning and union -------------------------------------------------------------
    def _prune(self, in_key, keep):
        """reference: CoordinateMapManager::prune (coordinate_map_manager.cpp) -> out key tuple.
        Rows of the pruned map are the kept rows in ascending input order (the insert numbers rows
        by first occurrence).  Not cached: every call makes a new key at the input's stride."""
        ik = self._k(in_key)
        _assert(ik in self._maps, ERROR_MAP_NOT_FOUND)
        in_map = self._maps[ik]
        valid = keep if keep.dtype == torch.uint8 else keep.view(torch.uint8)
        cmap, uidx, inv = _CoordinateMap.build(in_map.coords, in_map.tensor_stride,
                                              valid.contiguous())
        ok = self.get_random_string_id(in_map.tensor_stride, "")
        self._maps[ok] = cmap
        self._prunes[(ik, ok)] = (uidx, inv)
        return ok

    def _union(self, in_keys):
        """The union map of `in_keys` (cached per ordered tuple of keys, as kernel maps are): rows of
        input 0 in order, then the new rows of input 1 in order, and so on."""
        iks = tuple(self._k(k) for k in in_keys)
        um = self._unions.get(iks)
        if um is not None:
            return um
        _assert(len(iks) >= 1, "union_map needs at least one input")
        for k in iks:
            _assert(k in self._maps, ERROR_MAP_NOT_FOUND, list(k[0]), k[1])
        maps = [self._maps[k] for k in iks]
        ts0, nc0 = maps[0].tensor_stride, maps[0].ncols
        for k, m in zip(iks, maps):
            _assert(m.tensor_stride == ts0, "union_map: tensor stride", list(m.tensor_stride),
                    "of", list(k[0]), k[1], "!= tensor stride", list(ts0), "of the first input")
            _assert(m.ncols == nc0, "union_map: coordinate size", m.ncols, "!=", nc0)
        cand = torch.cat([m.coords for m in maps]).contiguous()
        cmap, _, inv = _CoordinateMap.build(cand, ts0)
        ok = self.get_random_string_id(ts0, "")
        self._maps[ok] = cmap
        um = _UnionMap()
        um.key, um.M = ok, cmap.size
        um.sizes = [m.size for m in maps]
        um.u = list(torch.split(inv, um.sizes))
        um.src = torch.full((len(maps), cmap.size), -1, dtype=torch.int32, device=cand.device)
        for i, (u, n) in enumerate(zip(um.u, um.sizes)):
            # unique targets (coordinates are unique within an input): a deterministic scatter
            um.src[i, u] = torch.arange(n, dtype=torch.int32, device=cand.device)
        self._unions[iks] = um
        return um

    def union_map(self, in_keys, out_key):
        """reference: union_map_th (coordinate_map_manager.cpp) -> per input int64 [2, n_i] of
        (input rows, union rows); sets `out_key`."""
        um = self._union(in_keys)
        out_key.set_key(list(um.key[0]), um.key[1])
        return [torch.stack([torch.arange(n, dtype=torch.int64, device=u.device), u])
                for u, n in zip(um.u, um.sizes)]

    # -- tensor fields -------------------------------------------------------------------
    def insert_field(self, coordinates, tensor_stride, string_id=""):
        """reference: coordinate_map_manager.cpp:145-181.  The field keeps the float32 points."""
        ts = _check_coordinates(coordinates, tensor_stride, torch.float32)
        key = self._free_key(ts, string_id, self._fields)
        self._fields[key] = coordinates
        return CoordinateMapKey(list(key[0]), key[1])

    def _field(self, field_key):
        fk = self._k(field_key)
        _assert(fk in self._fields, "field", ERROR_MAP_NOT_FOUND)
        return fk, self._fields[fk]

    def get_coordinate_field(self, field_key):
        return self._field(field_key)[1]

    def _field_to_sparse(self, field_key, tensor_stride, string_id=""):
        """Quantises the field at `tensor_stride` into a new inserted map (meb200_field_insert_and_map)
        -> map key tuple.  Cached per (field, stride, string id): quantising again returns the same
        map and grouping."""
        fk, field = self._field(field_key)
        ts = tuple(_check_coordinates(field, tensor_stride, torch.float32))
        ck = (fk, ts, string_id)
        sk = self._field_quant.get(ck)
        if sk is not None:
            return sk
        n, ncols = field.shape
        q = torch.empty((n, ncols), dtype=torch.int32, device=field.device)
        table, uniq, uidx, inv, scratch = _insert_buffers(n, ncols, field.device)
        m = ctypes.c_uint32(0)
        rc = _lib.load().meb200_field_insert_and_map(
            _lib.ptr(field), n, ncols, _c_ints(ts), _lib.ptr(q), _lib.ptr(table), table.numel(),
            _lib.ptr(uniq), _lib.ptr(uidx), _lib.ptr(inv), _lib.ptr(scratch), ctypes.byref(m),
            _lib.current_stream())
        if rc == _lib.ERR_DOMAIN:
            raise ValueError(ERROR_FIELD_DOMAIN)
        _lib.check(rc)
        self._field_valid.add(fk)
        m = int(m.value)
        key = self._free_key(ts, string_id, self._maps)
        self._add_inserted(key, _CoordinateMap(uniq[:m], table, table.numel(), ts))
        self._field_maps[(fk, key)] = _FieldToSparse(inv, m, uidx[:m])
        self._field_quant[ck] = key
        return key

    def field_to_sparse_insert_and_map(self, field_key, tensor_stride, string_id=""):
        """reference: coordinate_map_manager.cpp:188-254 -> (map key, (unique_index, inverse_map));
        the inverse map is empty when no two points share a voxel, as for insert_and_map."""
        fk = self._k(field_key)
        sk = self._field_to_sparse(field_key, tensor_stride, string_id)
        f2s = self._field_maps[(fk, sk)]
        inv = f2s.inverse if f2s.M < f2s.inverse.numel() else f2s.inverse[:0]
        return CoordinateMapKey(list(sk[0]), sk[1]), (f2s.unique_index, inv)

    def field_to_sparse_map(self, field_key, sparse_key):
        """reference: coordinate_map_manager.cpp:282-330.  The points of the field quantised at the
        map's stride and looked up in it -> (inverse_map int64 [N]: row of every point, -1 where the
        map lacks its voxel; unique_index int64 [M]: the first point of every row, -1 for a row
        without points).  A field that no quantisation has checked yet costs one host read (the
        validity of its coordinates), once."""
        f2s = self._field_sparse_record(field_key, sparse_key)
        return f2s.inverse, f2s.first_points()

    def _field_sparse_record(self, field_key, sparse_key):
        fk, field = self._field(field_key)
        sk = self._k(sparse_key)
        f2s = self._field_maps.get((fk, sk))
        if f2s is not None:
            return f2s
        cmap = self._get(sk)
        _assert(cmap.ncols == field.size(1), "The coordinate dimension mismatch.", field.size(1),
                "!=", cmap.ncols)
        n, ncols = field.shape
        q = torch.empty((n, ncols), dtype=torch.int32, device=field.device)
        # the validity of the coordinates reaches the host with the row count of the first map made
        # from the field; only a field never quantised before pays a read here, once
        bad = None if fk in self._field_valid else \
            torch.empty(1, dtype=torch.int32, device=field.device)
        _lib.check(_lib.load().meb200_quantize_field(_lib.ptr(field), n, ncols,
                                                     _c_ints(cmap.tensor_stride), _lib.ptr(q),
                                                     _lib.ptr(bad), _lib.current_stream()))
        if bad is not None:
            if int(bad.item()) != 0:
                raise ValueError(ERROR_FIELD_DOMAIN)
            self._field_valid.add(fk)
        f2s = _FieldToSparse(_find_rows(cmap, q), cmap.size)
        self._field_maps[(fk, sk)] = f2s
        return f2s

    def exists_field_to_sparse(self, field_key, sparse_key):
        return (self._k(field_key), self._k(sparse_key)) in self._field_maps

    def get_field_to_sparse_map(self, field_key, sparse_key):
        """reference: coordinate_map_manager.cpp:260-276 -> (unique_index, inverse_map)."""
        ent = self._field_maps.get((self._k(field_key), self._k(sparse_key)))
        _assert(ent is not None, "Field To Sparse Map doesn't exist")
        return ent.first_points(), ent.inverse

    def field_to_sparse_keys(self, field_key):
        fk = self._k(field_key)
        return [CoordinateMapKey(list(sk[0]), sk[1]) for f, sk in self._field_maps if f == fk]

    def _interp_map(self, key, query):
        """Dense interpolation map of float32 query points into map `key` (meb200_interp_map) ->
        (rows int32 [n, 2^D], weights fp32 [n, 2^D])."""
        cmap = self._get(key)
        _assert(query.dim() == 2 and query.size(1) == cmap.ncols, "query coordinates",
                tuple(query.shape), "do not have", cmap.ncols, "columns")
        n, ncols = query.shape
        K = 1 << (ncols - 1)
        rows = torch.empty((n, K), dtype=torch.int32, device=query.device)
        w = torch.empty((n, K), dtype=torch.float32, device=query.device)
        _lib.check(_lib.load().meb200_interp_map(
            _lib.ptr(query), n, ncols, _c_ints(cmap.tensor_stride), _lib.ptr(cmap.coords),
            _lib.ptr(cmap.table), cmap.capacity, _lib.ptr(rows), _lib.ptr(w), _lib.current_stream()))
        return rows, w

    def splat_insert_and_map(self, field_key):
        """reference: TensorField.splat (MinkowskiTensorField.py:53-73, 381-406).  The 2^D corners
        floor(x) + {0,1}^D of every point (meb200_splat_coords; the batch column floored, never
        offset), inserted point-major at tensor stride 1 as insert_and_map inserts, so rows are
        numbered by first occurrence and a corner of weight 0 is a voxel too -> map key."""
        _, field = self._field(field_key)
        n, ncols = field.shape
        dev = field.device
        corners = torch.empty((n << (ncols - 1), ncols), dtype=torch.int32, device=dev)
        bad = torch.empty(1, dtype=torch.int32, device=dev)
        _lib.check(_lib.load().meb200_splat_coords(_lib.ptr(field), n, ncols, _lib.ptr(corners),
                                                   _lib.ptr(bad), _lib.current_stream()))
        status = int(bad.item())
        if status & 1:
            raise ValueError(ERROR_FIELD_DOMAIN)
        if status & 2:
            raise ValueError("splat needs integer batch indices in the first coordinate column")
        key, _ = self.insert_and_map(corners, [1] * (ncols - 1), "")
        return key

    def interpolation_map_weight(self, key, query):
        """reference: coordinate_map_manager.cpp:1080 -> [in rows int32, out rows int32, weights fp32]
        of every present corner, ordered by query row, then corner."""
        rows, w = self._interp_map(key, query.float().contiguous())
        hit = rows >= 0
        q = torch.nonzero(hit)[:, 0].int()
        return [rows[hit], q, w[hit]]

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


class _OriginGrouping:
    """The rows of one coordinate map grouped by cloud (meb200_origin_group): segment s = the rows
    of origin row s, i.e. of the s-th smallest batch index."""

    __slots__ = ("n", "B", "row_seg", "order", "seg_start", "tile_start", "_counts")

    def counts(self):
        """fp32 [B] rows per cloud (device; exact up to 2^24 rows)."""
        if getattr(self, "_counts", None) is None:
            self._counts = (self.seg_start[1:] - self.seg_start[:-1]).float()
        return self._counts


class _FieldToSparse:
    """How the points of a tensor field fall into the M rows of a coordinate map: inverse int64 [N]
    (row of every point, -1 where the map lacks it) and, for a map made by quantising the field,
    unique_index int64 [M] (first point of every row).  The grouping of the points by row
    (meb200_group_by_row: start int32 [M+1], perm int32 [N]) is built on first use and cached."""

    __slots__ = ("inverse", "M", "unique_index", "_group")

    def __init__(self, inverse, M, unique_index=None):
        self.inverse, self.M, self.unique_index, self._group = inverse, int(M), unique_index, None

    def group(self):
        if self._group is None:
            self._group = group_by_row(self.inverse.int(), self.M)
        return self._group

    def first_points(self):
        if self.unique_index is None:
            start, perm = self.group()
            cnt = start[1:] - start[:-1]
            first = perm[start[:-1].clamp(max=max(perm.numel() - 1, 0)).long()].long() \
                if perm.numel() else torch.zeros(self.M, dtype=torch.int64, device=start.device)
            self.unique_index = torch.where(cnt > 0, first, torch.full_like(first, -1))
        return self.unique_index


class _UnionMap:
    """The union of N coordinate maps: `key` (M rows); u[i] int64 [n_i] = union row of every row of
    input i; src int32 [N, M] = row of input i holding union row u, or -1."""

    __slots__ = ("key", "M", "sizes", "u", "src")


# ----------------------------------------------------------------------------------------
def _check_feats(in_feat, manager, in_key, name="in_feat", is_field=False):
    """`is_field`: `in_key` names a tensor field (its rows are the field's points), not a map."""
    _assert(in_feat.is_cuda, f"{name} must be CUDA (this backend has no CPU path)")
    _assert(in_feat.is_contiguous(), f"{name} must be contiguous")
    _assert(in_feat.dim() == 2, f"{name}.dim():", in_feat.dim())
    if is_field:
        n = manager.get_coordinate_field(in_key).size(0)
    else:
        _assert(manager.exists(in_key), ERROR_MAP_NOT_FOUND)
        n = manager.size(in_key)
    _assert(in_feat.size(0) == n, "Invalid in_feat size", in_feat.size(0), "!=", n)


def _workspace(n_out, c_in, c_out, K, code, device):
    """Room for the row-split partial sums of a wgrad (added in a fixed order: deterministic)."""
    nbytes = int(_lib.load().meb200_conv_workspace_bytes(n_out, c_in, c_out, K, code))
    if nbytes == 0:
        return None, 0
    return torch.empty(nbytes, dtype=torch.uint8, device=device), nbytes


# ---- live per-kernel timing for bench.py's roofline (CUDA events on the launch stream) ------
_PROFILE = None   # None, or {"conv_fwd_dgrad": [...], "conv_wgrad": [...], "conv_wgrad_fp8": [...],
#                   "kernel_map": [...]}


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
    _PROFILE = {"conv_fwd_dgrad": [], "conv_wgrad": [], "conv_wgrad_fp8": [], "kernel_map": []}
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


def _conv_forward(in_feat, kernel, km, out_dtype=None, epilogue=None, fp8=False, act=None,
                  shadow=None):
    if _PROFILE is not None:
        esz = in_feat.element_size()
        K, c_in, c_out = kernel.shape
        P = km.n_pairs
        nbytes = km.n_in * c_in * esz + km.n_out * c_out * esz + K * c_in * c_out * esz + P * 8
        return _record("conv_fwd_dgrad",
                       lambda: _conv_forward_impl(in_feat, kernel, km, out_dtype, epilogue, fp8,
                                                  act, shadow),
                       2.0 * P * c_in * c_out, nbytes)
    return _conv_forward_impl(in_feat, kernel, km, out_dtype, epilogue, fp8, act, shadow)


# ---- packed weights: one cast + transpose per optimizer step, not per call -------------------
# An "operand" is what the convolution kernels multiply: a feature dtype, or TF32 (fp32 features,
# tf32 tensor-core math, fp32 packed weights rounded to tf32).
TF32 = "tf32"
_PACKED = {}   # id(kernel tensor) -> (weakref, version, data_ptr, operand, (w_cast, w_t))
_ERR_UNSUPPORTED = -3


class _PackJob(ctypes.Structure):      # == meb200_pack_job (include/meb200.h)
    _fields_ = [("w", ctypes.c_void_p), ("w_cast", ctypes.c_void_p), ("w_t", ctypes.c_void_p),
                ("K", ctypes.c_uint32), ("c_in", ctypes.c_uint32), ("c_out", ctypes.c_uint32),
                ("tile_begin", ctypes.c_uint32)]


def _operand(feat_dtype):
    """The operand of a convolution over `feat_dtype` features: TF32 for fp32 features while torch
    lets fp32 matmuls use TF32, else the dtype itself.  Read at every call, as torch reads its own
    flag at every matmul.  Only `fp32_precision` is read: it is right after every setter style,
    while `allow_tf32` and `get_float32_matmul_precision()` raise once the newer API was used."""
    if feat_dtype == torch.float32 and torch.backends.cuda.matmul.fp32_precision == "tf32":
        return TF32
    return feat_dtype


def _operand_storage(op):
    """torch dtype of an operand's packed weights."""
    return torch.float32 if op == TF32 else op


class _PackTable:
    """Every fp32 convolution kernel of one (device, operand) seen so far, with its packed
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
            jobs.append(_PackJob(ptr, _lib.ptr(w_cast), _lib.ptr(w_t), K, c_in, c_out, tile))
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


_PACK_TABLES = {}      # (device index, operand) -> _PackTable


def _is_master(kernel):
    """An fp32 contiguous master weight: re-packed with every other one by its _PackTable, and the
    only kind of kernel the stem kernels and the pair-list wgrad are used for."""
    return kernel.dtype == torch.float32 and kernel.is_contiguous()


def _cached(key, kernel, dtype):
    ent = _PACKED.get(key)
    if ent is not None and ent[0]() is kernel and ent[1] == kernel._version \
            and ent[2] == kernel.data_ptr() and ent[3] == dtype:
        return ent[4]
    return None


def _purge_packed():
    """Drops the cache entries of dead kernels (discarded networks) once there are many."""
    if len(_PACKED) > 4096:
        for k in [k for k, e in _PACKED.items() if e[0]() is None]:
            del _PACKED[k]


def _packed_weights(kernel, dtype):
    """(w_cast [K,Cin,Cout], w_t [K,Cout,Cin]) of a floating kernel for operand `dtype` (bf16,
    fp16 or TF32: the operand-B layouts of dgrad and forward), rebuilt only when the tensor was
    modified in place (its autograd version counter moved) or replaced.  A kernel that is not an
    fp32 master is packed alone from an fp32 copy: bf16 / fp16 values pass through fp32 exactly, so
    the bytes are kernel.to(dtype).  TF32 weights are fp32 words rounded to tf32."""
    key = id(kernel)
    packed = _cached(key, kernel, dtype)
    if packed is not None:
        return packed
    tbl = None
    if _is_master(kernel):
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
    src = kernel.detach().float().contiguous()
    buf = torch.empty((2, K * c_in * c_out), dtype=_operand_storage(dtype), device=kernel.device)
    w_cast, w_t = buf[0].view(K, c_in, c_out), buf[1].view(K, c_out, c_in)
    _lib.check(lib.meb200_conv_pack_weights(
        _lib.ptr(src), K, c_in, c_out, _lib.dtype_code(dtype), _lib.ptr(w_cast), _lib.ptr(w_t),
        _lib.current_stream()))
    _purge_packed()
    packed = (w_cast, w_t)
    _PACKED[key] = (weakref.ref(kernel), kernel._version, kernel.data_ptr(), dtype, packed)
    if tbl is not None:
        tbl.add(kernel, packed)            # first sight of this kernel: packed alone, batched next time
    return packed


def _feature_weights(kernel, dtype):
    """(w_cast, w_t) for operand `dtype`; exact fp32 reads the kernel itself (no w_t)."""
    if dtype == torch.float32:
        return kernel.float().contiguous(), None
    return _packed_weights(kernel, dtype)


def _is_stem(kernel, feat_dtype):
    """Layers with <= 4 input channels (the stem of a network) on the bf16/fp16 path: run over
    virtual channels (offset, channel) by the stem kernels (include/meb200.h)."""
    if not (kernel.dim() == 3 and kernel.shape[1] <= 4 and _is_master(kernel)):
        return False
    return bool(_lib.load().meb200_conv_stem_supported(_lib.dtype_code(feat_dtype), kernel.shape[0],
                                                       kernel.shape[2]))


def _stem_weights(kernel, dtype):
    """Packed weights of the stem's virtual K = 1 layer, [c_out, V] (cached like _packed_weights)."""
    key = (id(kernel), "stem")
    w_v = _cached(key, kernel, dtype)
    if w_v is not None:
        return w_v
    lib = _lib.load()
    K, c_in, c_out = kernel.shape
    V = int(lib.meb200_conv_stem_virtual_channels(K))
    wv = torch.zeros((V // 4, 4, c_out), dtype=torch.float32, device=kernel.device)
    wv[:K, :c_in] = kernel.detach()
    buf = torch.empty((2, V * c_out), dtype=dtype, device=kernel.device)
    _lib.check(lib.meb200_conv_pack_weights(
        _lib.ptr(wv), 1, V, c_out, _lib.dtype_code(dtype), _lib.ptr(buf[0]), _lib.ptr(buf[1]),
        _lib.current_stream()))
    w_v = buf[1].view(c_out, V)
    _purge_packed()
    _PACKED[key] = (weakref.ref(kernel), kernel._version, kernel.data_ptr(), dtype, w_v)
    return w_v


class _ConvEpilogue(ctypes.Structure):      # == meb200_conv_epilogue (include/meb200.h)
    _fields_ = [("scale", ctypes.c_void_p), ("shift", ctypes.c_void_p),
                ("residual", ctypes.c_void_p), ("relu", ctypes.c_int32)]


def _epilogue_struct(epilogue, out):
    """The native epilogue of `epilogue` = (scale, shift, residual or None, relu) for the output
    `out` (None -> None): fp32 [c_out] scale and shift, a residual shaped and typed as `out`."""
    if epilogue is None:
        return None
    scale, shift, residual, relu = epilogue
    c_out = out.shape[1]
    for t in (scale, shift):
        _assert(t.dtype == torch.float32 and t.is_contiguous() and t.shape == (c_out,)
                and t.device == out.device, "epilogue scale / shift must be fp32 [c_out] on",
                out.device)
    if residual is not None:
        _assert(residual.shape == out.shape and residual.dtype == out.dtype
                and residual.is_contiguous() and residual.device == out.device,
                "epilogue residual must be a contiguous", out.dtype, "tensor of shape",
                tuple(out.shape))
    return _ConvEpilogue(_lib.ptr(scale), _lib.ptr(shift), _lib.ptr(residual), 1 if relu else 0)


# ---- fp8 inference (DESIGN.md §3, §7) -----------------------------------------------------------
# Inside fp8_inference(), the convolution layers that need no gradient and whose shape is on the
# e4m3 grid run their forward on e4m3 operands: the features quantised per tensor, the weights per
# output channel, the products summed by the tensor cores (not in fp32: DESIGN.md §3), the scales
# folded into the epilogue.  Like torch's TF32 flag it is a choice of number format, read at every
# call; like torch.no_grad it holds for the thread that entered it.
FP8 = "e4m3"
# .depth: fp8_inference() blocks the thread is inside; .calibs: their calibrations (None: dynamic),
# innermost last; .observing: the Fp8Calibration whose observe() block the thread is inside
_FP8_STATE = threading.local()
_FP8_DTYPES = (torch.float32, torch.bfloat16, torch.float16)
_QUANT_WS = {}      # (device index, stream) -> zero-filled quantisation workspace


@contextlib.contextmanager
def fp8_inference(calibration=None):
    """Within the block, eval-mode sparse convolutions run on the Hopper e4m3 tensor cores where
    they can (no gradient needed, c_in a multiple of 32, c_out a multiple of 16); everything else
    runs as it does outside the block.  Results change: e4m3 keeps 3 mantissa bits.  Thread-local:
    other threads keep their own setting.

    calibration (an Fp8Calibration, DESIGN.md §3): the layers it calibrated quantise their input
    with their static scale, and the layers that feed one of them also write an e4m3 copy of their
    output for it (its shadow) in the same launch.  Other layers keep the per-tensor scale of their
    input's amax.  In nested blocks the innermost calibration holds."""
    if fp8_observer() is not None:
        raise RuntimeError("fp8_inference() inside Fp8Calibration.observe(): calibration observes "
                           "the layers as they run outside fp8")
    calibs = _FP8_STATE.__dict__.setdefault("calibs", [])
    _FP8_STATE.depth = getattr(_FP8_STATE, "depth", 0) + 1
    calibs.append(calibration)
    try:
        yield
    finally:
        calibs.pop()
        _FP8_STATE.depth -= 1


def fp8_enabled():
    return getattr(_FP8_STATE, "depth", 0) > 0


def fp8_calibration():
    """The calibration of the innermost fp8_inference() block of this thread (None: dynamic)."""
    calibs = getattr(_FP8_STATE, "calibs", None)
    return calibs[-1] if calibs else None


def fp8_observer():
    """The Fp8Calibration observing in this thread, or None."""
    return getattr(_FP8_STATE, "observing", None)


def fp8_supported(c_in, c_out):
    """Whether the e4m3 forward takes a layer of c_in -> c_out channels."""
    return bool(_lib.load().meb200_conv_fp8_supported(c_in, c_out))


def _fp8_weights(kernel):
    """(w_t e4m3 [K, Cout, Cin] as uint8, w_scale fp32 [Cout]) of a kernel, cached with the other
    packed operands and rebuilt only when the tensor was modified in place or replaced."""
    key = (id(kernel), FP8)
    packed = _cached(key, kernel, FP8)
    if packed is not None:
        return packed
    K, c_in, c_out = kernel.shape
    src = kernel.detach().float().contiguous()
    w_t = torch.empty((K, c_out, c_in), dtype=torch.uint8, device=kernel.device)
    w_scale = torch.empty(c_out, dtype=torch.float32, device=kernel.device)
    _lib.check(_lib.load().meb200_conv_pack_weights_e4m3(
        _lib.ptr(src), K, c_in, c_out, _lib.ptr(w_t), _lib.ptr(w_scale), _lib.current_stream()))
    packed = (w_t, w_scale)
    _purge_packed()
    _PACKED[key] = (weakref.ref(kernel), kernel._version, kernel.data_ptr(), FP8, packed)
    return packed


def _quantize_e4m3(feat):
    """(e4m3 bytes [n, c] as uint8, fp32 [2] = (scale, inv) on the device) of contiguous features."""
    return _quantize_dynamic(feat, "meb200_quantize_e4m3")


def _quantize_dynamic(feat, entry):
    """(fp8 bytes [n, c] as uint8, fp32 [2] = (scale, inv) on the device) of contiguous features,
    by `entry`, meb200_quantize_e4m3 or meb200_quantize_e5m2 (the two share the workspace)."""
    lib = _lib.load()
    stream = _lib.current_stream()
    wkey = (feat.device.index, stream)
    ws = _QUANT_WS.get(wkey)
    if ws is None:
        ws = _QUANT_WS[wkey] = torch.zeros(int(lib.meb200_quantize_e4m3_workspace_bytes()),
                                           dtype=torch.uint8, device=feat.device)
    n, c = feat.shape
    q = torch.empty((n, c), dtype=torch.uint8, device=feat.device)
    if n * c == 0:                    # nothing to convert: amax 0, scale = inv = 1
        return q, torch.ones(2, dtype=torch.float32, device=feat.device)
    scale = torch.empty(2, dtype=torch.float32, device=feat.device)
    _lib.check(getattr(lib, entry)(_lib.ptr(feat), _lib.dtype_code(feat.dtype), n, c,
                                   _lib.ptr(q), _lib.ptr(scale), _lib.ptr(ws), stream))
    return q, scale


def amax_accumulate(feat, amax):
    """amax (fp32 [1] on the device) = max(amax, max |feat| over the finite values): one launch,
    no host read (meb200_amax_accumulate)."""
    n, c = feat.shape
    _lib.check(_lib.load().meb200_amax_accumulate(_lib.ptr(feat), _lib.dtype_code(feat.dtype), n, c,
                                                  _lib.ptr(amax), _lib.current_stream()))


def e4m3_scales(amax):
    """fp32 [2] = (scale, inv) on the device of an amax on the device (meb200_e4m3_scales)."""
    scale = torch.empty(2, dtype=torch.float32, device=amax.device)
    _lib.check(_lib.load().meb200_e4m3_scales(_lib.ptr(amax), _lib.ptr(scale),
                                              _lib.current_stream()))
    return scale


def quantize_e4m3_static(feat, scale):
    """e4m3 bytes [n, c] as uint8 of contiguous features at a given scale (fp32 [2] on the device):
    the conversion launch alone (meb200_quantize_e4m3_static)."""
    n, c = feat.shape
    q = torch.empty((n, c), dtype=torch.uint8, device=feat.device)
    _lib.check(_lib.load().meb200_quantize_e4m3_static(
        _lib.ptr(feat), _lib.dtype_code(feat.dtype), n, c, _lib.ptr(q), _lib.ptr(scale),
        _lib.current_stream()))
    return q


def _conv_forward_fp8(in_feat, kernel, km, epilogue, act=None, shadow=None):
    """The e4m3 forward (meb200_conv_forward_fp8): the output in the feature dtype, the epilogue's
    scale multiplied by the weight scale on the device (no scale: the weight scale alone, no shift:
    zero).  act: the input already quantised, (e4m3 bytes, fp32 [2] scale), or None: quantised here
    at its amax.  shadow: as _conv_forward_impl."""
    lib = _lib.load()
    K, c_in, c_out = kernel.shape
    _assert(K == km.K, "kernel volume", K, "does not match the kernel map", km.K)
    out = torch.empty((km.n_out, c_out), dtype=in_feat.dtype, device=in_feat.device)
    scale, shift, residual, relu = epilogue if epilogue is not None else (None, None, None, False)
    w_t, w_scale = _fp8_weights(kernel)
    scale = w_scale if scale is None else w_scale * scale
    if shift is None:
        shift = torch.zeros(c_out, dtype=torch.float32, device=in_feat.device)
    epi = _epilogue_struct((scale, shift, residual, relu), out)
    q, a_scale = act if act is not None else _quantize_e4m3(in_feat)
    args = (_lib.ptr(q), _lib.ptr(a_scale), km.n_in, c_in, _lib.ptr(w_t), K, c_out,
            _lib.ptr(km.out_nbr), km.n_out, _lib.ptr(out), _lib.dtype_code(out.dtype),
            _lib.ptr(km.out_order), ctypes.addressof(epi))
    if shadow is None:
        _lib.check(lib.meb200_conv_forward_fp8(*args, _lib.current_stream()))
        return out
    q_out = torch.empty((km.n_out, c_out), dtype=torch.uint8, device=in_feat.device)
    _lib.check(lib.meb200_conv_forward_fp8_q(*args, _lib.ptr(q_out), _lib.ptr(shadow),
                                             _lib.current_stream()))
    return out, q_out


# ---- fp8 training (DESIGN.md §3, "fp8 training") -----------------------------------------------
# Inside fp8_training(), the convolution layers that need a gradient and whose shape is on the e4m3
# grid both ways run their forward on e4m3 operands (as fp8 inference does, without an epilogue)
# and their input gradient on e5m2 gradients against e4m3 weights scaled per input channel.  The
# weight gradient keeps the route of the feature dtype.  fp8_inference() only selects layers that
# need no gradient and fp8_training() only layers that need one: the two never meet.
FP8_DGRAD = "e4m3_dgrad"      # the packed-weight cache's operand of the dgrad's e4m3 weights


@contextlib.contextmanager
def fp8_training(*, weight_gradient=False, scaling=None):
    """Within the block, training sparse convolutions run their forward and input gradient on the
    Hopper fp8 tensor cores where they can (a gradient needed, c_in and c_out multiples of 32 up to
    1024, not a K = 1 stride-1 matrix product): the forward on e4m3 features and weights, the input
    gradient on the output gradient in e5m2 against e4m3 weights.  The weight gradient and every
    other layer run as they do outside the block.  Thread-local, and nestable with fp8_inference()
    either way.

    weight_gradient=True: the selected layers also run their weight gradient on fp8, the e4m3 input
    of the forward times the e5m2 output gradient of the input gradient (layers with over 1023
    kernel offsets keep the weight gradient of the feature dtype).  Forward outputs and input
    gradients are those of weight_gradient=False, bit for bit.  Nested blocks: the innermost
    decides.

    scaling (an Fp8DelayedScaling, DESIGN.md §3 "delayed scaling"): the selected layers of the
    model it is bound to quantise at the scales of its amax histories instead of their tensors'
    own amax, and the training batch norms that feed them write their fp8 operands.  Each entry
    into an outermost block with a given recipe is one step of it.  None: dynamic scales."""
    modes = _FP8_STATE.__dict__.setdefault("train_modes", [])
    if scaling is not None and all(m[1] is not scaling for m in modes):
        scaling._begin_step()
    modes.append((bool(weight_gradient), scaling))
    try:
        yield
    finally:
        modes.pop()


def fp8_training_enabled():
    return bool(getattr(_FP8_STATE, "train_modes", None))


def fp8_training_weight_gradient():
    """Whether the innermost fp8_training() block of this thread runs weight gradients on fp8."""
    modes = getattr(_FP8_STATE, "train_modes", None)
    return bool(modes) and modes[-1][0]


def fp8_training_scaling():
    """The Fp8DelayedScaling of the innermost fp8_training() block of this thread, or None."""
    modes = getattr(_FP8_STATE, "train_modes", None)
    return modes[-1][1] if modes else None


class _Fp8Out(ctypes.Structure):      # == meb200_fp8_out (include/meb200.h)
    _fields_ = [("q", ctypes.c_void_p), ("scale", ctypes.c_void_p), ("amax_slot", ctypes.c_void_p)]


def fp8_out(q, scale, slot):
    """The meb200_fp8_out of bytes `q`, a DEVICE fp32 [2] (scale, inv) and an fp32 [1] amax slot."""
    return _Fp8Out(_lib.ptr(q), _lib.ptr(scale), _lib.ptr(slot))


def quantize_fp8_record(feat, fmt, scale, slot):
    """fp8 bytes [n, c] as uint8 of contiguous features in `fmt` (_lib.FP8_E4M3 / FP8_E5M2) at a
    given scale (fp32 [2] on the device), max |feat| over the finite values maxed into `slot` (fp32
    [1] on the device): one launch, no host read (meb200_quantize_fp8_record)."""
    n, c = feat.shape
    q = torch.empty((n, c), dtype=torch.uint8, device=feat.device)
    fq = fp8_out(q, scale, slot)
    _lib.check(_lib.load().meb200_quantize_fp8_record(
        _lib.ptr(feat), _lib.dtype_code(feat.dtype), n, c, fmt, ctypes.byref(fq),
        _lib.current_stream()))
    return q


def fp8_roll(cur, hist, n_e4m3, n_e5m2, margin):
    """The step boundary of delayed scaling (meb200_fp8_roll): the slots `cur` [L] pushed into the
    histories `hist` [L, H] in place; returns (the next step's zeroed slots [L], scales [L, 2]), the
    first n_e4m3 entries in e4m3 and the rest in e5m2.  One launch, no host read."""
    L, H = hist.shape
    nxt = torch.empty(L, dtype=torch.float32, device=hist.device)
    scales = torch.empty((L, 2), dtype=torch.float32, device=hist.device)
    _lib.check(_lib.load().meb200_fp8_roll(_lib.ptr(cur), _lib.ptr(hist), n_e4m3, n_e5m2, H,
                                           int(margin), _lib.ptr(nxt), _lib.ptr(scales),
                                           _lib.current_stream()))
    return nxt, scales


def fp8_wgrad_supported(c_in, c_out, K):
    """Whether the fp8 weight gradient (meb200_conv_wgrad_fp8) takes a layer of this shape."""
    return bool(_lib.load().meb200_conv_wgrad_fp8_supported(c_in, c_out, K))


def _fp8_dgrad_weights(kernel):
    """(w_c e4m3 [K, Cin, Cout] as uint8, w_scale fp32 [Cin]) of a kernel, the dgrad's operand B with
    one scale per input channel, cached with the other packed operands and rebuilt only when the
    tensor was modified in place or replaced."""
    key = (id(kernel), FP8_DGRAD)
    packed = _cached(key, kernel, FP8_DGRAD)
    if packed is not None:
        return packed
    K, c_in, c_out = kernel.shape
    src = kernel.detach().float().contiguous()
    w_c = torch.empty((K, c_in, c_out), dtype=torch.uint8, device=kernel.device)
    w_scale = torch.empty(c_in, dtype=torch.float32, device=kernel.device)
    _lib.check(_lib.load().meb200_conv_pack_weights_e4m3_dgrad(
        _lib.ptr(src), K, c_in, c_out, _lib.ptr(w_c), _lib.ptr(w_scale), _lib.current_stream()))
    packed = (w_c, w_scale)
    _purge_packed()
    _PACKED[key] = (weakref.ref(kernel), kernel._version, kernel.data_ptr(), FP8_DGRAD, packed)
    return packed


def _conv_dgrad_fp8(grad_out, kernel, km, dtype, grad_q=None):
    """The input gradient in `dtype` on the fp8 tensor cores (meb200_conv_dgrad_fp8): grad_out (in
    `dtype`, contiguous) quantised to e5m2 at its amax, the weights from _fp8_dgrad_weights.
    grad_q: grad_out already quantised, (e5m2 bytes, fp32 [2] scale), or None: quantised here."""
    K, c_in, c_out = kernel.shape
    _assert(K == km.K, "kernel volume", K, "does not match the kernel map", km.K)
    if km.n_out == 0 or km.n_in == 0:      # no output rows: no neighbour contributes
        return torch.zeros((km.n_in, c_in), dtype=dtype, device=grad_out.device)
    grad_in = torch.empty((km.n_in, c_in), dtype=dtype, device=grad_out.device)
    w_c, w_scale = _fp8_dgrad_weights(kernel)
    q, g_scale = grad_q if grad_q is not None else _quantize_dynamic(grad_out, "meb200_quantize_e5m2")
    _lib.check(_lib.load().meb200_conv_dgrad_fp8(
        _lib.ptr(q), _lib.ptr(g_scale), km.n_out, c_out, _lib.ptr(w_c), _lib.ptr(w_scale), K, c_in,
        _lib.ptr(km.in_nbr), km.n_in, _lib.ptr(grad_in), _lib.dtype_code(dtype),
        _lib.ptr(km.in_order), _lib.current_stream()))
    return grad_in


def _conv_wgrad_fp8(act, grad_q, kernel, km):
    """The weight gradient on the fp8 tensor cores (meb200_conv_wgrad_fp8), in the kernel's dtype:
    act = (e4m3 bytes [n_in, c_in], fp32 [2] scale) the forward multiplied, grad_q = (e5m2 bytes
    [n_out, c_out], fp32 [2] scale) the dgrad multiplied, over the map's pair lists.  An empty map
    gives zero without a launch."""
    K, c_in, c_out = kernel.shape
    _assert(K == km.K, "kernel volume", K, "does not match the kernel map", km.K)
    if km.n_out == 0 or km.n_in == 0:
        return torch.zeros((K, c_in, c_out), dtype=kernel.dtype, device=kernel.device)
    lib = _lib.load()
    q, a_scale = act
    g, g_scale = grad_q
    grad_w = torch.empty((K, c_in, c_out), dtype=torch.float32, device=kernel.device)
    pin, pout, seg, nch = km.pair_lists()
    nbytes = int(lib.meb200_conv_wgrad_fp8_workspace_bytes(km.n_out, c_in, c_out, K))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=kernel.device) if nbytes else None
    _lib.check(lib.meb200_conv_wgrad_fp8(
        _lib.ptr(q), _lib.ptr(a_scale), _lib.ptr(g), _lib.ptr(g_scale), c_in, K, c_out,
        _lib.ptr(pin), _lib.ptr(pout), _lib.ptr(seg), nch, km.n_out, _lib.ptr(grad_w), _lib.ptr(ws),
        nbytes, _lib.current_stream()))
    return grad_w if grad_w.dtype == kernel.dtype else grad_w.to(kernel.dtype)


def _conv_backward_fp8w(act, dtype, grad_out, kernel, km, need_in=True, need_w=True, grad_q=None):
    """(grad_in or None, grad_w or None) of a layer run in fp8_training(weight_gradient=True), from
    act = (e4m3 bytes, scale) of its forward and its feature dtype: grad_out quantised to e5m2 once,
    for the input gradient (_conv_dgrad_fp8, as in fp8_training()) and the weight gradient
    (_conv_wgrad_fp8).  grad_q: grad_out already quantised (delayed scaling), or None."""
    if grad_out.dtype != dtype:
        grad_out = grad_out.to(dtype)
    grad_out = grad_out.contiguous()
    if grad_q is None and km.n_out > 0 and km.n_in > 0:
        grad_q = _quantize_dynamic(grad_out, "meb200_quantize_e5m2")
    if _PROFILE is None:
        return (_conv_dgrad_fp8(grad_out, kernel, km, dtype, grad_q) if need_in else None,
                _conv_wgrad_fp8(act, grad_q, kernel, km) if need_w else None)
    K, c_in, c_out = kernel.shape
    P = km.n_pairs
    flops = 2.0 * P * c_in * c_out
    gi = gw = None
    esz = torch.empty((), dtype=dtype).element_size()
    if need_in:
        nb = km.n_out * c_out * esz + km.n_in * c_in * esz + K * c_in * c_out * esz + P * 8
        gi = _record("conv_fwd_dgrad", lambda: _conv_dgrad_fp8(grad_out, kernel, km, dtype, grad_q),
                     flops, nb)
    if need_w:    # e4m3 in and e5m2 dOut, dW (fp32) out, pairs
        nb = km.n_in * c_in + km.n_out * c_out + K * c_in * c_out * 4 + P * 8
        gw = _record("conv_wgrad_fp8", lambda: _conv_wgrad_fp8(act, grad_q, kernel, km), flops, nb)
    return gi, gw


def _pad4(feat):
    c = feat.shape[1]
    return feat.contiguous() if c == 4 else torch.nn.functional.pad(feat, (0, 4 - c))


def _conv_forward_impl(in_feat, kernel, km, out_dtype=None, epilogue=None, fp8=False, act=None,
                       shadow=None):
    """out = in_feat * kernel over km; `epilogue` (scale, shift, residual or None, relu), or None:
    out = relu?(acc * scale + shift [+ residual]) from the fp32 accumulator, in the same launch.
    fp8: on e4m3 operands (_conv_forward_fp8 with `act`; the caller has checked fp8_supported).
    shadow (fp32 [2] static scale on the device, with an epilogue): returns (out, q), q the e4m3
    copy of out at that scale written by the same launch (the _q entries of include/meb200.h), or
    None where the route writes none (TF32, small-cin and SIMT kernels)."""
    if fp8:
        return _conv_forward_fp8(in_feat, kernel, km, epilogue, act, shadow)
    _assert(shadow is None or epilogue is not None, "a shadow is written by the epilogue")
    lib = _lib.load()
    op = _operand(in_feat.dtype)
    code = _lib.dtype_code(op)
    K, c_in, c_out = kernel.shape
    _assert(K == km.K, "kernel volume", K, "does not match the kernel map", km.K)
    out = torch.empty((km.n_out, c_out), dtype=out_dtype or in_feat.dtype, device=in_feat.device)
    epi = _epilogue_struct(epilogue, out)
    epi_ptr = None if epi is None else ctypes.addressof(epi)
    q = None
    if shadow is not None:
        q = torch.empty((km.n_out, c_out), dtype=torch.uint8, device=in_feat.device)
    done = lambda: out if shadow is None else (out, q)          # noqa: E731
    if _is_stem(kernel, in_feat.dtype):
        # (named, so that they outlive the argument list: a temporary freed before the call can
        # be handed by the allocator to the next temporary and overwritten before the kernel runs)
        in4, w_v = _pad4(in_feat), _stem_weights(kernel, in_feat.dtype)
        args = (_lib.ptr(in4), code, K, _lib.ptr(w_v), c_out, _lib.ptr(km.out_nbr), km.n_out,
                _lib.ptr(out), _lib.dtype_code(out.dtype), epi_ptr)
        if shadow is None:
            rc = lib.meb200_conv_stem_forward(*args, _lib.current_stream())
        else:
            rc = lib.meb200_conv_stem_forward_q(*args, _lib.ptr(q), _lib.ptr(shadow),
                                                _lib.current_stream())
        if rc != _ERR_UNSUPPORTED:
            _lib.check(rc)
            return done()
    w_cast, w_t = _feature_weights(kernel, op)
    args = (_lib.ptr(in_feat), code, km.n_in, c_in, _lib.ptr(w_cast), _lib.ptr(w_t), K, c_out,
            _lib.ptr(km.out_nbr), km.n_out, _lib.ptr(out), _lib.dtype_code(out.dtype),
            _lib.ptr(km.out_order), epi_ptr)
    if shadow is not None and op in (torch.bfloat16, torch.float16):
        rc = lib.meb200_conv_forward_q(*args, _lib.ptr(q), _lib.ptr(shadow), _lib.current_stream())
        if rc != _ERR_UNSUPPORTED:
            _lib.check(rc)
            return done()
    q = None                               # a route without shadows: the next layer quantises
    _lib.check(lib.meb200_conv_forward(*args, _lib.current_stream()))
    return done()


def _grad_q(grad_q):
    """The keyword of an output gradient quantised beforehand (delayed scaling), or none: without
    one the backward calls keep the arguments they have under fp8_training()."""
    return {} if grad_q is None else {"grad_q": grad_q}


def _conv_backward(in_feat, grad_out, kernel, km, need_in=True, need_w=True, fp8=False,
                   grad_q=None):
    if _PROFILE is not None:
        esz = in_feat.element_size()
        K, c_in, c_out = kernel.shape
        P = km.n_pairs
        flops = 2.0 * P * c_in * c_out
        gi = gw = None
        if need_in:   # dgrad alone: dOut in, dIn out, W, table
            nb = km.n_out * c_out * esz + km.n_in * c_in * esz + K * c_in * c_out * esz + P * 8
            gi, _ = _record("conv_fwd_dgrad", lambda: _conv_backward_impl(
                in_feat, grad_out, kernel, km, True, False, fp8, **_grad_q(grad_q)), flops, nb)
        if need_w:    # wgrad alone: In and dOut in, dW (fp32) out, table
            nb = km.n_in * c_in * esz + km.n_out * c_out * esz + K * c_in * c_out * 4 + P * 8
            _, gw = _record("conv_wgrad", lambda: _conv_backward_impl(
                in_feat, grad_out, kernel, km, False, True), flops, nb)
        return gi, gw
    return _conv_backward_impl(in_feat, grad_out, kernel, km, need_in, need_w, fp8,
                               **_grad_q(grad_q))


def _conv_backward_impl(in_feat, grad_out, kernel, km, need_in=True, need_w=True, fp8=False,
                        grad_q=None):
    """(grad_in or None, grad_w or None).  fp8 (the caller has checked the grid both ways): the
    input gradient on e5m2 x e4m3 (_conv_dgrad_fp8, with grad_q when given); the weight gradient as
    without it."""
    lib = _lib.load()
    op = _operand(in_feat.dtype)
    code = _lib.dtype_code(op)
    if grad_out.dtype != in_feat.dtype:
        grad_out = grad_out.to(in_feat.dtype)
    grad_out = grad_out.contiguous()
    if fp8 and need_in:
        grad_in = _conv_dgrad_fp8(grad_out, kernel, km, in_feat.dtype, **_grad_q(grad_q))
        if not need_w:
            return grad_in, None
        return grad_in, _conv_backward_impl(in_feat, grad_out, kernel, km, False, True)[1]
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
        ws, ws_bytes = _workspace(n_out, V, c_out, 1, code, in_feat.device)
        rc = lib.meb200_conv_stem_wgrad(
            _lib.ptr(in4), _lib.ptr(grad_out), code, K, c_out, _lib.ptr(km.out_nbr),
            n_out, _lib.ptr(gwv), _lib.ptr(ws), ws_bytes, _lib.current_stream())
        if rc != _ERR_UNSUPPORTED:
            _lib.check(rc)
            return None, gwv[:K, :c_in].contiguous()
    w_cast = _feature_weights(kernel, op)[0] if need_in else None    # the wgrad reads no weights
    pin = pout = seg = None
    nch = 0
    ws, ws_bytes = None, 0
    if need_w:
        # a kernel that is not an fp32 master keeps the dense-table wgrad: the two reduce in
        # different orders, so switching would change its bits
        if _is_master(kernel) and lib.meb200_conv_wgrad_uses_pairs(code, c_in, c_out, K):
            pin, pout, seg, nch = km.pair_lists()
        ws, ws_bytes = _workspace(n_out, c_in, c_out, K, code, in_feat.device)
    _lib.check(lib.meb200_conv_backward(
        _lib.ptr(in_feat), _lib.ptr(grad_out), code, n_in, c_in, _lib.ptr(w_cast), K, c_out,
        _lib.ptr(km.out_nbr), _lib.ptr(km.in_nbr) if need_in else None, n_out, _lib.ptr(grad_in),
        _lib.dtype_code(in_feat.dtype), _lib.ptr(grad_w), _lib.ptr(pin), _lib.ptr(pout),
        _lib.ptr(seg), nch, _lib.ptr(ws), ws_bytes, _lib.ptr(km.in_order) if need_in else None,
        _lib.current_stream()))
    if grad_w is not None and grad_w.dtype != kernel.dtype:
        grad_w = grad_w.to(kernel.dtype)
    return grad_in, grad_w


def _set_strided_key(manager, in_key, out_key, kernel_stride, region=None):
    """Sets an unset `out_key` to the map at the tensor stride of `in_key` times `kernel_stride`:
    the strided map, or with region = (region_type, kernel_size, dilation, offset) the map of the
    regions around the input rows (expand_coordinates)."""
    if out_key.is_key_set():
        return
    if region is None:
        ok, _ = manager._stride(in_key, kernel_stride)
    else:
        ik = manager._k(in_key)
        out_ts = [t * int(s) for t, s in zip(ik[0], kernel_stride)]
        ok, _ = manager._stride_region(in_key, *region, ik[0], out_ts, False, True)
    out_key.set_key(list(ok[0]), ok[1])


def _set_transposed_key(manager, in_key, out_key, kernel_stride, region, expand_coordinates):
    """Sets an unset `out_key` to the map at the tensor stride of `in_key` divided by
    `kernel_stride`, made from the regions = (region_type, kernel_size, dilation, offset) around
    the input rows."""
    if out_key.is_key_set():
        return
    ik = manager._k(in_key)
    for t, s in zip(ik[0], kernel_stride):
        _assert(t % int(s) == 0, "Invalid up stride on tensor stride:", list(ik[0]),
                "kernel stride:", list(kernel_stride))
    out_ts = [t // int(s) for t, s in zip(ik[0], kernel_stride)]
    ok, _ = manager._stride_region(in_key, *region, out_ts, out_ts, True, expand_coordinates)
    out_key.set_key(list(ok[0]), ok[1])


def ConvolutionForwardGPU(in_feat, kernel, kernel_size, kernel_stride, kernel_dilation,
                          region_type, offset, expand_coordinates, convolution_mode, in_key,
                          out_key, manager, epilogue=None, fp8=False, act=None, shadow=None):
    """reference: ConvolutionForwardGPU src/convolution_gpu.cu:45-159 (CPU twin
    convolution_cpu.cpp:42-135).  Mutates `out_key` when it is unset.  `epilogue`, `fp8`, `act`,
    `shadow`: as _conv_forward_impl (no autograd: for callers that need no gradient)."""
    _assert(kernel.dim() == 3, "kernel.dim():", kernel.dim())
    _assert(kernel.is_cuda, "kernel must be CUDA")
    _check_feats(in_feat, manager, in_key)
    _assert(in_feat.size(1) == kernel.size(1), "Input feature size and kernel size mismatch")
    _set_strided_key(manager, in_key, out_key, kernel_stride,
                     (region_type, kernel_size, kernel_dilation, offset) if expand_coordinates
                     else None)
    km = manager._kernel_map(in_key, out_key, kernel_size, kernel_stride, kernel_dilation,
                             region_type, offset, False, False)
    return _conv_forward(in_feat, kernel, km, epilogue=epilogue, fp8=fp8, act=act, shadow=shadow)


def ConvolutionBackwardGPU(in_feat, grad_out_feat, kernel, kernel_size, kernel_stride,
                           kernel_dilation, region_type, offset, convolution_mode, in_key,
                           out_key, manager, need_in=True, need_w=True, fp8=False, act=None,
                           grad_q=None):
    """reference: ConvolutionBackwardGPU src/convolution_gpu.cu:161-244.  fp8: as _conv_backward_impl.
    act: (e4m3 bytes, fp32 [2] scale, feature dtype) of the input of a layer run in
    fp8_training(weight_gradient=True), in place of in_feat (None): both gradients on fp8
    (_conv_backward_fp8w).  grad_q: (e5m2 bytes, fp32 [2] scale) of grad_out_feat (delayed
    scaling), or None: quantised at its amax."""
    _check_feats(in_feat if act is None else act[0], manager, in_key)
    _assert(manager.exists(out_key), ERROR_MAP_NOT_FOUND)
    _assert(grad_out_feat.size(0) == manager.size(out_key), "Invalid grad_out size")
    km = manager._kernel_map(in_key, out_key, kernel_size, kernel_stride, kernel_dilation,
                             region_type, offset, False, False)
    if act is not None:
        return _conv_backward_fp8w(act[:2], act[2], grad_out_feat, kernel, km, need_in, need_w,
                                   **_grad_q(grad_q))
    return _conv_backward(in_feat, grad_out_feat, kernel, km, need_in, need_w, fp8,
                          **_grad_q(grad_q))


def ConvolutionTransposeForwardGPU(in_feat, kernel, kernel_size, kernel_stride,
                                   kernel_dilation, region_type, offset,
                                   generate_new_coordinates, convolution_mode, in_key, out_key,
                                   manager, epilogue=None, fp8=False, act=None, shadow=None):
    """reference: src/convolution_transpose_gpu.cu (CPU twin convolution_transpose_cpu.cpp:42-125).
    `epilogue`, `fp8`, `act`, `shadow`: as ConvolutionForwardGPU."""
    _assert(kernel.dim() == 3, "kernel.dim():", kernel.dim())
    _check_feats(in_feat, manager, in_key)
    _assert(in_feat.size(1) == kernel.size(1), "Input feature size and kernel size mismatch")
    _set_transposed_key(manager, in_key, out_key, kernel_stride,
                        (region_type, kernel_size, kernel_dilation, offset),
                        generate_new_coordinates)
    km = manager._kernel_map(in_key, out_key, kernel_size, kernel_stride, kernel_dilation,
                             region_type, offset, True, False)
    return _conv_forward(in_feat, kernel, km, epilogue=epilogue, fp8=fp8, act=act, shadow=shadow)


def ConvolutionTransposeBackwardGPU(in_feat, grad_out_feat, kernel, kernel_size, kernel_stride,
                                    kernel_dilation, region_type, offset, convolution_mode,
                                    in_key, out_key, manager, need_in=True, need_w=True, fp8=False,
                                    act=None, grad_q=None):
    """`fp8`, `act`, `grad_q`: as ConvolutionBackwardGPU."""
    _check_feats(in_feat if act is None else act[0], manager, in_key)
    _assert(manager.exists(out_key), ERROR_MAP_NOT_FOUND)
    km = manager._kernel_map(in_key, out_key, kernel_size, kernel_stride, kernel_dilation,
                             region_type, offset, True, False)
    if act is not None:
        return _conv_backward_fp8w(act[:2], act[2], grad_out_feat, kernel, km, need_in, need_w,
                                   **_grad_q(grad_q))
    return _conv_backward(in_feat, grad_out_feat, kernel, km, need_in, need_w, fp8,
                          **_grad_q(grad_q))


_POOL_CODE = {PoolingMode.LOCAL_SUM_POOLING: _lib.POOL_SUM,
              PoolingMode.LOCAL_AVG_POOLING: _lib.POOL_AVG,
              PoolingMode.LOCAL_MAX_POOLING: _lib.POOL_MAX}


def LocalPoolingForwardGPU(in_feat, kernel_size, kernel_stride, kernel_dilation, region_type,
                           offset, pooling_mode, in_key, out_key, manager):
    """reference: LocalPoolingForwardGPU src/local_pooling_gpu.cu:46-137 (CPU twin
    local_pooling_cpu.cpp:43-120) -> (out_feat, num_nonzero | max_index)"""
    _check_feats(in_feat, manager, in_key)
    _assert(pooling_mode in _POOL_CODE, "Invalid pooling mode", pooling_mode)
    _set_strided_key(manager, in_key, out_key, kernel_stride)
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
    grad_in = torch.empty_like(in_feat)       # every mode writes every element once
    _lib.check(lib.meb200_pool_backward(
        _lib.ptr(grad_out_feat), _lib.dtype_code(in_feat.dtype), km.n_in, C, _lib.ptr(km.in_nbr),
        km.K, km.n_out, mode, _lib.ptr(num_nonzero) if num_nonzero.numel() else None,
        _lib.ptr(grad_in), _lib.current_stream()))
    return grad_in


def LocalPoolingTransposeForwardGPU(in_feat, kernel_size, kernel_stride, kernel_dilation,
                                    region_type, offset, expand_coordinates, pooling_mode, in_key,
                                    out_key, manager):
    """reference: LocalPoolingTransposeForwardGPU src/local_pooling_transpose_gpu.cu (CPU twin
    local_pooling_transpose_cpu.cpp).  Both reference backends sum, whatever `pooling_mode` says
    (use_avg = false): out[o] = sum_k in[out_nbr[k][o]] over the transposed pooling map; the
    second result (num_nonzero) is empty.  Mutates `out_key` when it is unset."""
    _check_feats(in_feat, manager, in_key)
    _set_transposed_key(manager, in_key, out_key, kernel_stride,
                        (region_type, kernel_size, kernel_dilation, offset), expand_coordinates)
    km = manager._kernel_map(in_key, out_key, kernel_size, kernel_stride, kernel_dilation,
                             region_type, offset, True, True)
    C = in_feat.size(1)
    out = torch.empty((km.n_out, C), dtype=in_feat.dtype, device=in_feat.device)
    _lib.check(_lib.load().meb200_pool_forward(
        _lib.ptr(in_feat), _lib.dtype_code(in_feat.dtype), km.n_in, C, _lib.ptr(km.out_nbr),
        km.K, km.n_out, _lib.POOL_SUM, _lib.ptr(out), None, _lib.current_stream()))
    return out, torch.empty(0, dtype=in_feat.dtype, device=in_feat.device)


def LocalPoolingTransposeBackwardGPU(in_feat, grad_out_feat, num_nonzero, kernel_size,
                                     kernel_stride, kernel_dilation, region_type, offset,
                                     pooling_mode, in_key, out_key, manager):
    """reference: LocalPoolingTransposeBackwardGPU src/local_pooling_transpose_gpu.cu: the sum's
    adjoint, grad_in[i] = sum_k grad_out[in_nbr[k][i]] (one write per element)."""
    _check_feats(in_feat, manager, in_key)
    _assert(manager.exists(out_key), ERROR_MAP_NOT_FOUND)
    grad_out_feat = grad_out_feat.contiguous()
    _assert(in_feat.dtype == grad_out_feat.dtype, "type mismatch")
    km = manager._kernel_map(in_key, out_key, kernel_size, kernel_stride, kernel_dilation,
                             region_type, offset, True, True)
    _assert(grad_out_feat.size(0) == km.n_out, "Invalid grad_out size")
    C = in_feat.size(1)
    grad_in = torch.empty_like(in_feat)
    _lib.check(_lib.load().meb200_pool_backward(
        _lib.ptr(grad_out_feat), _lib.dtype_code(in_feat.dtype), km.n_in, C, _lib.ptr(km.in_nbr),
        km.K, km.n_out, _lib.POOL_SUM, None, _lib.ptr(grad_in), _lib.current_stream()))
    return grad_in


# ---- channel-wise (depthwise) convolution ------------------------------------------------------
def _chwise_map(in_feat, kernel, kernel_size, kernel_stride, kernel_dilation, region_type, offset,
                in_key, out_key, manager):
    """The convolution's own kernel map (is_transpose = is_pool = False): a MinkowskiConvolution
    of the same geometry shares the cache entry, and the map prefetch predicts it."""
    km = manager._kernel_map(in_key, out_key, kernel_size, kernel_stride, kernel_dilation,
                             region_type, offset, False, False)
    _assert(kernel.dim() == 2 and kernel.size(0) == km.K, "kernel shape", list(kernel.shape),
            "does not match the kernel volume", km.K)
    _assert(kernel.size(1) == in_feat.size(1), "Input feature size and kernel size mismatch")
    return km


def ChannelwiseConvolutionForwardGPU(in_feat, kernel, kernel_size, kernel_stride, kernel_dilation,
                                     region_type, offset, in_key, out_key, manager):
    """y[o, c] = sum_k kernel[k, c] * in_feat[out_nbr[k, o], c] in the feature dtype (reference:
    MinkowskiChannelwiseConvolution.py:142-191, a per-offset torch loop).  The kernel is read as
    fp32 [K, C] whatever its dtype.  Mutates `out_key` when it is unset."""
    _check_feats(in_feat, manager, in_key)
    _assert(kernel.is_cuda, "kernel must be CUDA")
    _set_strided_key(manager, in_key, out_key, kernel_stride)
    km = _chwise_map(in_feat, kernel, kernel_size, kernel_stride, kernel_dilation, region_type,
                     offset, in_key, out_key, manager)
    lib = _lib.load()
    C = in_feat.size(1)
    w = kernel.detach().float().contiguous()
    out = torch.empty((km.n_out, C), dtype=in_feat.dtype, device=in_feat.device)
    _lib.check(lib.meb200_chwise_gather(
        _lib.ptr(in_feat), _lib.dtype_code(in_feat.dtype), km.n_in, C, _lib.ptr(w),
        _lib.ptr(km.out_nbr), km.K, km.n_out, _lib.ptr(out), _lib.current_stream()))
    return out


def ChannelwiseConvolutionBackwardGPU(in_feat, grad_out_feat, kernel, kernel_size, kernel_stride,
                                      kernel_dilation, region_type, offset, in_key, out_key,
                                      manager, need_in=True, need_w=True):
    """(grad_in in the feature dtype, grad_kernel in the kernel's dtype; None where not needed).
    grad_in[i, c] = sum_k kernel[k, c] * grad_out[in_nbr[k, i], c] (the forward's gather over the
    reverse table, built only when asked for); grad_kernel[k, c] = sum_o in[out_nbr[k, o], c] *
    grad_out[o, c], accumulated in fp32."""
    _check_feats(in_feat, manager, in_key)
    _assert(kernel.is_cuda, "kernel must be CUDA")
    _assert(manager.exists(out_key), ERROR_MAP_NOT_FOUND)
    _assert(grad_out_feat.size(0) == manager.size(out_key), "Invalid grad_out size")
    km = _chwise_map(in_feat, kernel, kernel_size, kernel_stride, kernel_dilation, region_type,
                     offset, in_key, out_key, manager)
    lib = _lib.load()
    code = _lib.dtype_code(in_feat.dtype)
    grad_out = grad_out_feat.to(in_feat.dtype).contiguous()
    K, C = kernel.shape
    grad_in = grad_w = None
    if need_in:
        w = kernel.detach().float().contiguous()
        grad_in = torch.empty_like(in_feat)
        _lib.check(lib.meb200_chwise_gather(
            _lib.ptr(grad_out), code, km.n_out, C, _lib.ptr(w), _lib.ptr(km.in_nbr), K, km.n_in,
            _lib.ptr(grad_in), _lib.current_stream()))
    if need_w:
        grad_w = torch.empty((K, C), dtype=torch.float32, device=in_feat.device)
        nbytes = int(lib.meb200_chwise_wgrad_workspace_bytes(km.n_out, C, K, code))
        ws = torch.empty(nbytes, dtype=torch.uint8, device=in_feat.device) if nbytes else None
        _lib.check(lib.meb200_chwise_wgrad(
            _lib.ptr(in_feat), _lib.ptr(grad_out), code, km.n_in, C, _lib.ptr(km.out_nbr), K,
            km.n_out, _lib.ptr(grad_w), _lib.ptr(ws), nbytes, _lib.current_stream()))
        if grad_w.dtype != kernel.dtype:
            grad_w = grad_w.to(kernel.dtype)
    return grad_in, grad_w


# ---- global pooling and broadcast over the origin map ------------------------------------------
_GLOBAL_CODE = {PoolingMode.GLOBAL_SUM_POOLING_DEFAULT: _lib.SEG_SUM,
                PoolingMode.GLOBAL_SUM_POOLING_KERNEL: _lib.SEG_SUM,
                PoolingMode.GLOBAL_SUM_POOLING_PYTORCH_INDEX: _lib.SEG_SUM,
                PoolingMode.GLOBAL_AVG_POOLING_DEFAULT: _lib.SEG_AVG,
                PoolingMode.GLOBAL_AVG_POOLING_KERNEL: _lib.SEG_AVG,
                PoolingMode.GLOBAL_AVG_POOLING_PYTORCH_INDEX: _lib.SEG_AVG,
                PoolingMode.GLOBAL_MAX_POOLING_DEFAULT: _lib.SEG_MAX,
                PoolingMode.GLOBAL_MAX_POOLING_KERNEL: _lib.SEG_MAX,
                PoolingMode.GLOBAL_MAX_POOLING_PYTORCH_INDEX: _lib.SEG_MAX}
_BCAST_CODE = {BroadcastMode.ELEMENTWISE_ADDITON: _lib.BCAST_ADD,
               BroadcastMode.ELEMENTWISE_MULTIPLICATION: _lib.BCAST_MUL}


def _segment_reduce(a, grp, mode, b=None, aux=None):
    """fp32 [B, C] per-cloud SUM / AVG / MAX of a (or of a * b) over the rows of `grp`."""
    lib = _lib.load()
    n, C = a.shape
    out = torch.empty((grp.B, C), dtype=torch.float32, device=a.device)
    nbytes = int(lib.meb200_segment_workspace_bytes(n, C, grp.B))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=a.device)
    _lib.check(lib.meb200_segment_reduce(
        _lib.ptr(a), _lib.ptr(b), _lib.dtype_code(a.dtype), n, C, _lib.ptr(grp.order),
        _lib.ptr(grp.seg_start), _lib.ptr(grp.tile_start), grp.B, mode, _lib.ptr(out),
        _lib.ptr(aux), _lib.ptr(ws), nbytes, _lib.current_stream()))
    return out


def _broadcast(x, g32, grp, op, out_dtype=None, argmax=None, n=None, C=None):
    """[n, C] x op g32[segment of the row] (g32: fp32 [B, C])."""
    lib = _lib.load()
    if x is not None:
        n, C = x.shape
    out_dtype = out_dtype or x.dtype
    out = torch.empty((n, C), dtype=out_dtype, device=g32.device)
    code = _lib.dtype_code(x.dtype if x is not None else out_dtype)
    _lib.check(lib.meb200_broadcast(
        _lib.ptr(x), code, _lib.ptr(g32), _lib.ptr(argmax), _lib.ptr(grp.row_seg), n, C, op,
        _lib.ptr(out), _lib.dtype_code(out_dtype), _lib.current_stream()))
    return out


def _broadcast_fma(x, g32, grp, z=None, h32=None, k32=None):
    """x * g32[s] + z * h32[s] + k32[s] per row (s = the row's cloud), in x's dtype."""
    lib = _lib.load()
    n, C = x.shape
    out = torch.empty_like(x)
    _lib.check(lib.meb200_broadcast_fma(
        _lib.ptr(x), _lib.ptr(z), _lib.dtype_code(x.dtype), _lib.ptr(g32), _lib.ptr(h32),
        _lib.ptr(k32), _lib.ptr(grp.row_seg), n, C, _lib.ptr(out), _lib.current_stream()))
    return out


def _f32c(t):
    return t if (t.dtype == torch.float32 and t.is_contiguous()) else t.float().contiguous()


def _check_glob(manager, in_feat, glob_feat, glob_key):
    _assert(glob_feat.is_cuda, "in_feat_glob must be CUDA (this backend has no CPU path)")
    _assert(glob_feat.dim() == 2, "Invalid in_feat_glob.dim():", glob_feat.dim())
    _assert(manager.exists(glob_key), ERROR_MAP_NOT_FOUND)
    B = manager.origin_map_size()
    _assert(glob_feat.size(0) == B, "Invalid in_feat_glob size", glob_feat.size(0), "!=", B)
    _assert(in_feat.size(1) == glob_feat.size(1), "Invalid feature sizes", in_feat.size(1), "!=",
            glob_feat.size(1))
    _assert(in_feat.dtype == glob_feat.dtype, "Incompatible scalar_type. Use the same float type "
            "for both in_feat and in_feat_glob.")


def GlobalPoolingForwardGPU(in_feat, pooling_mode, in_key, out_key, manager, is_field=False):
    """reference: GlobalPoolingForwardCPU src/global_pooling_cpu.cpp:43-200 -> (out_feat [B, C],
    num_nonzero [B] (sum / avg, feature dtype) | max_index int32 [B, C] (flat row*C + c)).
    Mutates `out_key` (-> the origin key) when it is unset.  All nine GLOBAL_* modes are accepted;
    the _DEFAULT / _KERNEL / _PYTORCH_INDEX variants select a strategy in the reference, not a
    result, and run the same kernels here.  `is_field`: `in_key` is a tensor field key and the
    rows are its points (a field key may equal a map key, so the caller says which it holds)."""
    _check_feats(in_feat, manager, in_key, is_field=is_field)
    _assert(pooling_mode in _GLOBAL_CODE, "Invalid pooling mode", pooling_mode)
    okey = manager._origin()
    if not out_key.is_key_set():
        out_key.set_key(list(okey[0]), okey[1])
    grp = manager._grouping(in_key, is_field)
    mode = _GLOBAL_CODE[pooling_mode]
    if mode == _lib.SEG_MAX:
        aux = torch.empty((grp.B, in_feat.size(1)), dtype=torch.int32, device=in_feat.device)
    else:
        aux = torch.empty(grp.B, dtype=torch.float32, device=in_feat.device)
    out = _segment_reduce(in_feat, grp, mode, aux=aux)
    if mode != _lib.SEG_MAX:
        aux = aux.to(in_feat.dtype)
    return out.to(in_feat.dtype), aux


def GlobalPoolingBackwardGPU(in_feat, grad_out_feat, num_nonzero, pooling_mode, in_key, out_key,
                             manager, is_field=False):
    """reference: GlobalPoolingBackwardCPU src/global_pooling_cpu.cpp:221-330.  The average's
    divisor is the exact per-cloud row count of the grouping (num_nonzero may be rounded in
    bf16 / fp16); the max gradient goes to the row max_index names, whatever the cloud count."""
    _check_feats(in_feat, manager, in_key, is_field=is_field)
    _assert(pooling_mode in _GLOBAL_CODE, "Invalid pooling mode", pooling_mode)
    _assert(manager.exists(out_key), ERROR_MAP_NOT_FOUND)
    grp = manager._grouping(in_key, is_field)
    _assert(grad_out_feat.dim() == 2 and grad_out_feat.size(0) == grp.B,
            "Invalid grad_out size", tuple(grad_out_feat.shape))
    _assert(in_feat.size(1) == grad_out_feat.size(1), "Input feature size and kernel size mismatch")
    _assert(in_feat.dtype == grad_out_feat.dtype, "type mismatch")
    mode = _GLOBAL_CODE[pooling_mode]
    g = _f32c(grad_out_feat)
    if mode == _lib.SEG_MAX:
        _assert(num_nonzero.dtype == torch.int32 and num_nonzero.shape == grad_out_feat.shape,
                "max_index must be int32 [B, C]")
        return _broadcast(None, g, grp, _lib.BCAST_MAXGRAD, in_feat.dtype,
                          argmax=num_nonzero.contiguous(), n=grp.n, C=in_feat.size(1))
    if mode == _lib.SEG_AVG:
        g = (g / grp.counts().clamp(min=1.0)[:, None]).contiguous()
    return _broadcast(None, g, grp, _lib.BCAST_COPY, in_feat.dtype, n=grp.n, C=in_feat.size(1))


def BroadcastForwardGPU(in_feat, in_feat_glob, broadcast_mode, in_key, glob_key, manager,
                        is_field=False):
    """reference: BroadcastForwardCPU src/broadcast_cpu.cpp:44-90:
    out[i] = in_feat[i] + / * in_feat_glob[cloud of i].  `is_field`: `in_key` is a tensor field."""
    _check_feats(in_feat, manager, in_key, is_field=is_field)
    _assert(broadcast_mode in _BCAST_CODE, "Invalid broadcast mode", broadcast_mode)
    _check_glob(manager, in_feat, in_feat_glob, glob_key)
    grp = manager._grouping(in_key, is_field)
    return _broadcast(in_feat, _f32c(in_feat_glob), grp, _BCAST_CODE[broadcast_mode])


def BroadcastBackwardGPU(in_feat, in_feat_glob, grad_out_feat, broadcast_mode, in_key, glob_key,
                         manager, is_field=False):
    """reference: BroadcastBackwardCPU src/broadcast_cpu.cpp:92-150 (broadcast_kernel.hpp):
    add: dx = dy, dg[b] = sum_{i in b} dy;  mul: dx = dy * g[b(i)], dg[b] = sum_{i in b} dy * x."""
    _check_feats(in_feat, manager, in_key, is_field=is_field)
    _assert(broadcast_mode in _BCAST_CODE, "Invalid broadcast mode", broadcast_mode)
    _check_glob(manager, in_feat, in_feat_glob, glob_key)
    grad_out_feat = grad_out_feat.contiguous()
    _assert(grad_out_feat.shape == in_feat.shape and grad_out_feat.dtype == in_feat.dtype,
            "Incompatible grad_out_feat")
    grp = manager._grouping(in_key, is_field)
    if broadcast_mode == BroadcastMode.ELEMENTWISE_ADDITON:
        grad_in = grad_out_feat
        grad_glob = _segment_reduce(grad_out_feat, grp, _lib.SEG_SUM)
    else:
        grad_in = _broadcast(grad_out_feat, _f32c(in_feat_glob), grp, _lib.BCAST_MUL)
        grad_glob = _segment_reduce(grad_out_feat, grp, _lib.SEG_SUM, b=in_feat)
    return grad_in, grad_glob.to(in_feat_glob.dtype)


# ---- pruning, union and arithmetic between different coordinate maps ---------------------------
def _gather_rows(src, idx, n_out):
    """[n_out, C] rows src[idx[j]] (zero where idx[j] < 0): meb200_gather_rows."""
    out = torch.empty((n_out, src.size(1)), dtype=src.dtype, device=src.device)
    _lib.check(_lib.load().meb200_gather_rows(
        _lib.ptr(src), _lib.dtype_code(src.dtype), src.size(0), src.size(1), _lib.ptr(idx), n_out,
        _lib.ptr(out), _lib.current_stream()))
    return out


def PruningForwardGPU(in_feat, keep, in_key, out_key, manager):
    """reference: PruningForwardGPU (pybind/extern.hpp:414-421, validation of
    src/pruning_cpu.cpp:49-69).  Mutates `out_key` (-> a new key at the input's tensor stride, rows
    = the kept rows in ascending input order) when it is unset."""
    _assert(in_feat.is_contiguous(), "in_feat must be contiguous")
    _assert(keep.is_contiguous(), "keep must be contiguous")
    _assert(keep.dtype in (torch.bool, torch.uint8), "keep must be a boolean tensor")
    _assert(in_feat.dim() == 2, "in_feat.dim():", in_feat.dim())
    _assert(keep.dim() == 1, "keep.dim():", keep.dim())
    N = in_feat.size(0)
    _assert(N == keep.size(0), "Input feature size and keep size mismatch")
    _assert(manager.exists(in_key), ERROR_MAP_NOT_FOUND)
    _assert(N == manager.size(in_key), "Invalid in_feat size", N, "!=", manager.size(in_key))
    _assert(in_feat.is_cuda, "in_feat must be CUDA (this backend has no CPU path)")
    _assert(keep.device == in_feat.device, "keep must be on the device of in_feat")
    ik = manager._k(in_key)
    if not out_key.is_key_set():
        ok = manager._prune(in_key, keep)
        out_key.set_key(list(ok[0]), ok[1])
    ent = manager._prunes.get((ik, manager._k(out_key)))
    _assert(ent is not None, "out_key", out_key, "is not a pruning of in_key", in_key)
    uidx, _ = ent
    if uidx.numel() == 0:
        warnings.warn("MinkowskiPruning: Generating an empty SparseTensor")
    return _gather_rows(in_feat, uidx, uidx.numel())


def PruningBackwardGPU(grad_out_feat, in_key, out_key, manager):
    """reference: PruningBackwardGPU (pybind/extern.hpp:423-430): grad_in[r] = grad_out[row of r in
    the pruned map], 0 for pruned rows (fully written, no zero fill)."""
    grad_out_feat = grad_out_feat.contiguous()
    _assert(grad_out_feat.is_cuda, "grad_out_feat must be CUDA (this backend has no CPU path)")
    _assert(grad_out_feat.dim() == 2, "grad_out_feat.dim():", grad_out_feat.dim())
    ik, ok = manager._k(in_key), manager._k(out_key)
    ent = manager._prunes.get((ik, ok))
    _assert(ent is not None, "out_key", out_key, "is not a pruning of in_key", in_key)
    uidx, inv = ent
    _assert(grad_out_feat.size(0) == uidx.numel(), "Invalid grad_out_feat size",
            grad_out_feat.size(0), "!=", uidx.numel())
    return _gather_rows(grad_out_feat, inv, manager.size(in_key))


def _pointer_table(feats):
    """(DEVICE int64 [N] of the feature pointers, largest power of two <= 16 dividing all of them)."""
    ptrs = [t.data_ptr() for t in feats]
    align = 16
    for p in ptrs:
        while p % align:
            align //= 2
    table = torch.tensor(ptrs, dtype=torch.int64).to(feats[0].device, non_blocking=True)
    return table, align


def _check_union_feats(feats, um):
    _assert(len(feats) == len(um.sizes), "The input features and keys must have the same length")
    f0 = feats[0]
    for i, (f, n) in enumerate(zip(feats, um.sizes)):
        _assert(f.dim() == 2 and f.size(0) == n, "input", i, "features", tuple(f.shape),
                "do not match its map of", n, "rows")
        _assert(f.size(1) == f0.size(1), "input", i, "has", f.size(1), "channels,", f0.size(1),
                "expected")
        _assert(f.dtype == f0.dtype, "input", i, "dtype", f.dtype, "!=", f0.dtype)
    _check_union_devices(feats)


def _check_union_devices(feats):
    for i, f in enumerate(feats):
        _assert(f.is_cuda and f.device == feats[0].device, "input", i, "must be a CUDA tensor on",
                feats[0].device, "(this backend has no CPU path)")


def union_fold_forward(feats, um, op):
    """[M, C] fold of the inputs over union map `um` (meb200_union_fold_forward)."""
    feats = [f.contiguous() for f in feats]
    _check_union_feats(feats, um)
    C = feats[0].size(1)
    out = torch.empty((um.M, C), dtype=feats[0].dtype, device=feats[0].device)
    if um.M == 0 or C == 0:
        return out
    table, align = _pointer_table(feats)
    _lib.check(_lib.load().meb200_union_fold_forward(
        _lib.ptr(table), len(feats), align, _lib.ptr(um.src), um.M, C,
        _lib.dtype_code(feats[0].dtype), op, _lib.ptr(out), _lib.current_stream()))
    return out


def union_fold_backward(grad_out, feats, um, op, needs=None):
    """Gradients of union_fold_forward for every input (None where needs[i] is False)."""
    feats = [f.contiguous() for f in feats]
    grad_out = grad_out.contiguous()
    _check_union_feats(feats, um)
    C = feats[0].size(1)
    _assert(grad_out.shape == (um.M, C) and grad_out.dtype == feats[0].dtype,
            "Invalid grad_out_feat", tuple(grad_out.shape), grad_out.dtype)
    table, align = _pointer_table(feats)
    lib = _lib.load()
    grads = []
    for i, f in enumerate(feats):
        if needs is not None and not needs[i]:
            grads.append(None)
            continue
        g = torch.empty_like(f)
        _lib.check(lib.meb200_union_fold_backward(
            _lib.ptr(table), len(feats), align, _lib.ptr(um.src), um.M, C, _lib.dtype_code(f.dtype),
            op, _lib.ptr(grad_out), i, _lib.ptr(um.u[i]), um.sizes[i], _lib.ptr(g),
            _lib.current_stream()))
        grads.append(g)
    return grads


# ---- tensor fields: points <-> voxels, interpolation ----------------------------------------------
def group_by_row(keys, M):
    """(start int32 [M+1], perm int32 [P]): the entries of int32 keys grouped by key in [0, M),
    ascending entry order inside a key (meb200_group_by_row)."""
    lib = _lib.load()
    P = keys.numel()
    dev = keys.device
    start = torch.empty(M + 1, dtype=torch.int32, device=dev)
    perm = torch.empty(P, dtype=torch.int32, device=dev)
    nbytes = int(lib.meb200_group_by_row_scratch_bytes(P, M)) if P else 0
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev) if P else None
    _lib.check(lib.meb200_group_by_row(_lib.ptr(keys), P, M, _lib.ptr(start), _lib.ptr(perm),
                                       _lib.ptr(scratch), nbytes, _lib.current_stream()))
    return start, perm


def field_reduce(src, group, M, mode, weight=None, src_div=1, src_row=None):
    """[M, C] reduction of the rows of `src` over a grouping (meb200_field_reduce) -> (out, argmax
    int32 [M, C] for MAX else None).  Entry j reads row src_row[j] when src_row (int32, range
    checked by the caller) is given, else row j // src_div."""
    src = src.contiguous()
    start, perm = group
    C = src.size(1)
    out = torch.empty((M, C), dtype=src.dtype, device=src.device)
    argmax = torch.empty((M, C), dtype=torch.int32, device=src.device) \
        if mode == _lib.FIELD_MAX else None
    _lib.check(_lib.load().meb200_field_reduce(
        _lib.ptr(src), _lib.dtype_code(src.dtype), src.size(0), C, _lib.ptr(perm), _lib.ptr(start),
        M, _lib.ptr(weight), _lib.ptr(src_row), src_div, mode, _lib.ptr(out), _lib.ptr(argmax),
        _lib.current_stream()))
    return out, argmax


def field_expand(g, inv, mode, start=None, argmax=None, unique_index=None):
    """[N, C] rows g[inv[i]] scaled per mode (meb200_field_expand): the backward of field_reduce."""
    g = g.contiguous()
    n, C = inv.numel(), g.size(1)
    out = torch.empty((n, C), dtype=g.dtype, device=g.device)
    _lib.check(_lib.load().meb200_field_expand(
        _lib.ptr(g), _lib.dtype_code(g.dtype), g.size(0), C, _lib.ptr(inv), n, mode, _lib.ptr(start),
        _lib.ptr(argmax), _lib.ptr(unique_index), _lib.ptr(out), _lib.current_stream()))
    return out


def gather_rows(src, idx, n_out):
    """Public name of the row gather (meb200_gather_rows) for the tensor-field functions."""
    return _gather_rows(src.contiguous(), idx, n_out)


def interp_forward(F, rows, w):
    """[n, C] = sum_k w[q, k] * F[rows[q, k]] in ascending k (meb200_interp_forward)."""
    F = F.contiguous()
    n, K = rows.shape
    out = torch.empty((n, F.size(1)), dtype=F.dtype, device=F.device)
    _lib.check(_lib.load().meb200_interp_forward(
        _lib.ptr(F), _lib.dtype_code(F.dtype), F.size(0), F.size(1), _lib.ptr(rows), _lib.ptr(w), n,
        K, _lib.ptr(out), _lib.current_stream()))
    return out


# ---- COO sparse matrix times dense matrix, direct max pooling (pybind/extern.hpp:497-506, 654-665)
_INDEX_LIMIT = 0x7FFFFFFF       # rows, columns and flat mask sizes are int32 keys below this


def _index32(t):
    """int32 form of an index tensor: int32 as it is; int64 and float as the reference's `.int()`
    (float truncated towards zero), with values outside int32 clamped to -1 or 2^31 - 1 so that
    they stay out of range instead of wrapping into it.  The caller's tensor is never written."""
    t = t.reshape(-1)
    if t.dtype == torch.int32:
        return t.contiguous()
    return t.long().clamp(-1, 2 ** 31 - 1).int()


def _check_dim(n, what):
    _assert(0 <= int(n) < _INDEX_LIMIT, what, "must lie in [0, 2^31 - 1), got", n)
    return int(n)


def _pair_list(rows, cols, n_rows, n_cols, device):
    """int32 (rows, cols) of a pair list on `device`, every rows[p] in [0, n_rows) and cols[p] in
    [0, n_cols) (meb200_check_pairs: one kernel and one host synchronisation), else RuntimeError."""
    _assert(rows.is_cuda and cols.is_cuda, "index tensors must be CUDA (this backend has no CPU path)")
    _assert(rows.device == device and cols.device == device, "all inputs must be on", device)
    r, c = _index32(rows), _index32(cols)
    _assert(r.numel() == c.numel(), "Invalid length", r.numel(), c.numel())
    _assert(r.numel() < _INDEX_LIMIT, "too many entries:", r.numel())
    status = torch.empty(1, dtype=torch.int32, device=device)
    _lib.check(_lib.load().meb200_check_pairs(_lib.ptr(r), _lib.ptr(c), r.numel(), n_rows, n_cols,
                                              _lib.ptr(status), _lib.current_stream()))
    return r, c


def _check_mat(mat, what="mat"):
    _assert(mat.is_cuda, what, "must be CUDA (this backend has no CPU path)")
    _assert(mat.dim() == 2, what, "must be a matrix, got shape", tuple(mat.shape))
    _lib.dtype_code(mat.dtype)      # fp32 / bf16 / fp16, else BackendError
    return mat.contiguous()


def _coo_reduce(r, c, M, mat, mode, weight=None, group=None):
    """[M, C] reduction over the entries (r[p], c[p]) of the rows mat[c[p]] into rows r[p], in entry
    order (meb200_group_by_row + meb200_field_reduce with src_row = c) -> (out, argmax for MAX).
    Without entries or channels nothing is launched: the output is 0 and argmax -1."""
    C = mat.size(1)
    if r.numel() == 0 or M == 0 or C == 0:
        out = torch.zeros((M, C), dtype=mat.dtype, device=mat.device)
        argmax = torch.full((M, C), -1, dtype=torch.int32, device=mat.device) \
            if mode == _lib.FIELD_MAX else None
        return out, argmax
    if group is None:
        group = group_by_row(r, M)
    return field_reduce(mat, group, M, mode, weight=weight, src_row=c)


def coo_spmm_int32(rows, cols, vals, dim_i, dim_j, mat, spmm_algorithm_id=1, is_sorted=False):
    """[dim_i, C] = A @ mat for the COO matrix A (dim_i x dim_j) with entries vals[p] at
    (rows[p], cols[p]): out[r] = sum over the entries of row r, in entry order, of
    fp32(vals[p]) * mat[cols[p]], accumulated in fp32 and rounded once to mat's dtype.  Duplicate
    entries are summed; a row without entries is 0.  Out-of-range indices raise RuntimeError, which
    costs one host synchronisation.  `spmm_algorithm_id` (a cuSPARSE algorithm in the reference) and
    `is_sorted` are accepted and ignored: the result does not depend on either."""
    mat = _check_mat(mat)
    dim_i, dim_j = _check_dim(dim_i, "dim_i"), _check_dim(dim_j, "dim_j")
    _assert(mat.size(0) == dim_j, "mat must have dim_j =", dim_j, "rows, got", mat.size(0))
    _assert(vals.dtype == mat.dtype, "dtype mismatch", vals.dtype, mat.dtype)
    _assert(vals.device == mat.device, "device mismatch", vals.device, mat.device)
    r, c = _pair_list(rows, cols, dim_i, dim_j, mat.device)
    _assert(vals.numel() == r.numel(), "Invalid length", vals.numel(), r.numel())
    w = vals.reshape(-1).float().contiguous()    # bf16 / fp16 values widen exactly
    return _coo_reduce(r, c, dim_i, mat, _lib.FIELD_SUM, weight=w)[0]


def coo_spmm_average_int32(rows, cols, dim_i, dim_j, mat, spmm_algorithm_id=1):
    """[result, COO, vals]: result[r] = the mean of mat[cols[p]] over the entries of row r (the
    fp32 sum over the exact count, rounded once; 0 without entries); COO = int64 [2, P] of the
    entries stably sorted by row; vals = 1 / (entries of the row) in mat's dtype, so that
    coo_spmm_int32(COO[1], COO[0], vals, dim_j, dim_i, g) is the backward.  Out-of-range indices
    raise RuntimeError (one host synchronisation); `spmm_algorithm_id` is ignored."""
    mat = _check_mat(mat)
    dim_i, dim_j = _check_dim(dim_i, "dim_i"), _check_dim(dim_j, "dim_j")
    _assert(mat.size(0) == dim_j, "mat must have dim_j =", dim_j, "rows, got", mat.size(0))
    r, c = _pair_list(rows, cols, dim_i, dim_j, mat.device)
    if r.numel() == 0:
        out = torch.zeros((dim_i, mat.size(1)), dtype=mat.dtype, device=mat.device)
        return [out, torch.zeros((2, 0), dtype=torch.int64, device=mat.device),
                torch.zeros(0, dtype=mat.dtype, device=mat.device)]
    start, perm = group_by_row(r, dim_i)
    out, _ = _coo_reduce(r, c, dim_i, mat, _lib.FIELD_AVG, group=(start, perm))
    order = perm.long()
    coo = torch.stack((r[order], c[order])).long()
    count = start[1:] - start[:-1]
    vals = (1 / count[coo[0]]).to(mat.dtype)
    return [out, coo, vals]


def _direct_max_pool(in_map, out_map, in_feat, out_nrows, need_mask):
    """Direct max pooling forward -> (out, mask or None, winner, out_rows, in_rows): winner int32
    [out_nrows, C] is the winning pair of every output element (-1 for none), out_rows / in_rows the
    range-checked int32 maps."""
    _assert(in_feat.is_cuda, "in_feat must be CUDA (this backend has no CPU path)")
    _assert(in_feat.dim() == 2, "in_feat must be a matrix, got shape", tuple(in_feat.shape))
    n_in, C = _check_dim(in_feat.size(0), "in_nrows"), _check_dim(in_feat.size(1), "C")
    M = _check_dim(out_nrows, "out_nrows")
    bits = 64 if in_map.dtype == torch.int64 else 32
    lib = _lib.load()
    if need_mask:   # the size check of the flat mask (no launch without rows), before any copy
        _lib.check(lib.meb200_flat_mask(None, None, 0, C, n_in, bits, None, _lib.current_stream()))
    in_feat = _check_mat(in_feat, "in_feat")
    o, i = _pair_list(out_map, in_map, M, n_in, in_feat.device)
    out, winner = _coo_reduce(o, i, M, in_feat, _lib.FIELD_MAX)
    mask = None
    if need_mask:
        mask = torch.empty((M, C), dtype=torch.int64 if bits == 64 else torch.int32,
                           device=in_feat.device)
        if o.numel() == 0:
            mask.fill_(-1)
        else:
            _lib.check(lib.meb200_flat_mask(_lib.ptr(winner), _lib.ptr(i), M, C, n_in, bits,
                                            _lib.ptr(mask), _lib.current_stream()))
    return out, mask, winner, o, i


def direct_max_pool_fw(in_map, out_map, in_feat, out_nrows, is_sorted=False):
    """(out [out_nrows, C], mask [out_nrows, C]): out[o, c] = the maximum of in_feat[i, c] over the
    pairs (in_map[p], out_map[p]) = (i, o), the first pair in list order winning a tie, and
    mask[o, c] = i * C + c of that pair, in in_map's integer dtype (int32 for float maps).  An
    output row without pairs is 0 with mask -1.  Out-of-range maps raise RuntimeError (one host
    synchronisation), as does an int32 mask that cannot hold in_nrows * C - 1; `is_sorted` is
    ignored."""
    out, mask, _, _, _ = _direct_max_pool(in_map, out_map, in_feat, out_nrows, True)
    return out, mask


def direct_max_pool_bw(grad_out_feat, mask_index, in_nrows):
    """grad_in [in_nrows, C]: grad_out[o, c] added at the flat input element mask[o, c] of the
    forward, each (o, c) once.  The elements are grouped by their flat index (a stable radix sort of
    out_nrows * C int32 keys) and each input element sums its own in ascending (o, c) order, so the
    result is bit-identical run to run without atomics.  Mask entries outside [0, in_nrows * C), -1
    among them, send no gradient.  The int32 keys limit in_nrows * C to below 2^31 - 1 whatever the
    mask's dtype, which is stricter than the reference: MinkowskiDirectMaxPoolingFunction does not
    go through here and has no such limit (direct_max_pool_pairs_bw)."""
    g = _check_mat(grad_out_feat, "grad_out_feat")
    _assert(mask_index.is_cuda and mask_index.device == g.device, "mask must be on", g.device)
    _assert(tuple(mask_index.shape) == tuple(g.shape), "mask shape", tuple(mask_index.shape),
            "differs from grad_out_feat", tuple(g.shape))
    n_in, C = _check_dim(in_nrows, "in_nrows"), g.size(1)
    M = n_in * C
    _assert(M < _INDEX_LIMIT, "the flat mask in_nrows * C =", M, "must be below 2^31 - 1 here")
    if g.numel() == 0 or M == 0:
        return torch.zeros((n_in, C), dtype=g.dtype, device=g.device)
    group = group_by_row(_index32(mask_index), M)
    out, _ = field_reduce(g.view(-1, 1), group, M, _lib.FIELD_SUM)
    return out.view(n_in, C)


def direct_max_pool_pairs_bw(grad_out_feat, winner, out_rows, in_rows, in_nrows):
    """The backward of _direct_max_pool from its winning pairs: every pair p takes
    grad_out[out_rows[p], c] where it won (meb200_field_expand MAX over the P pairs, [P, C]), and
    each input row sums its pairs in pair order (meb200_group_by_row over in_rows +
    meb200_field_reduce SUM).  Each (o, c) has one winning pair, so it counts once even when a pair
    repeats; bit-identical run to run, no atomics.  It sorts P keys where direct_max_pool_bw sorts
    out_nrows * C (BASELINE.md §16)."""
    g = grad_out_feat.contiguous()
    C = g.size(1)
    if in_rows.numel() == 0 or C == 0:
        return torch.zeros((in_nrows, C), dtype=g.dtype, device=g.device)
    per_pair = field_expand(g, out_rows.long(), _lib.FIELD_MAX, argmax=winner)
    out, _ = field_reduce(per_pair, group_by_row(in_rows, in_nrows), in_nrows, _lib.FIELD_SUM)
    return out
