"""TEST INFRASTRUCTURE — numpy restatement of the reference's CPU path.

Every function restates one piece of NVIDIA/MinkowskiEngine v0.5.4 (reference paths are
relative to /root/reference).  It is pinned two ways (tests/test_oracle.py): against the
reference's own golden vectors (tests/golden/reference_goldens.json, transcribed from
tests/cpp/kernel_region_cpu_test.py:24-82, tests/cpp/coordinate_map_cpu_test.py:49-125,
tests/python/coordinate_manager.py:183-200) and against outputs of the compiled reference
(`oracle/_ref`, fixtures in tests/golden/ref_*.npz made by tests/golden/make_fixtures.py).

Row order of derived maps is implementation-defined in the reference (hash-table iteration
order, coordinate_map_cpu.hpp:429-434), so derived maps are returned in lexicographic row
order and comparisons canonicalise both sides (`canonical_*` helpers).
"""
import numpy as np

HYPER_CUBE, HYPER_CROSS, CUSTOM = 0, 1, 2
POOL_SUM, POOL_AVG, POOL_MAX = 0, 1, 2


# ---- coordinates -------------------------------------------------------------------------
def insert_and_map(coords):
    """CoordinateMapCPU::insert_and_map<true> (src/coordinate_map_cpu.hpp:353-380):
    serial insert; the first occurrence of a coordinate wins and unique rows are numbered
    by rank of first occurrence.  Returns (unique_index[M], inverse_map[N])."""
    coords = np.ascontiguousarray(coords, dtype=np.int32)
    n = coords.shape[0]
    if n == 0:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    _, first, inv = np.unique(coords, axis=0, return_index=True, return_inverse=True)
    inv = inv.reshape(-1)
    order = np.argsort(first, kind="stable")          # unique groups by first occurrence
    rank = np.empty_like(order)
    rank[order] = np.arange(len(order))
    return first[order].astype(np.int64), rank[inv].astype(np.int64)


def stride_coordinate(coords, out_tensor_stride):
    """detail::stride_coordinate (src/coordinate_map.hpp:58-76): per spatial axis
    floor((float)c / s) * s — the reference does this in single precision."""
    coords = np.asarray(coords, dtype=np.int32)
    out = coords.copy()
    s = np.asarray(out_tensor_stride, dtype=np.int32)
    q = np.floor(coords[:, 1:].astype(np.float32) / s.astype(np.float32))
    out[:, 1:] = (q * s.astype(np.float32)).astype(np.int32)
    return out


def lexsort_rows(a):
    a = np.asarray(a)
    if a.shape[0] == 0:
        return np.zeros(0, np.int64)
    return np.lexsort(a.T[::-1])


def unique_rows(a):
    """Unique rows in lexicographic order (the canonical order used for derived maps)."""
    a = np.ascontiguousarray(a, dtype=np.int32)
    if a.shape[0] == 0:
        return a
    return np.unique(a, axis=0)


def stride_map_coords(coords, tensor_stride, kernel_stride):
    """CoordinateMapCPU::stride (src/coordinate_map_cpu.hpp:418-437) + stride_tensor_stride
    (src/coordinate_map.hpp:78-96).  Returns (out_coords in canonical order, out_tensor_stride)."""
    out_ts = [int(t) * int(s) for t, s in zip(tensor_stride, kernel_stride)]
    return unique_rows(stride_coordinate(coords, out_ts)), out_ts


def stride_region_coords(coords, offsets, out_tensor_stride, is_transpose):
    """CoordinateMapCPU::stride_region (src/coordinate_map_cpu.hpp:446-487): every input row
    moved by every region offset; the forward (expanding) form keeps only the coordinates that
    are multiples of the out tensor stride, the transposed form keeps them all.  Returns the
    unique coordinates in canonical order."""
    coords = np.asarray(coords, np.int32)
    offs = np.asarray(offsets, np.int32)
    cand = np.repeat(coords, len(offs), axis=0)
    cand[:, 1:] += np.tile(offs, (len(coords), 1))
    if not is_transpose:
        s = np.asarray(out_tensor_stride, np.int32)[None, :]
        cand = cand[(cand[:, 1:] % s == 0).all(axis=1)]
    return unique_rows(cand)


def region_offsets(region_type, kernel_size, dilation, tensor_stride, custom=None):
    """kernel_region::coordinate_at (src/kernel_region.hpp:198-247) as an offset table
    [K, D]; volume per set_volume (:250-270)."""
    D = len(kernel_size)
    if region_type == HYPER_CUBE:
        K = int(np.prod(kernel_size))
        offs = np.zeros((K, D), np.int32)
        for k in range(K):
            rem = k
            for a in range(D):
                ks = kernel_size[a]
                i = rem % ks
                rem //= ks
                if ks % 2 == 0:
                    offs[k, a] = dilation[a] * tensor_stride[a] * i
                else:
                    offs[k, a] = (i - ks // 2) * dilation[a] * tensor_stride[a]
        return offs
    if region_type == HYPER_CROSS:
        K = 1 + sum(k - 1 for k in kernel_size)
        offs = np.zeros((K, D), np.int32)
        for k in range(1, K):
            ind, axis = k - 1, 0
            while axis < D:
                if ind < kernel_size[axis] - 1:
                    break
                ind -= kernel_size[axis] - 1
                axis += 1
            r = (kernel_size[axis] - 1) // 2
            off = (ind + 1) if ind < r else (ind - 2 * r)
            offs[k, axis] = off * dilation[axis] * tensor_stride[axis]
        return offs
    if region_type == CUSTOM:
        return (np.asarray(custom, np.int32) * np.asarray(tensor_stride, np.int32)[None, :])
    raise ValueError(region_type)


def region_coordinates(coords, region_type, kernel_size, dilation, tensor_stride):
    """Golden-test form (tests/cpp/kernel_region_cpu_test.py): for each coordinate, the K
    region coordinates in kernel-index order."""
    offs = region_offsets(region_type, kernel_size, dilation, tensor_stride)
    coords = np.asarray(coords, np.int32)
    out = []
    for c in coords:
        for d in offs:
            out.append([int(c[0])] + [int(v) for v in (c[1:] + d)])
    return out


class RowIndex:
    """Exact row lookup for int32 coordinate rows (the role of robin_hood's map in
    src/coordinate_map_cpu.hpp:291-300); sort + searchsorted on a void view."""

    def __init__(self, coords):
        coords = np.ascontiguousarray(coords, dtype=np.int32)
        self.ncols = coords.shape[1]
        keys = self._keys(coords)
        self.order = np.argsort(keys, kind="stable")
        self.sorted = keys[self.order]

    @staticmethod
    def _keys(c):
        # order-preserving byte key: flip the sign bit, store big-endian
        u = (np.ascontiguousarray(c, dtype=np.int32).view(np.uint32) ^ np.uint32(0x80000000))
        be = u.astype(">u4")
        return np.ascontiguousarray(be).view(np.dtype((np.void, 4 * c.shape[1]))).reshape(-1)

    def find(self, query):
        if len(self.sorted) == 0 or len(query) == 0:
            return np.full(len(query), -1, np.int64)
        q = self._keys(query)
        pos = np.searchsorted(self.sorted, q)
        pos = np.minimum(pos, len(self.sorted) - 1)
        hit = self.sorted[pos] == q
        return np.where(hit, self.order[pos], -1).astype(np.int64)


def map_find(map_coords, queries):
    """CoordinateMapCPU::find (src/coordinate_map_cpu.hpp:388-412):
    (valid_query_index, query_result)."""
    r = RowIndex(map_coords).find(np.asarray(queries, np.int32))
    valid = np.nonzero(r >= 0)[0]
    return valid, r[valid]


def kernel_map(in_coords, out_coords, offsets):
    """CoordinateMapCPU::kernel_map (src/coordinate_map_cpu.hpp:569-670): for every out row
    and kernel index k probe in_map at out + offset_k.  Returns (in_maps, out_maps): lists
    over k of int64 arrays, pairs ordered by out row (the reference's order within an offset
    is nondeterministic, :642-649)."""
    in_coords = np.ascontiguousarray(in_coords, np.int32)
    out_coords = np.ascontiguousarray(out_coords, np.int32)
    idx = RowIndex(in_coords)
    in_maps, out_maps = [], []
    for d in np.asarray(offsets, np.int32):
        q = out_coords.copy()
        q[:, 1:] += d[None, :]
        r = idx.find(q)
        o = np.nonzero(r >= 0)[0]
        in_maps.append(r[o])
        out_maps.append(o.astype(np.int64))
    return in_maps, out_maps


def transposed_kernel_map(in_coords, out_coords, offsets):
    """Transposed convolution map (src/coordinate_map_manager.cpp:789-811): iterate the
    coarse INPUT rows, probe the fine OUTPUT map at in + offset_k (offsets in output-stride
    units), pairs (k, in = iterated row, out = found row)."""
    a, b = kernel_map(out_coords, in_coords, offsets)   # 'found' rows, iterated rows
    return b, a


def stride_map(in_coords, out_coords, out_tensor_stride):
    """CoordinateMapCPU::stride_map (src/coordinate_map_cpu.hpp:672-722): every input row ->
    the row of its strided coordinate in the out map; one group."""
    q = stride_coordinate(in_coords, out_tensor_stride)
    r = RowIndex(out_coords).find(q)
    assert (r >= 0).all(), "Invalid out_coordinate_map"
    return [np.arange(len(in_coords), dtype=np.int64)], [r]


def kernel_map_triples(in_coords, out_coords, in_maps, out_maps):
    """Canonical form: set of (k, in coordinate..., out coordinate...) tuples."""
    rows = []
    for k, (i, o) in enumerate(zip(in_maps, out_maps)):
        if len(i) == 0:
            continue
        kk = np.full((len(i), 1), k, np.int64)
        rows.append(np.concatenate([kk, np.asarray(in_coords)[np.asarray(i)],
                                    np.asarray(out_coords)[np.asarray(o)]], axis=1))
    if not rows:
        return np.zeros((0, 1 + 2 * np.asarray(in_coords).shape[1]), np.int64)
    t = np.concatenate(rows, axis=0).astype(np.int64)
    return t[lexsort_rows(t)]


# ---- convolution -------------------------------------------------------------------------
def conv_forward(in_feat, kernel, in_maps, out_maps, n_out):
    """ConvolutionForwardKernelCPU (src/convolution_kernel.hpp:33-79): per offset gather ->
    GEMM -> add into the output rows.  Accumulates in float64 so the oracle is the
    well-conditioned side of any fp32 comparison."""
    c_out = kernel.shape[2]
    out = np.zeros((n_out, c_out), np.float64)
    w = kernel.astype(np.float64)
    x = in_feat.astype(np.float64)
    for k, (i, o) in enumerate(zip(in_maps, out_maps)):
        if len(i):
            np.add.at(out, o, x[i] @ w[k])
    return out


def conv_backward(in_feat, grad_out, kernel, in_maps, out_maps):
    """ConvolutionBackwardKernelCPU (src/convolution_kernel.hpp:81-144):
    dIn[i] += dOut[o] W_k^T ; dW_k += In[i]^T dOut[o]."""
    x, g, w = in_feat.astype(np.float64), grad_out.astype(np.float64), kernel.astype(np.float64)
    grad_in = np.zeros_like(x)
    grad_w = np.zeros_like(w)
    for k, (i, o) in enumerate(zip(in_maps, out_maps)):
        if len(i):
            np.add.at(grad_in, i, g[o] @ w[k].T)
            grad_w[k] = x[i].T @ g[o]
    return grad_in, grad_w


# ---- pooling -----------------------------------------------------------------------------
def pool_forward(in_feat, in_maps, out_maps, n_out, mode):
    """NonzeroAvgPoolingForwardKernelCPU (src/pooling_avg_kernel.hpp:40-101) and
    MaxPoolingForwardKernelCPU (src/pooling_max_kernel.hpp:35-90).  Returns (out, aux):
    aux = num_nonzero[n_out] (avg), max_index int32 [n_out, C] (max), None (sum)."""
    x = in_feat.astype(np.float64)
    C = x.shape[1]
    if mode == POOL_MAX:
        out = np.full((n_out, C), -np.finfo(np.float32).max, np.float64)
        mask = np.full((n_out, C), -1, np.int64)
        for i_k, o_k in zip(in_maps, out_maps):          # ascending k, strict '<'
            for i, o in zip(i_k, o_k):
                better = out[o] < x[i]
                out[o] = np.where(better, x[i], out[o])
                mask[o] = np.where(better, i * C + np.arange(C), mask[o])
        return out, mask.astype(np.int32)
    out = np.zeros((n_out, C), np.float64)
    cnt = np.zeros(n_out, np.float64)
    for i_k, o_k in zip(in_maps, out_maps):
        if len(i_k):
            np.add.at(out, o_k, x[i_k])
            np.add.at(cnt, o_k, 1.0)
    if mode == POOL_AVG:
        nz = cnt > 0
        out[nz] /= cnt[nz, None]
        return out, cnt
    return out, None


def pool_backward(grad_out, n_in, in_maps, out_maps, mode, aux):
    """NonzeroAvgPoolingBackwardKernelCPU (src/pooling_avg_kernel.hpp:103-150) and
    MaxPoolingBackwardKernelCPU (src/pooling_max_kernel.hpp:92-115)."""
    g = grad_out.astype(np.float64)
    C = g.shape[1]
    grad_in = np.zeros((n_in, C), np.float64)
    if mode == POOL_MAX:
        flat = grad_in.reshape(-1)
        m = np.asarray(aux).reshape(-1)
        ok = m >= 0
        np.add.at(flat, m[ok], g.reshape(-1)[ok])
        return grad_in
    for i_k, o_k in zip(in_maps, out_maps):
        if len(i_k) == 0:
            continue
        if mode == POOL_AVG:
            cnt = np.asarray(aux, np.float64)[o_k]
            contrib = np.where(cnt[:, None] > 0, g[o_k] / np.maximum(cnt, 1)[:, None], 0.0)
        else:
            contrib = g[o_k]
        np.add.at(grad_in, i_k, contrib)
    return grad_in


# ---- canonicalisation helpers for parity tests -------------------------------------------
def canonical_rows(coords, feats=None):
    """Rows sorted lexicographically by coordinate; returns (coords, feats, perm)."""
    p = lexsort_rows(coords)
    return np.asarray(coords)[p], (None if feats is None else np.asarray(feats)[p]), p


# ---- synthetic inputs (SURVEY.md §8d) ----------------------------------------------------
from examples.synthetic import surface_cloud  # noqa: E402,F401  (neutral input generator, re-exported)
