"""float64 numpy restatement of unpooling and splatting (tests/test_unpool_splat_cpu.py pins it to
the compiled reference's fixtures; tests/test_gpu_unpool_splat.py compares the GPU against it).

Unpooling (MinkowskiPooling.py:441-580, src/local_pooling_transpose_cpu.cpp:40-100): both
backends call the non-zero-average kernel with use_avg = false, so the output is the SUM over the
transposed pooling map: out[o] = sum of in[i] over the pairs (i, o).  With kernel size = stride the
map is the stride map (coordinate_map_cpu.hpp:672-722): a fine row's only pair is its strided
parent.  Otherwise fine row o pairs with every coarse row at o + d * s_out, d in the region of the
kernel (coordinate_map_manager.cpp:789-811, offsets in output-stride units).

Splatting (MinkowskiTensorField.py:53-73, 381-406): every point adds w * F to each of its 2^D
corners floor(x) + {0,1}^D (the batch column floored, never offset), corner k with the upper end of
axis j when bit D-j of k is set; w = prod_j (1 - |x_j - c_j|) (coordinate_map_cpu.hpp:139-240 at
tensor stride 1).  The corners are inserted point-major; rows are numbered by first occurrence."""
import itertools

import numpy as np


def canon(coords):
    c = np.asarray(coords)
    return np.lexsort(c.T[::-1])


def _rows(coords):
    return {tuple(r): i for i, r in enumerate(np.asarray(coords).tolist())}


# ---- unpooling ------------------------------------------------------------------------------------
def region(D, k):
    """Offsets of a HYPER_CUBE kernel of size k in units of one stride: k odd -> [-(k-1)/2, (k-1)/2],
    k even -> [0, k)."""
    r = range(-(k // 2), k // 2 + 1) if k % 2 else range(k)
    return [np.array(d) for d in itertools.product(r, repeat=D)]


def unpool_pairs(in_coords, in_ts, out_coords, k, s):
    """(in_rows, out_rows) int64 of the transposed pooling map from the coarse map `in_coords`
    (tensor stride in_ts) onto the fine map `out_coords` (stride in_ts / s)."""
    D = np.asarray(in_coords).shape[1] - 1
    out_ts = in_ts // s
    look = _rows(in_coords)
    ii, oo = [], []
    for o, c in enumerate(np.asarray(out_coords).tolist()):
        if k == s:
            p = [c[0]] + [(v // in_ts) * in_ts for v in c[1:]]   # floor: the strided parent
            cands = [p]
        else:
            cands = [[c[0]] + [v + dv * out_ts for v, dv in zip(c[1:], d)] for d in region(D, k)]
        for p in cands:
            i = look.get(tuple(p))
            if i is not None:
                ii.append(i)
                oo.append(o)
    return np.array(ii, np.int64), np.array(oo, np.int64)


def expand_coords(in_coords, in_ts, k, s):
    """The fine coordinates expand_coordinates=True generates: every coarse row plus the kernel's
    offsets at the output stride (a set; canonical order)."""
    D = np.asarray(in_coords).shape[1] - 1
    out_ts = in_ts // s
    cand = [np.concatenate([[0], d * out_ts]) + r for r in np.asarray(in_coords)
            for d in region(D, k)]
    u = np.unique(np.array(cand), axis=0)
    return u[canon(u)]


def unpool_forward(x, pairs, n_out):
    i, o = pairs
    out = np.zeros((n_out, x.shape[1]))
    np.add.at(out, o, np.asarray(x, np.float64)[i])
    return out


def unpool_backward(g, pairs, n_in):
    i, o = pairs
    out = np.zeros((n_in, g.shape[1]))
    np.add.at(out, i, np.asarray(g, np.float64)[o])
    return out


# ---- splatting ------------------------------------------------------------------------------------
def corner_offsets(D):
    """[2^D, D+1] offsets; row k has 1 on axis j (1-based) when bit D-j of k is set."""
    K = 1 << D
    off = np.zeros((K, D + 1), np.int64)
    for k in range(K):
        for j in range(1, D + 1):
            off[k, j] = (k >> (D - j)) & 1
    return off


def splat_map(pts):
    """(map coords int64 [M, D+1] in first-occurrence order, rows int64 [n, 2^D], weights float64
    [n, 2^D]) of the splat of float points `pts` [n, D+1]."""
    p = np.asarray(pts, np.float64)
    D = p.shape[1] - 1
    corners = np.floor(p).astype(np.int64)[:, None, :] + corner_offsets(D)[None]
    flat = corners.reshape(-1, D + 1)
    _, first, inv = np.unique(flat, axis=0, return_index=True, return_inverse=True)
    order = np.argsort(first)                 # unique rows by first occurrence
    rank = np.empty_like(order)
    rank[order] = np.arange(len(order))
    coords = flat[np.sort(first)]
    rows = rank[inv.ravel()].reshape(len(p), 1 << D)
    w = np.prod(1.0 - np.abs(p[:, None, 1:] - corners[:, :, 1:]), axis=2)
    return coords, rows, w


def splat_forward(F, rows, w, M):
    out = np.zeros((M, F.shape[1]))
    np.add.at(out, rows.ravel(), (w[:, :, None] * np.asarray(F, np.float64)[:, None, :]).reshape(
        -1, F.shape[1]))
    return out


def splat_backward(g, rows, w):
    """The interpolation forward: out[q] = sum_k w[q, k] * g[rows[q, k]]."""
    return np.einsum("qk,qkc->qc", w, np.asarray(g, np.float64)[rows])
