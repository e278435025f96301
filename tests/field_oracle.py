"""numpy restatement of the TensorField operations (reference: MinkowskiTensorField.py,
coordinate_map_cpu.hpp:139-240 and :994-1037, src/interpolation_cpu.cpp), in float64 over the given
inputs.  Coordinates are quantised and interpolation weights computed in float32, as the reference
computes them; the sums are float64.  Pinned to the compiled reference's fixtures by
tests/test_field_cpu.py; the GPU tests compare against it element by element."""
import numpy as np

SUM, AVG, MAX, SUBSAMPLE = "UNWEIGHTED_SUM", "UNWEIGHTED_AVERAGE", "MAX_POOL", "RANDOM_SUBSAMPLE"


def quantize(points, stride):
    """int64 [N, D+1]: batch lroundf(x0), axes s * floorf(x / s) in float32."""
    p = np.asarray(points, np.float32)
    s = np.float32(stride)
    q = np.empty(p.shape, np.int64)
    b = p[:, 0]
    q[:, 0] = np.where(b >= 0, np.floor(b + np.float32(0.5)), np.ceil(b - np.float32(0.5)))
    q[:, 1:] = (s * np.floor(p[:, 1:] / s)).astype(np.int64)
    return q


def insert(q):
    """(unique rows in first-occurrence order, unique_index [M], inverse [N])."""
    _, first, inv = np.unique(q, axis=0, return_index=True, return_inverse=True)
    order = np.argsort(first, kind="stable")
    rank = np.empty_like(order)
    rank[order] = np.arange(len(order))
    return q[first[order]], first[order], rank[inv.reshape(-1)]


def reduce(feats, inv, M, mode):
    """(out [M, C] float64, argmax [M, C] point index or -1 for MAX)."""
    x = np.asarray(feats, np.float64)
    C = x.shape[1]
    out = np.zeros((M, C))
    arg = np.full((M, C), -1, np.int64)
    valid = inv >= 0
    if mode in (SUM, AVG):
        np.add.at(out, inv[valid], x[valid])
        if mode == AVG:
            cnt = np.bincount(inv[valid], minlength=M)
            out[cnt > 0] /= cnt[cnt > 0, None]
    elif mode == MAX:
        for i in np.nonzero(valid)[0]:          # field order: the first point wins a tie
            r = inv[i]
            upd = (arg[r] < 0) | (x[i] > out[r])
            out[r, upd] = x[i, upd]
            arg[r, upd] = i
    else:
        first = np.full(M, -1, np.int64)
        for i in np.nonzero(valid)[0][::-1]:
            first[inv[i]] = i
        out[first >= 0] = x[first[first >= 0]]
    return out, arg


def reduce_backward(grad_out, feats, inv, M, mode):
    """Gradient of reduce() with respect to the point features."""
    g = np.asarray(grad_out, np.float64)
    N = len(inv)
    valid = inv >= 0
    grad = np.zeros((N, g.shape[1]))
    if mode == SUM:
        grad[valid] = g[inv[valid]]
    elif mode == AVG:
        cnt = np.bincount(inv[valid], minlength=M)
        grad[valid] = g[inv[valid]] / cnt[inv[valid], None]
    elif mode == MAX:
        _, arg = reduce(feats, inv, M, MAX)
        rows = np.arange(N)
        for i in np.nonzero(valid)[0]:
            hit = arg[inv[i]] == rows[i]
            grad[i, hit] = g[inv[i], hit]
    else:
        first = np.full(M, -1, np.int64)
        for i in np.nonzero(valid)[0][::-1]:
            first[inv[i]] = i
        keep = valid & (first[np.maximum(inv, 0)] == np.arange(N))
        grad[keep] = g[inv[keep]]
    return grad


def slice_forward(F, inv):
    F = np.asarray(F, np.float64)
    out = np.zeros((len(inv), F.shape[1]))
    out[inv >= 0] = F[inv[inv >= 0]]
    return out


def slice_backward(grad_out, inv, M):
    return reduce(grad_out, inv, M, SUM)[0]


def find(map_coords, q):
    """Row of every query row in map_coords (-1 where absent)."""
    index = {tuple(r): i for i, r in enumerate(np.asarray(map_coords).tolist())}
    return np.array([index.get(tuple(r), -1) for r in np.asarray(q).tolist()], np.int64)


def interp_map(query, map_coords, stride):
    """(rows [N, 2^D], weights fp32 [N, 2^D]); bit D-j of corner k selects the upper end of axis
    j; weights prod_j (1 - |x_j - c_j| / s) in float32, 0 where the corner is absent."""
    q = np.asarray(query, np.float32)
    N, ncols = q.shape
    D = ncols - 1
    K = 1 << D
    s = np.float32(stride)
    lower = quantize(q, stride)
    rows = np.empty((N, K), np.int64)
    w = np.zeros((N, K), np.float32)
    index = {tuple(r): i for i, r in enumerate(np.asarray(map_coords).tolist())}
    for k in range(K):
        c = lower.copy()
        for j in range(1, ncols):
            if (k >> (D - j)) & 1:
                c[:, j] += int(stride)
        rows[:, k] = [index.get(tuple(r), -1) for r in c.tolist()]
        wk = np.ones(N, np.float32)
        for j in range(1, ncols):
            wk = wk * (np.float32(1) - np.abs(q[:, j] - c[:, j].astype(np.float32)) / s)
        w[:, k] = np.where(rows[:, k] >= 0, wk, np.float32(0))
    return rows, w


def interp_forward(F, rows, w):
    F = np.asarray(F, np.float64)
    out = np.zeros((rows.shape[0], F.shape[1]))
    for k in range(rows.shape[1]):
        hit = rows[:, k] >= 0
        out[hit] += w[hit, k, None].astype(np.float64) * F[rows[hit, k]]
    return out


def interp_backward(grad_out, rows, w, M):
    g = np.asarray(grad_out, np.float64)
    grad = np.zeros((M, g.shape[1]))
    for k in range(rows.shape[1]):
        hit = rows[:, k] >= 0
        np.add.at(grad, rows[hit, k], w[hit, k, None].astype(np.float64) * g[hit])
    return grad


def canon(coords):
    return np.lexsort(np.asarray(coords).T[::-1])
