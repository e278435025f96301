"""TEST INFRASTRUCTURE — numpy restatement of the reference's global pooling, broadcast and
instance normalisation over the origin map (reference paths relative to the reference tree, as in
oracle/oracle_np.py).  Pinned against the compiled reference's fixtures tests/golden/ref_global_*,
ref_broadcast_*, ref_instnorm (tests/test_global_cpu.py); those are written by
tests/golden/make_global_fixtures.py."""
import numpy as np

from oracle.oracle_np import POOL_AVG, POOL_MAX, POOL_SUM  # noqa: F401  (re-exported)


def origin_segments(coords):
    """The origin map (coordinate_map_cpu.hpp:492-513: one row (b, 0, ..., 0) per batch index)
    with its rows in ascending batch order, and origin_map (:724-783): the origin row of every
    input row.  Returns (origin_coords [B, D+1], row_seg [n])."""
    coords = np.asarray(coords)
    batches, row_seg = np.unique(coords[:, 0], return_inverse=True)
    origin = np.zeros((len(batches), coords.shape[1]), np.int32)
    origin[:, 0] = batches
    return origin, row_seg.reshape(-1).astype(np.int64)


def global_pool_forward(in_feat, row_seg, B, mode):
    """GlobalPoolingForwardCPU (src/global_pooling_cpu.cpp:43-200) with the _KERNEL modes:
    NonzeroAvgPoolingForwardKernelCPU / MaxPoolingForwardKernelCPU over the origin map
    (pooling_avg_kernel.hpp:40-101, pooling_max_kernel.hpp:35-90; rows visited in ascending
    order, strict '<' => the lowest row wins a tie).  Returns (out [B, C], aux): aux = row counts
    (sum / avg) or max_index int32 [B, C] = row*C + c (max).  An empty cloud gives 0 (index -1)."""
    x = np.asarray(in_feat, np.float64)
    n, C = x.shape
    if mode == POOL_MAX:
        out = np.zeros((B, C), np.float64)
        idx = np.full((B, C), -1, np.int64)
        for s in range(B):
            rows = np.nonzero(row_seg == s)[0]
            if len(rows):
                arg = np.argmax(x[rows], axis=0)          # first maximum = lowest row
                out[s] = x[rows[arg], np.arange(C)]
                idx[s] = rows[arg] * C + np.arange(C)
        return out, idx.astype(np.int32)
    out = np.zeros((B, C), np.float64)
    np.add.at(out, row_seg, x)
    cnt = np.bincount(row_seg, minlength=B).astype(np.float64)
    if mode == POOL_AVG:
        out /= np.maximum(cnt, 1)[:, None]
    return out, cnt


def global_pool_backward(grad_out, row_seg, n, mode, aux):
    """GlobalPoolingBackwardCPU (src/global_pooling_cpu.cpp:221-330): sum / avg copy the cloud's
    gradient (divided by its row count) to every row; max sends it to the row of the maximum
    (pooling_max_kernel.hpp:92-115)."""
    g = np.asarray(grad_out, np.float64)
    C = g.shape[1]
    if mode == POOL_MAX:
        grad_in = np.zeros((n, C), np.float64).reshape(-1)
        m = np.asarray(aux).reshape(-1)
        ok = m >= 0
        np.add.at(grad_in, m[ok], g.reshape(-1)[ok])
        return grad_in.reshape(n, C)
    if mode == POOL_AVG:
        g = g / np.maximum(np.asarray(aux, np.float64), 1)[:, None]
    return g[row_seg]


BCAST_ADD, BCAST_MUL = 0, 1


def broadcast_forward(x, g, row_seg, op):
    """BroadcastForwardKernelCPU (src/broadcast_kernel.hpp): y[i] = x[i] + / * g[origin row of i]."""
    x, g = np.asarray(x, np.float64), np.asarray(g, np.float64)
    return x + g[row_seg] if op == BCAST_ADD else x * g[row_seg]


def broadcast_backward(x, g, grad_out, row_seg, op):
    """BroadcastBackwardKernelCPU (src/broadcast_kernel.hpp): add: dx = dy, dg[b] = sum dy;
    mul: dx = dy * g[b(i)], dg[b] = sum dy * x."""
    x, g, dy = (np.asarray(a, np.float64) for a in (x, g, grad_out))
    dg = np.zeros_like(g)
    if op == BCAST_ADD:
        np.add.at(dg, row_seg, dy)
        return dy.copy(), dg
    np.add.at(dg, row_seg, dy * x)
    return dy * g[row_seg], dg


def instance_norm_forward(x, row_seg, B, eps=1e-8):
    """MinkowskiInstanceNormFunction.forward (MinkowskiNormalization.py:194-252): mean, centre,
    mean of squares, scale by 1/sqrt(var + 1e-8).  Returns (y, inv_std [B, C])."""
    mean, _ = global_pool_forward(x, row_seg, B, POOL_AVG)
    c = np.asarray(x, np.float64) - mean[row_seg]
    var, _ = global_pool_forward(c * c, row_seg, B, POOL_AVG)
    inv_std = 1.0 / np.sqrt(var + eps)
    return c * inv_std[row_seg], inv_std


def instance_norm_backward(grad_out, y, inv_std, row_seg, B):
    """MinkowskiInstanceNormFunction.backward (MinkowskiNormalization.py:254-310):
    dx = (dy - y * avg(dy * y) - avg(dy)) * inv_std."""
    dy = np.asarray(grad_out, np.float64)
    y = np.asarray(y, np.float64)
    md, _ = global_pool_forward(dy, row_seg, B, POOL_AVG)
    mdy, _ = global_pool_forward(dy * y, row_seg, B, POOL_AVG)
    return (dy - y * mdy[row_seg] - md[row_seg]) * inv_std[row_seg]
