"""TEST INFRASTRUCTURE — float64 restatement of the reference's channel-wise convolution
(MinkowskiEngine/MinkowskiChannelwiseConvolution.py:142-191: out[o] += in[i] * kernel[k] for every
pair (i, o) of offset k, backward by autograd) over k-major neighbour tables.  Pinned against the
compiled reference's fixtures tests/golden/ref_chwise_* (tests/test_chwise_cpu.py), written by
tests/golden/make_chwise_fixtures.py.

Every function takes numpy arrays or torch tensors (any device) and computes in float64.  Next to
each result it returns A, the same reduction over absolute values: the scale of the fp32
accumulation error, for helpers.assert_one_rounding."""
import numpy as np


def _is_np(a):
    return isinstance(a, np.ndarray)


def _f64(a):
    return np.asarray(a, np.float64) if _is_np(a) else a.double()


def _zeros(like, shape):
    if _is_np(like):
        return np.zeros(shape, np.float64)
    import torch
    return torch.zeros(shape, dtype=torch.float64, device=like.device)


def tables(in_maps, out_maps, n_in, n_out):
    """(out_nbr [K, n_out], in_nbr [K, n_in]) int32 from per-offset pair lists: out_nbr[k, o] = i
    and in_nbr[k, i] = o for every pair (i, o) of offset k, -1 elsewhere."""
    K = len(in_maps)
    out_nbr = np.full((K, n_out), -1, np.int32)
    in_nbr = np.full((K, n_in), -1, np.int32)
    for k, (i, o) in enumerate(zip(in_maps, out_maps)):
        out_nbr[k, np.asarray(o)] = np.asarray(i)
        in_nbr[k, np.asarray(i)] = np.asarray(o)
    return out_nbr, in_nbr


def gather(x, W, nbr):
    """y[r, c] = sum_k W[k, c] * x[nbr[k, r], c] over the entries nbr[k, r] >= 0 (a row appears
    once per offset).  The forward (nbr = out_nbr) and the input gradient (x = the output gradient,
    nbr = in_nbr).  Returns (y, A) [n_rows, C]."""
    x, W = _f64(x), _f64(W)
    K, n_rows = nbr.shape
    y = _zeros(x, (n_rows, x.shape[1]))
    A = _zeros(x, (n_rows, x.shape[1]))
    for k in range(K):
        hit = nbr[k] >= 0
        src = x[nbr[k][hit].astype(np.int64) if _is_np(nbr) else nbr[k][hit].long()]
        y[hit] += src * W[k]
        A[hit] += abs(src) * abs(W[k])
    return y, A


def wgrad(x, g, out_nbr):
    """dW[k, c] = sum_o x[out_nbr[k, o], c] * g[o, c].  Returns (dW, A) [K, C]."""
    x, g = _f64(x), _f64(g)
    K = out_nbr.shape[0]
    dW = _zeros(x, (K, x.shape[1]))
    A = _zeros(x, (K, x.shape[1]))
    for k in range(K):
        hit = out_nbr[k] >= 0
        src = x[out_nbr[k][hit].astype(np.int64) if _is_np(out_nbr) else out_nbr[k][hit].long()]
        dW[k] = (src * g[hit]).sum(0)
        A[k] = (abs(src) * abs(g[hit])).sum(0)
    return dW, A


def forward(in_feat, kernel, in_maps, out_maps, n_out, bias=None):
    """The layer's output in float64 (bias added when given)."""
    out_nbr, _ = tables(in_maps, out_maps, len(in_feat), n_out)
    y, _ = gather(in_feat, kernel, out_nbr)
    return y if bias is None else y + np.asarray(bias, np.float64).reshape(1, -1)


def backward(in_feat, grad_out, kernel, in_maps, out_maps):
    """(grad_in, grad_kernel) in float64."""
    out_nbr, in_nbr = tables(in_maps, out_maps, len(in_feat), len(grad_out))
    grad_in, _ = gather(grad_out, kernel, in_nbr)
    grad_kernel, _ = wgrad(in_feat, grad_out, out_nbr)
    return grad_in, grad_kernel
