"""Shared test helpers: seeded inputs, oracle-side evaluation of one layer, stored results of the
compiled reference (tests/golden/)."""
import hashlib
import os

import numpy as np
import torch

from oracle import oracle_np as O


def random_cloud(n, extent, seed, D=3, batches=1, allow_negative=False):
    g = torch.Generator().manual_seed(seed)
    lo = -extent if allow_negative else 0
    c = torch.randint(lo, extent, (n, D), generator=g, dtype=torch.int32)
    b = torch.randint(0, batches, (n, 1), generator=g, dtype=torch.int32)
    return torch.cat([b, c], 1)


def unique_cloud(n, extent, seed, D=3, batches=1, allow_negative=False):
    c = random_cloud(n, extent, seed, D, batches, allow_negative)
    return torch.unique(c, dim=0)[torch.randperm(
        len(torch.unique(c, dim=0)), generator=torch.Generator().manual_seed(seed + 1))]


def kmap_lists(kdict, K):
    """{k: IntTensor[2,n]} -> (in_maps, out_maps) numpy lists of length K."""
    im, om = [], []
    for k in range(K):
        if k in kdict:
            t = kdict[k].cpu().numpy().astype(np.int64)
            im.append(t[0]); om.append(t[1])
        else:
            im.append(np.zeros(0, np.int64)); om.append(np.zeros(0, np.int64))
    return im, om


def oracle_conv_layer(in_coords, tensor_stride, kernel_size, stride, dilation, transposed=False,
                      out_coords=None, region_type=O.HYPER_CUBE):
    """Oracle-side coordinate + kernel-map construction of one (transposed) conv layer.
    Returns (out_coords canonical, in_maps, out_maps)."""
    D = in_coords.shape[1] - 1
    ks, st, dl = [kernel_size] * D, [stride] * D, [dilation] * D
    if not transposed:
        if out_coords is None:
            out_coords, _ = O.stride_map_coords(in_coords, tensor_stride, st)
        offs = O.region_offsets(region_type, ks, dl, tensor_stride)
        im, om = O.kernel_map(in_coords, out_coords, offs)
    else:
        out_ts = [t // s for t, s in zip(tensor_stride, st)]
        assert out_coords is not None
        offs = O.region_offsets(region_type, ks, dl, out_ts)
        im, om = O.transposed_kernel_map(in_coords, out_coords, offs)
    return out_coords, im, om


def layer_out_ts(meta):
    """The output tensor stride of a layer fixture (tests/golden/ref_layer_*.npz), but for one
    deliberate difference: the reference's convolution passes `expand_coordinates` to
    `_get_coordinate_map_key` in the place of its `tensor_stride` argument
    (MinkowskiConvolution.py:311-313), so output coordinates given as a tensor are inserted at
    tensor stride 0 there.  This package inserts them at tensor stride 1, the default of that
    argument; the map and the features are the same."""
    if meta["given"] == "tensor":
        assert meta["out_ts"] == [0] * meta["D"]
        return [1] * meta["D"]
    return meta["out_ts"]


def rel_err(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def one_rounding_bound(ref, A, dtype, acc=1.0):
    """Per-element bound for a reduction accumulated in fp32 and stored in `dtype`, against its
    float64 value `ref`: delta = acc * 2^-20 * A, A the same reduction over absolute values, plus
    half an ulp of `dtype` at |ref| + delta when the result is stored in bf16 / fp16 (one
    rounding).  `acc` = 1 for the CUDA-core kernels; the wgmma kernels use TC_ACC."""
    ref, A = ref.double(), A.double()
    delta = A * (acc * 2.0 ** -20)
    if dtype == torch.float32:
        return delta
    return half_ulp(ref.abs() + delta, dtype) + delta


def half_ulp(v, dtype):
    """Half an ulp of bf16 / fp16 at the magnitudes `v` (float64, >= 0): the largest error of one
    rounding to `dtype` of a value of magnitude at most v."""
    p, emin = {torch.bfloat16: (7, -126), torch.float16: (10, -14)}[dtype]
    _, e = torch.frexp(v)                        # v = m * 2^e, m in [0.5, 1)
    e = torch.where(v > 0, e - 1, torch.full_like(e, emin)).clamp(min=emin)
    return torch.ldexp(torch.full_like(v, 0.5), e - p)


# The wgmma kernels' fp32 accumulation of bf16 / fp16 products is less accurate than the CUDA
# cores' fma chain, and its error grows with the reduction length (about as its square root), as
# a truncating accumulation does.  Measured on an H100 80GB HBM3 (700 W), worst |err| / (2^-20 A)
# over all elements: forward 1.54 and dgrad 1.48 (256 -> 256, K = 125, ~29k products per element),
# a one-split pair-list wgrad 2.00 (70k pairs per offset); the CUDA-core forward on the same
# values 0.24.  The excess is spread over every row and column position of the tiles: every
# position of a 128-row tile and of a 64-column block reaches at least 0.8 of the worst.
# These figures are of zero-mean operands, whose truncation losses cancel; TC_ACC holds only for
# them.  On one-signed operands (ReLU outputs times gradients of one sign) the losses add up, and
# the error grows with the number of wgmma steps one accumulator takes: WG_STEP below.
TC_ACC = 4.0

# The tensor-core wgrad on one-signed operands: |err| <= WG_STEP * steps * 2^-24 * A, steps = the
# 16-pair wgmma steps of the CTA's share (tests/test_gpu_wgrad_accumulation.py).  Measured on an
# H100 80GB HBM3 (700 W) on all-positive operands, one share of 256 to 16384 steps: worst
# |err| / (steps 2^-24 A) 0.82 - 1.54 in bf16 and 1.59 - 1.63 in fp16, about an ulp and a half of
# the running sum lost per step; WG_STEP is about twice the worst, as TC_ACC is.
WG_STEP = 3.5


def assert_one_rounding(y, ref, A, what="", acc=1.0):
    """|y - ref| <= one_rounding_bound(ref, A, y.dtype, acc), element by element."""
    bound = one_rounding_bound(ref, A, y.dtype, acc)
    err = (y.double() - ref.double()).abs()
    bad = ~(err <= bound)
    if bool(bad.any()):
        j = int(torch.nonzero(bad.flatten())[0])
        raise AssertionError(
            f"{what}: {int(bad.sum())} of {bad.numel()} elements outside one rounding; first at "
            f"flat index {j}: got {y.flatten()[j].item()!r}, float64 {ref.flatten()[j].item()!r}, "
            f"|err| {err.flatten()[j].item():.3e} > bound {bound.flatten()[j].item():.3e}")


def one_rounding_ratio(y, ref, A, acc=1.0):
    """max |y - ref| / one_rounding_bound(ref, A, y.dtype, acc) over the elements with a nonzero
    bound: how close the error comes to the bound (at most 1 passes)."""
    err = (y.double() - ref.double()).abs()
    bound = one_rounding_bound(ref, A, y.dtype, acc)
    m = bound > 0
    return float((err[m] / bound[m]).max()) if bool(m.any()) else 0.0


# ---- convolution layers on random neighbour tables, and their float64 restatement --------------
def _table(K, n_rows, n_other, density, seed, device):
    """Random k-major neighbour table [K, n_rows] with fully empty rows and an all-empty offset."""
    g = torch.Generator().manual_seed(seed)
    idx = torch.randint(0, n_other, (K, n_rows), generator=g, dtype=torch.int32)
    idx[torch.rand((K, n_rows), generator=g) > density] = -1
    idx[:, ::97] = -1                     # rows without any neighbour
    if K > 1:
        idx[K // 2] = -1                  # an offset without any pair
    return idx.to(device)


def _pairs(nbr):
    """[(rows of the other side, table rows)] per offset of a k-major table."""
    out = []
    for k in range(nbr.shape[0]):
        o = torch.nonzero(nbr[k] >= 0).flatten()
        out.append((nbr[k][o].long(), o))
    return out


def ref_conv(x, w, pairs, n_out):
    """float64 y[o] = sum over offsets k and pairs (i, o) of x[i] @ w[k]; and the same reduction
    over |x| and |w| (the scale of the accumulation error)."""
    x, w = x.double(), w.double()
    y = torch.zeros((n_out, w.shape[2]), dtype=torch.float64, device=x.device)
    A = torch.zeros_like(y)
    for k, (i, o) in enumerate(pairs):
        if len(i):
            y.index_add_(0, o, x[i] @ w[k])
            A.index_add_(0, o, x[i].abs() @ w[k].abs())
    return y, A


def ref_wgrad(x, g, pairs):
    """float64 dW[k] = sum over pairs (i, o) of x[i]^T g[o], and over |x|, |g|."""
    x, g = x.double(), g.double()
    K = len(pairs)
    gw = torch.zeros((K, x.shape[1], g.shape[1]), dtype=torch.float64, device=x.device)
    A = torch.zeros_like(gw)
    for k, (i, o) in enumerate(pairs):
        if len(i):
            gw[k] = x[i].t() @ g[o]
            A[k] = x[i].abs().t() @ g[o].abs()
    return gw, A


def _inputs(cin, cout, n_in, n_out, K, dtype, device, seed):
    g = torch.Generator().manual_seed(seed)
    feats = (torch.rand(n_in, cin, generator=g) - 0.5).to(dtype).to(device)
    gout = (torch.rand(n_out, cout, generator=g) - 0.5).to(dtype).to(device)
    w = ((torch.rand(K, cin, cout, generator=g) - 0.5) / (cin ** 0.5)).to(device)  # fp32 master
    return feats, gout, w


class _Route:
    """Counts tensor-core launches over a block and checks the route the case is meant to take."""

    def __init__(self, tc, what):
        self.tc, self.what = tc, what

    def __enter__(self):
        from minkowskiengine_b200 import _lib
        self.n0 = _lib.tc_launch_count()
        return self

    def __exit__(self, *exc):
        from minkowskiengine_b200 import _lib
        if exc[0] is None:
            n = _lib.tc_launch_count() - self.n0
            assert (n > 0) == self.tc, \
                f"{self.what}: {n} tensor-core launches, expected {'some' if self.tc else 'none'}"


def lib_conv_backward(feats, gout, w, km, grad_in_dtype=None, need_w=False, pairs=False,
                      workspace=None, grad_w=None):
    """One `meb200_conv_backward` call with the caller's choices, which `backend` makes itself:
    the dtype of grad_in (None: no dgrad; fp32 gives the accumulator before any rounding), the
    pair-list or the dense-table wgrad, and the workspace, given as a uint8 tensor (its size, or
    None for no workspace).  `grad_w`: the fp32 tensor the wgrad writes (default: a new one).
    Returns (grad_in, grad_w)."""
    from minkowskiengine_b200 import _lib, backend
    lib = _lib.load()
    dt = feats.dtype
    code = _lib.dtype_code(dt)
    K, c_in, c_out = w.shape
    w_cast, _ = backend._feature_weights(w, dt)
    gi = None if grad_in_dtype is None else \
        torch.empty((km.n_in, c_in), dtype=grad_in_dtype, device=feats.device)
    gw = None
    if need_w:
        gw = grad_w if grad_w is not None else \
            torch.empty((K, c_in, c_out), dtype=torch.float32, device=feats.device)
    pin = pout = seg = None
    nch = 0
    if pairs:
        pin, pout, seg, nch = km.pair_lists()
    _lib.check(lib.meb200_conv_backward(
        _lib.ptr(feats), _lib.ptr(gout), code, km.n_in, c_in, _lib.ptr(w_cast), K, c_out,
        _lib.ptr(km.out_nbr), _lib.ptr(km.in_nbr) if gi is not None else None, km.n_out,
        _lib.ptr(gi), _lib.dtype_code(grad_in_dtype or dt), _lib.ptr(gw), _lib.ptr(pin),
        _lib.ptr(pout), _lib.ptr(seg), nch, _lib.ptr(workspace),
        0 if workspace is None else workspace.numel(), _lib.current_stream()))
    return gi, gw


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def golden(name):
    """A results file of the compiled reference (written by tests/golden/make_reference_runs.py)."""
    return np.load(os.path.join(GOLDEN, name))


def digest(t):
    """SHA-256 of a tensor's values in a fixed dtype per kind (int -> int64, float -> float32)."""
    a = np.ascontiguousarray(np.asarray(t.detach().cpu() if torch.is_tensor(t) else t))
    a = a.astype(np.int64) if a.dtype.kind in "iub" else a.astype(np.float32)
    return np.frombuffer(hashlib.sha256(a.tobytes() + str(a.shape).encode()).digest(), np.uint8)


def state_digest(module):
    """Digest of a module's state_dict (parameters and buffers, in key order)."""
    h = hashlib.sha256()
    for k, v in module.state_dict().items():
        h.update(k.encode())
        h.update(digest(v).tobytes())
    return np.frombuffer(h.digest(), np.uint8)
