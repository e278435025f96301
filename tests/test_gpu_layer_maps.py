"""Coordinate maps, kernel maps and convolutions of the CUDA path against the compiled reference,
one layer per fixture (tests/golden/ref_layer_*.npz, written by tests/golden/make_layer_fixtures.py;
their oracle side is tests/test_layer_maps_cpu.py), through the public API:

- coordinates: the insert's `unique_index` / `inverse_map` bit-exact, the stride-3 (or stride-4)
  map and the layer's output coordinates and tensor stride equal as sets;
- kernel map: equal to the reference's (k, in coordinate, out coordinate) triples, and `in_nbr`
  exactly the transpose of `out_nbr` (after the deferred build where K >= LAZY_REVERSE_K);
- features and gradients: fp32 within 1e-5 relative of the reference, and fp32, bf16 and fp16
  element by element within `one_rounding_bound` of a float64 restatement whose pairs come from
  the FIXTURE's triples, mapped to this package's rows by coordinate — so a wrong map cannot hide
  behind a restatement built on the same map.  The bound takes TC_ACC where the tensor-core launch
  counter shows a wgmma kernel ran; fp32 is pinned to "ieee" (CUDA cores);
- repeats: a second run gives bit-identical features and gradients."""
import glob
import json
import os

import numpy as np
import pytest
import torch

from helpers import TC_ACC, assert_one_rounding, kmap_lists, layer_out_ts, ref_conv, ref_wgrad
from oracle import oracle_np as O

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
FIXTURES = sorted(glob.glob(os.path.join(GOLD, "ref_layer_*.npz")))
CONV = [p for p in FIXTURES if json.loads(str(np.load(p)["meta"]))["kind"] != "pool"]
POOL = [p for p in FIXTURES if p not in CONV]
DTYPES = [torch.float32, torch.bfloat16, torch.float16]


def _id(path):
    return os.path.basename(path)[len("ref_layer_"):-len(".npz")]


@pytest.fixture(autouse=True)
def exact_fp32():
    saved = torch.backends.cuda.matmul.fp32_precision
    torch.backends.cuda.matmul.fp32_precision = "ieee"
    yield
    torch.backends.cuda.matmul.fp32_precision = saved


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30)) if b.size else 0.0


def _rows(coords, query):
    """Rows of `coords` holding each query coordinate (all must be found)."""
    r = O.RowIndex(coords).find(np.asarray(query, np.int32))
    assert (r >= 0).all(), "a fixture coordinate is missing from the map"
    return r


def _tc():
    from minkowskiengine_b200 import _lib
    return _lib.tc_launch_count()


class Layer:
    """The fixture's layer on CUDA: its input map (inserted, then strided by `pre_stride`), the
    input rows of the fixture in this package's row order, and the layer module."""

    def __init__(self, ME, f, m, cuda):
        self.ME, self.f, self.m, self.cuda = ME, f, m, cuda
        D = m["D"]
        self.cm = ME.CoordinateManager(D=D)
        raw = torch.from_numpy(f["raw_coords"]).to(cuda)
        self.key0, (self.uidx, self.inv) = self.cm.insert_and_map(raw, m["ts_in"])
        self.in_key = self.key0 if m["pre_stride"] is None else \
            self.cm.stride(self.key0, m["pre_stride"])
        self.in_c = self.cm.get_coordinates(self.in_key).cpu().numpy()
        self.in_rows = _rows(f["in_coords"], self.in_c)    # fixture row of each of our rows
        rt = {"cube": ME.RegionType.HYPER_CUBE, "cross": ME.RegionType.HYPER_CROSS}[m["region"]]
        self.rt = rt
        kg = ME.KernelGenerator(kernel_size=m["kernel_size"], stride=m["stride"],
                                dilation=m["dilation"], region_type=rt,
                                expand_coordinates=m["kind"] == "generative" or
                                m["given"] == "expand", dimension=D)
        if m["kind"] == "pool":
            self.layer = None
        else:
            cls = {"conv": ME.MinkowskiConvolution,
                   "transpose": ME.MinkowskiConvolutionTranspose,
                   "generative": ME.MinkowskiGenerativeConvolutionTranspose}[m["kind"]]
            kw = {"expand_coordinates": True} if m["given"] == "expand" else {}
            self.layer = cls(m["cin"], m["cout"], kernel_generator=kg, dimension=D, **kw).to(cuda)
            with torch.no_grad():
                self.layer.kernel.copy_(torch.from_numpy(f["weight"]))
        self.given_key = None
        if m["given"] == "key":
            gc = torch.from_numpy(f["given_coords"]).to(cuda)
            self.given_key = self.cm.insert_and_map(gc, 1, "given")[0]

    def input(self, dtype, requires_grad):
        x = torch.from_numpy(self.f["in_feats"][self.in_rows]).to(self.cuda, dtype)
        x.requires_grad_(requires_grad)
        return x, self.ME.SparseTensor(x, coordinate_map_key=self.in_key,
                                       coordinate_manager=self.cm)

    def __call__(self, st):
        g = self.m["given"]
        if g == "tensor":
            return self.layer(st, torch.from_numpy(self.f["given_coords"]).to(self.cuda))
        if g == "key":
            return self.layer(st, self.given_key)
        return self.layer(st)

    def kernel_map(self, out_key, is_pool=False):
        m = self.m
        args = (self.in_key, out_key, m["kernel_size"], m["stride"], m["dilation"], self.rt,
                torch.IntTensor(), m["kind"] in ("transpose", "generative"), is_pool)
        return self.cm._manager._kernel_map(*args)

    def pairs(self, out_c):
        """Per offset (our input rows, our output rows) of the FIXTURE's kernel map."""
        t = self.f["kmap"].astype(np.int64)
        nc = self.m["D"] + 1
        i = _rows(self.in_c, t[:, 1:1 + nc])
        o = _rows(out_c, t[:, 1 + nc:])
        out = []
        for k in range(self.m["K"]):
            s = t[:, 0] == k
            out.append((torch.from_numpy(i[s]).to(self.cuda), torch.from_numpy(o[s]).to(self.cuda)))
        return out


def _check_coordinates(L, y):
    f, m = L.f, L.m
    assert list(y.tensor_stride) == layer_out_ts(m)
    out_c = y.C.cpu().numpy()
    oc, _, _ = O.canonical_rows(out_c)
    assert oc.shape == f["out_coords"].shape and np.array_equal(oc, f["out_coords"])
    return out_c


def _check_kernel_map(L, y, out_c, is_pool=False):
    m = L.m
    kd = L.cm.kernel_map(L.in_key, y.coordinate_map_key, stride=m["stride"],
                         kernel_size=m["kernel_size"], dilation=m["dilation"],
                         region_type=L.rt, is_transpose=m["kind"] in ("transpose", "generative"),
                         is_pool=is_pool)
    K = 1 if is_pool and m["kernel_size"] == m["stride"] else m["K"]   # a stride map: one group
    tri = O.kernel_map_triples(L.in_c, out_c, *kmap_lists(kd, K))
    assert tri.shape == L.f["kmap"].shape and np.array_equal(tri, L.f["kmap"])
    return L.kernel_map(y.coordinate_map_key, is_pool)


def _check_transpose(km):
    """in_nbr[k, i] == o exactly where out_nbr[k, o] == i."""
    out_nbr, in_nbr = km.out_nbr.long(), km.in_nbr.long()
    exp = torch.full(in_nbr.shape, -1, dtype=torch.long, device=out_nbr.device)
    kk, oo = torch.nonzero(out_nbr >= 0, as_tuple=True)
    exp[kk, out_nbr[kk, oo]] = oo
    assert torch.equal(exp, in_nbr), "in_nbr is not the transpose of out_nbr"


@pytest.mark.parametrize("path", FIXTURES, ids=_id)
def test_insert_and_stride_maps(ME, cuda, path):
    f = np.load(path)
    m = json.loads(str(f["meta"]))
    L = Layer(ME, f, m, cuda)
    assert np.array_equal(L.uidx.cpu().numpy(), f["unique_index"])
    assert np.array_equal(L.inv.cpu().numpy(), f["inverse_map"])
    assert np.array_equal(L.cm.get_coordinates(L.key0).cpu().numpy(),
                          f["raw_coords"][f["unique_index"]])
    assert np.array_equal(O.canonical_rows(L.in_c)[0], f["in_coords"])
    if m["extra_stride"] is not None:
        sk = L.cm.stride(L.key0, m["extra_stride"])
        sc = L.cm.get_coordinates(sk).cpu().numpy()
        assert np.array_equal(O.canonical_rows(sc)[0], f["xs_coords"])
        i, o = L.cm.stride_map(L.key0, sk)
        c0 = L.cm.get_coordinates(L.key0).cpu().numpy()
        pairs = O.kernel_map_triples(c0, sc, [i.cpu().numpy()], [o.cpu().numpy()])[:, 1:]
        assert np.array_equal(pairs, f["xs_pairs"])


@pytest.mark.parametrize("dtype", DTYPES, ids=["fp32", "bf16", "fp16"])
@pytest.mark.parametrize("path", CONV, ids=_id)
def test_conv_layer(ME, cuda, path, dtype):
    f = np.load(path)
    m = json.loads(str(f["meta"]))
    L = Layer(ME, f, m, cuda)
    what = f"{_id(path)} {dtype}"
    w = L.layer.kernel
    # forward and dgrad (the kernel takes no gradient, so the backward runs the dgrad alone)
    w.requires_grad_(False)
    x, st = L.input(dtype, True)
    n0 = _tc()
    y = L(st)
    fwd_acc = TC_ACC if _tc() > n0 else 1.0
    out_c = _check_coordinates(L, y)
    km = _check_kernel_map(L, y, out_c)
    lazy = m["kind"] == "conv" and m["K"] >= L.cm._manager.LAZY_REVERSE_K
    assert (km._in_nbr is None) == lazy, "reverse table built eagerly or not at all"
    out_rows = _rows(out_c, f["out_coords"])              # our row of each fixture row
    gout = torch.empty((len(out_c), m["cout"]), dtype=dtype, device=cuda)
    gout[torch.from_numpy(out_rows).to(cuda)] = torch.from_numpy(f["grad_out"]).to(cuda, dtype)
    n0 = _tc()
    y.F.backward(gout)
    dgrad_acc = TC_ACC if _tc() > n0 else 1.0
    _check_transpose(km)                                   # (deferred build done by the dgrad)

    pairs = L.pairs(out_c)
    wl = w.detach().to(dtype)
    y_ref, y_A = ref_conv(x.detach(), wl, pairs, len(out_c))
    assert_one_rounding(y.F.detach(), y_ref, y_A, f"{what} forward", fwd_acc)
    gi_ref, gi_A = ref_conv(gout, wl.transpose(1, 2), [(o, i) for i, o in pairs], len(L.in_c))
    assert_one_rounding(x.grad, gi_ref, gi_A, f"{what} dgrad", dgrad_acc)
    if dtype == torch.float32:
        assert _rel(y.F.detach().cpu().numpy()[out_rows], f["out_feats"]) < 1e-5
        assert _rel(x.grad.cpu().numpy(), f["grad_in"][L.in_rows]) < 1e-5

    # weight gradient alone
    w.requires_grad_(True)
    x2, st2 = L.input(dtype, False)
    y2 = L(st2)
    assert torch.equal(y2.F.detach(), y.F.detach()), f"{what}: forward differs run to run"
    n0 = _tc()
    y2.F.backward(gout)
    wgrad_acc = TC_ACC if _tc() > n0 else 1.0
    gw = w.grad.clone()
    gw_ref, gw_A = ref_wgrad(x2, gout, pairs)
    assert_one_rounding(gw, gw_ref, gw_A, f"{what} wgrad", wgrad_acc)
    if dtype == torch.float32:
        assert _rel(gw.cpu().numpy(), f["grad_weight"]) < 1e-5

    # repeats: dgrad and wgrad again, bit for bit
    w.grad = None
    x3, st3 = L.input(dtype, True)
    L(st3).F.backward(gout)
    assert torch.equal(x3.grad, x.grad), f"{what}: dgrad differs run to run"
    assert torch.equal(w.grad, gw), f"{what}: wgrad differs run to run"


@pytest.mark.parametrize("mode", ["max", "avg"])
@pytest.mark.parametrize("path", POOL, ids=_id)
def test_pool_layer(ME, cuda, path, mode):
    """Both pooling modes on both maps (a pooling map does not depend on the mode); the mode the
    reference ran is also compared with its outputs.  The dilated window at a strided input holds
    no input for some output rows: those hold the lowest finite value (max) or zero (avg), and
    pass no gradient back."""
    f = np.load(path)
    m = json.loads(str(f["meta"]))
    L = Layer(ME, f, m, cuda)
    cls = {"max": ME.MinkowskiMaxPooling, "avg": ME.MinkowskiAvgPooling}[mode]
    layer = cls(kernel_size=m["kernel_size"], stride=m["stride"], dilation=m["dilation"],
                dimension=m["D"])
    x, st = L.input(torch.float32, True)
    y = layer(st)
    out_c = _check_coordinates(L, y)
    _check_transpose(_check_kernel_map(L, y, out_c, is_pool=True))
    out_rows = _rows(out_c, f["out_coords"])
    gout = torch.empty((len(out_c), m["cin"]), device=cuda)
    gout[torch.from_numpy(out_rows).to(cuda)] = torch.from_numpy(f["grad_out"]).to(cuda)
    y.F.backward(gout)

    # float64 restatement on the fixture's pairs
    pairs = L.pairs(out_c)
    i = torch.cat([p[0] for p in pairs])
    o = torch.cat([p[1] for p in pairs])
    xd, gd = x.detach().double(), gout.double()
    C, n_out = xd.shape[1], len(out_c)
    cnt = torch.zeros(n_out, dtype=torch.float64, device=cuda).index_add_(
        0, o, torch.ones_like(o, dtype=torch.float64))
    if m["dilation"] != [1] * m["D"]:
        assert bool((cnt == 0).any()), "expected output rows with an empty window"
    if mode == "max":
        ref = torch.full((n_out, C), -torch.finfo(torch.float32).max, dtype=torch.float64,
                         device=cuda)
        ref.scatter_reduce_(0, o[:, None].expand(-1, C), xd[i], "amax")
        assert torch.equal(y.F.detach().double(), ref), "max pooling differs from float64"
        win = (xd[i] == ref[o]).double()           # features are all different: one winner
        gi_ref = torch.zeros_like(xd).index_add_(0, i, win * gd[o])
        assert torch.equal(x.grad.double(), gi_ref), "max pooling gradient differs"
    else:
        cnt = cnt.clamp(min=1)
        s = torch.zeros((n_out, C), dtype=torch.float64, device=cuda).index_add_(0, o, xd[i])
        A = torch.zeros_like(s).index_add_(0, o, xd[i].abs())
        assert_one_rounding(y.F.detach(), s / cnt[:, None], A / cnt[:, None], "avg pooling")
        g = gd[o] / cnt[o, None]
        gi_ref = torch.zeros_like(xd).index_add_(0, i, g)
        gi_A = torch.zeros_like(xd).index_add_(0, i, g.abs())
        assert_one_rounding(x.grad, gi_ref, gi_A, "avg pooling gradient")
    if mode == m["pool"]:
        assert np.abs(y.F.detach().cpu().numpy()[out_rows] - f["out_feats"]).max() < 1e-5
        assert np.abs(x.grad.cpu().numpy() - f["grad_in"][L.in_rows]).max() < 1e-5


def test_given_rows_out_of_reach_are_zero(ME, cuda):
    """conv(x, coordinates=C): rows of C that no input reaches exist in the output, all zero."""
    for name in ("given_tensor", "given_key"):
        f = np.load(os.path.join(GOLD, f"ref_layer_{name}.npz"))
        m = json.loads(str(f["meta"]))
        L = Layer(ME, f, m, cuda)
        _, st = L.input(torch.float32, False)
        y = L(st)
        out_c = y.C.cpu().numpy()
        reached = np.zeros(len(out_c), bool)
        reached[_rows(out_c, f["kmap"][:, 2 + m["D"]:])] = True      # out coordinate columns
        assert (~reached).any()
        assert not y.F[torch.from_numpy(~reached).to(cuda)].any()


def test_stride_of_large_coordinates_is_exact(ME, cuda):
    """Coordinates within 2^10 of +-2^30 at tensor stride 1, strided by 4 and 3: floor division in
    integers.  (The reference divides in float32, exact only below 2^24 — coordinate_map.hpp:64;
    this package's integer division is the documented difference, DESIGN.md.)"""
    g = torch.Generator().manual_seed(7)
    n = 2000
    c = torch.randint(-1000, 1000, (n, 3), generator=g, dtype=torch.int64)
    c += torch.where(torch.rand(n, 3, generator=g) < 0.5, -(2 ** 30), 2 ** 30 - 1024)
    coords = torch.cat([torch.randint(0, 2, (n, 1), generator=g), c], 1).int()
    cm = ME.CoordinateManager(D=3)
    key, _ = cm.insert_and_map(coords.to(cuda), 1)
    for s in (4, 3):
        sc = cm.get_coordinates(cm.stride(key, s)).cpu().numpy()
        u = np.unique(coords.numpy(), axis=0).astype(np.int64)
        exp = u.copy()
        exp[:, 1:] = np.floor_divide(u[:, 1:], s) * s
        assert np.array_equal(O.canonical_rows(sc)[0], np.unique(exp, axis=0))


def test_width_9_is_rejected(ME, cuda):
    """A 9-column input (D = 8) fails at once with the library's unsupported-width error."""
    g = torch.Generator().manual_seed(3)
    coords = torch.cat([torch.zeros(64, 1, dtype=torch.int32),
                        torch.randint(-4, 4, (64, 8), generator=g, dtype=torch.int32)], 1)
    with pytest.raises(Exception, match="unsupported coordinate width"):
        ME.SparseTensor(torch.rand(64, 4), coords, device=cuda)
    torch.cuda.synchronize()
