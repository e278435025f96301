"""Layer-by-layer audit of a network's training step (or eval forward) against float64.

A network built on `RecordingHandle(ME, audit)` (examples/minkunet.py takes any module handle) is
the unchanged network: its convolutions and batch norms are subclasses of the package's, so
parameter creation and `isinstance` are unchanged, and `fused_conv_bn_relu`, `fused_bn_relu` and
`cat` call the package's functions.  Every call checks the layer against a float64 restatement on
the inputs that layer received in the step, so errors do not compound through the network and each
layer is held to its kernel's own per-element bound (tests/helpers.py, DESIGN.md §6):

* the forward as the call returns;
* the input gradient in the backward of an identity "tap" on the layer's input features (a
  tensor with two consumers gets one tap per consumer, so each contribution is checked alone),
  from the output gradient its output tap recorded;
* parameter gradients in a post-accumulate hook on the parameter.

Kernel maps are restated here from the coordinates the layer saw (`x.C`, `y.C`): int64 keys,
`sort` + `searchsorted`, offsets in `oracle_np.region_offsets`' kernel-index order.  Nothing comes
from the library's hash tables or kernel maps.

Each check records its worst ratio |error| / bound (at most 1 passes) in `StepAudit.rows`; the
test asserts on them, so that one run prints every layer before it fails."""
import os
import sys
from collections import Counter

import numpy as np
import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
if _HERE not in sys.path:            # the suite's helper modules import each other by bare name
    sys.path.insert(0, _HERE)

from helpers import TC_ACC, WG_STEP, half_ulp, one_rounding_bound, ref_conv, ref_wgrad  # noqa: E402
from oracle import oracle_np as O  # noqa: E402

U = 2.0 ** -24
ACC_TF32 = TC_ACC + 2.0 ** 11        # (2^-9 + TC_ACC 2^-20) A: arbitrary fp32 operands in TF32


# ---- the kernel-map restatement ---------------------------------------------------------------
class RowLookup:
    """Exact row lookup of int32 (b, x, y, z...) coordinates: rows packed into int64 keys over the
    box [lo, lo + span) per spatial axis, sorted once, queried with searchsorted."""

    def __init__(self, coords, lo, span):
        self.lo, self.span = int(lo), int(span)
        self.D = coords.shape[1] - 1
        nb = int(coords[:, 0].max()) + 1 if len(coords) else 1
        assert int(coords[:, 0].min() if len(coords) else 0) >= 0, "negative batch index"
        assert nb * self.span ** self.D < 2 ** 62, "coordinate range does not fit an int64 key"
        keys = self._keys(coords)
        self.sorted, self.order = torch.sort(keys)
        assert len(keys) < 2 or bool((self.sorted[1:] != self.sorted[:-1]).all()), \
            "duplicate coordinates in a map"

    def _inside(self, c):
        s = c[:, 1:].long()
        return ((s >= self.lo) & (s < self.lo + self.span)).all(1)

    def _keys(self, c):
        c = c.long()
        k = c[:, 0]
        for a in range(1, self.D + 1):
            k = k * self.span + (c[:, a] - self.lo).clamp(0, self.span - 1)
        return k

    def find(self, q):
        """Row of every query in the map, or -1."""
        if len(self.sorted) == 0 or len(q) == 0:
            return torch.full((len(q),), -1, dtype=torch.int64, device=q.device)
        keys = self._keys(q)
        pos = torch.searchsorted(self.sorted, keys).clamp(max=len(self.sorted) - 1)
        hit = (self.sorted[pos] == keys) & self._inside(q)
        return torch.where(hit, self.order[pos], torch.full_like(pos, -1))


def _box(coord_sets, offsets):
    """(lo, span) of a key box holding every coordinate of `coord_sets` moved by any offset."""
    lo = min(int(c[:, 1:].min()) for c in coord_sets if len(c))
    hi = max(int(c[:, 1:].max()) for c in coord_sets if len(c))
    r = int(np.abs(offsets).max()) if len(offsets) else 0
    return lo - r, hi - lo + 2 * r + 1


def offsets_of(kernel_size, dilation, tensor_stride):
    """Hyper-cube region offsets [K, D] in the kernel-index order of W[k]."""
    return O.region_offsets(O.HYPER_CUBE, list(kernel_size), list(dilation), list(tensor_stride))


def conv_pairs(in_c, out_c, offsets, transposed=False):
    """[(input rows, output rows)] per offset k: a forward map probes the input coordinates at
    out + offset_k; a transposed map probes the output coordinates at in + offset_k (the swapped
    probe of oracle_np.transposed_kernel_map).  Pairs come in ascending order of the probing row."""
    if len(in_c) == 0 or len(out_c) == 0:
        return [(torch.zeros(0, dtype=torch.int64, device=in_c.device),) * 2 for _ in offsets]
    lo, span = _box([in_c, out_c], offsets)
    probe, table = (in_c, out_c) if transposed else (out_c, in_c)
    look = RowLookup(table, lo, span)
    off = torch.as_tensor(np.asarray(offsets), dtype=probe.dtype, device=probe.device)
    pairs = []
    for k in range(len(off)):
        q = probe.clone()
        q[:, 1:] += off[k]
        r = look.find(q)
        p = torch.nonzero(r >= 0).flatten()
        pairs.append((p, r[p]) if transposed else (r[p], p))
    return pairs


def strided_coords(coords, out_tensor_stride):
    """Unique rows of the coordinates floored to multiples of `out_tensor_stride` (lexicographic
    order)."""
    s = torch.as_tensor(list(out_tensor_stride), dtype=coords.dtype, device=coords.device)
    c = coords.clone()
    c[:, 1:] = torch.div(c[:, 1:], s, rounding_mode="floor") * s
    return torch.unique(c, dim=0)


def same_rows(a, b):
    """Whether two coordinate matrices hold the same set of rows (each without duplicates)."""
    if a.shape != b.shape:
        return False
    return torch.equal(torch.unique(a, dim=0), torch.unique(b, dim=0))


# ---- checks -----------------------------------------------------------------------------------
def _ratio(got, ref, bound):
    """(worst |got - ref| / bound, description of the first element beyond the bound or None).
    An element with a zero bound must match exactly."""
    err = (got.detach().double() - ref.detach().double()).abs()
    bound = bound.double().expand_as(err) if torch.is_tensor(bound) else \
        torch.full_like(err, float(bound))
    bad = ~(err <= bound)
    m = bound > 0
    worst = float((err[m] / bound[m]).max()) if bool(m.any()) else 0.0
    if not bool(bad.any()):
        return worst, None
    j = int(torch.nonzero(bad.flatten())[0])
    return max(worst, float("inf") if bound.flatten()[j] == 0 else worst), (
        f"{int(bad.sum())} of {bad.numel()} elements beyond the bound; first at flat index {j}: "
        f"got {got.flatten()[j].item()!r}, float64 {ref.flatten()[j].item()!r}, |err| "
        f"{err.flatten()[j].item():.3e} > {bound.flatten()[j].item():.3e}")


def _exact(got, want):
    """Ratio 0 when bit for bit equal, inf otherwise (with where)."""
    if got.shape == want.shape and torch.equal(got, want):
        return 0.0, None
    if got.shape != want.shape:
        return float("inf"), f"shape {tuple(got.shape)} != {tuple(want.shape)}"
    d = torch.nonzero((got != want).flatten())
    return float("inf"), f"{len(d)} of {got.numel()} elements differ, first at flat index {int(d[0])}"


def _cdiv(a, b):
    return -(-a // b)


def wgrad_share_steps(pairs, n_in, n_out, c_in, sms):
    """Per offset, an upper bound on the 16-pair wgmma steps one CTA of the pair-list
    k_wgrad_wg adds into one accumulator, from the offsets' pair counts `pairs` and the split
    plan of run_wgrad (csrc/conv_tc.cu, tc::wgrad_splits): splits planned from n_out / 192 + 1
    stages, held by a workspace sized for ceil(n_out / 64) stages (a larger workspace only gives
    more splits, so shorter shares).  A CTA takes a share of whole 64-pair stages of every row
    chunk (262144 rows or more) of the offset's list."""
    K, m = len(pairs), _cdiv(c_in, 128)

    def splits(stages):
        return max(1, min(_cdiv(2 * sms, K * m), max(1, stages // 4), 65535))
    ws = splits(_cdiv(n_out, 64))
    S = 1 if ws <= 1 else min(splits(n_out // 192 + 1), ws)
    nch = _cdiv(max(n_in, n_out, 1), 262144)
    return [4 * (_cdiv(_cdiv(P, 64) + nch, S) + nch) for P in pairs]


class _Tap(torch.autograd.Function):
    """Identity whose backward hands the gradient crossing it to `cb`."""

    @staticmethod
    def forward(ctx, x, cb):
        ctx.cb = cb
        return x.view_as(x)

    @staticmethod
    def backward(ctx, g):
        ctx.cb(g)
        return g, None


def tap(x, cb):
    return _Tap.apply(x, cb) if x.requires_grad else x


class Row:
    """One audited call: what it was, and its worst ratio per checked quantity."""

    def __init__(self, step, name, kind, rows, K, c_in, c_out):
        self.step, self.name, self.kind = step, name, kind
        self.rows, self.K, self.c_in, self.c_out = rows, K, c_in, c_out
        self.route = ""
        self.ratios = {}
        self.failures = []
        self.notes = []
        self.expect = Counter()     # checks the call must run, and how many times
        self.seen = Counter()

    def put(self, what, result):
        r, why = result
        self.seen[what] += 1
        self.ratios[what] = max(self.ratios.get(what, 0.0), r)
        if why is not None:
            self.failures.append(f"{what}: {why}")

    @property
    def worst(self):
        return max(self.ratios.values(), default=0.0)

    def line(self):
        q = ", ".join(f"{k} {v:.3g}" for k, v in self.ratios.items())
        shape = f"K={self.K} {self.c_in}->{self.c_out}" if self.K else f"C={self.c_in}"
        return (f"step {self.step} {self.name:<22} {self.kind:<9} rows {self.rows:>7} {shape:<16} "
                f"{self.route:<8} {q}")


# ---- the audit --------------------------------------------------------------------------------
class StepAudit:
    """Checks every convolution, batch norm and `cat` of a network built on a RecordingHandle.

    `names(net)` gives the modules their qualified names; `step` numbers the rows.  After the
    calls, `rows` holds one Row per audited call and `calls` counts the audited calls per
    (step, module name)."""

    def __init__(self, ME):
        self.ME = ME
        self.step = 0
        self.enabled = True
        self.rows = []
        self.calls = Counter()
        self.cats = Counter()
        self._names = {}
        self._pairs = {}
        self._coords_by_ts = {}
        self._bwd_tc = {}
        self._conv_entered = None
        self._last_conv = None

    # -- bookkeeping --
    def names(self, net):
        from minkowskiengine_b200.convolution import MinkowskiConvolutionBase
        for n, m in net.named_modules():
            self._names[id(m)] = n
        for m in net.modules():
            if isinstance(m, MinkowskiConvolutionBase):
                m.kernel.register_post_accumulate_grad_hook(self._kernel_grad)
                if m.bias is not None:
                    m.bias.register_post_accumulate_grad_hook(self._bias_grad)
            if isinstance(m, self.ME.MinkowskiBatchNorm) and m.bn.affine:
                m.bn.weight.register_post_accumulate_grad_hook(self._bn_weight_grad)
                m.bn.bias.register_post_accumulate_grad_hook(self._bn_bias_grad)
        self._owner = {}
        for m in net.modules():
            if isinstance(m, MinkowskiConvolutionBase):
                self._owner[id(m.kernel)] = m
                if m.bias is not None:
                    self._owner[id(m.bias)] = m
            if isinstance(m, self.ME.MinkowskiBatchNorm) and m.bn.affine:
                self._owner[id(m.bn.weight)] = m
                self._owner[id(m.bn.bias)] = m

    def begin_step(self, step):
        self.step = step
        self._pairs.clear()
        self._coords_by_ts.clear()
        self._bwd_tc.clear()

    def missing(self):
        """'step name: check' for every expected check that did not run (as often as expected)."""
        return [f"step {r.step} {r.name}: {k}" for r in self.rows for k, n in r.expect.items()
                if r.seen[k] < n]

    def _name(self, m):
        return self._names.get(id(m), type(m).__name__)

    def _row(self, module, kind, rows, K, c_in, c_out, count=True):
        r = Row(self.step, self._name(module), kind, rows, K, c_in, c_out)
        self.rows.append(r)
        if count:
            self.calls[(self.step, r.name)] += 1
        return r

    def backward_routes(self):
        """A context that wraps the convolution backward entry points of `backend` to note, per
        kernel, whether its backward launched tensor-core kernels (dgrad and wgrad are one library
        call: a layer gets the tensor-core bound in both directions when either launched one)."""
        from minkowskiengine_b200 import _lib, backend
        audit = self

        class _Routes:
            def __enter__(self):
                self.saved = (backend.ConvolutionBackwardGPU, backend.ConvolutionTransposeBackwardGPU)

                def wrap(fn):
                    def call(in_feat, grad_out, kernel, *a, **kw):
                        tc0 = _lib.tc_launch_count()
                        out = fn(in_feat, grad_out, kernel, *a, **kw)
                        audit._bwd_tc[id(kernel)] = _lib.tc_launch_count() > tc0
                        return out
                    return call
                backend.ConvolutionBackwardGPU = wrap(self.saved[0])
                backend.ConvolutionTransposeBackwardGPU = wrap(self.saved[1])
                return self

            def __exit__(self, *exc):
                backend.ConvolutionBackwardGPU, backend.ConvolutionTransposeBackwardGPU = self.saved
        return _Routes()

    # -- convolutions --
    def _acc(self, dtype, tc):
        if not tc:
            return 1.0
        if dtype == torch.float32:     # fp32 features on the tensor cores: TF32, under its switch
            return ACC_TF32 if torch.backends.cuda.matmul.fp32_precision == "tf32" else 1.0
        return TC_ACC

    def _conv_geometry(self, mod, x, y):
        """Independent pairs of the layer and checks of its output coordinates."""
        from minkowskiengine_b200.enums import RegionType
        kg = mod.kernel_generator
        assert kg.region_type == RegionType.HYPER_CUBE, "only hyper-cube regions are restated"
        x_ts, y_ts = list(x.tensor_stride), list(y.tensor_stride)
        checks = {}
        if mod.is_transpose:
            assert [a // int(s) for a, s in zip(x_ts, kg.kernel_stride)] == y_ts
            target = self._coords_by_ts.get(tuple(y_ts))
            checks["coords"] = (0.0, None) if target is not None and same_rows(y.C, target) else \
                (float("inf"), "the output coordinates are not those of the target map")
        elif any(int(s) > 1 for s in kg.kernel_stride):
            assert [a * int(s) for a, s in zip(x_ts, kg.kernel_stride)] == y_ts
            want = strided_coords(x.C, y_ts)
            ok = len(torch.unique(y.C, dim=0)) == len(y.C) and same_rows(y.C, want)
            checks["coords"] = (0.0, None) if ok else \
                (float("inf"), "the output coordinates are not the floored input coordinates")
        else:
            ok = y.coordinate_map_key == x.coordinate_map_key and torch.equal(y.C, x.C)
            checks["coords"] = (0.0, None) if ok else \
                (float("inf"), "a stride-1 layer changed the coordinate map")
        self._coords_by_ts.setdefault(tuple(x_ts), x.C)
        self._coords_by_ts.setdefault(tuple(y_ts), y.C)
        key = (x.coordinate_map_key._tuple(), y.coordinate_map_key._tuple(),
               tuple(kg.kernel_size), tuple(kg.kernel_stride), tuple(kg.kernel_dilation),
               bool(mod.is_transpose))
        pairs = self._pairs.get(key)
        if pairs is None:
            offs = offsets_of(kg.kernel_size, kg.kernel_dilation, y_ts if mod.is_transpose else x_ts)
            pairs = self._pairs[key] = conv_pairs(x.C, y.C, offs, mod.is_transpose)
        return pairs, checks

    def _weights(self, mod, dtype, tc=True):
        """The weights a route multiplies: the feature dtype's rounding; fp32 under the TF32
        switch off the tensor cores reads the packed weights, rounded to tf32 (ties away)."""
        w = mod.kernel.detach()
        if dtype != torch.float32:
            return w.to(dtype)
        if not tc and torch.backends.cuda.matmul.fp32_precision == "tf32":
            from test_gpu_tf32 import _tf32_rna
            return _tf32_rna(w)
        return w

    def conv_call(self, mod, forward, x, coordinates):
        """A convolution module's forward, audited (the subclasses' forward)."""
        from minkowskiengine_b200 import _lib
        if not self.enabled:
            return forward(x, coordinates)
        self._conv_entered = mod
        grad = torch.is_grad_enabled()
        dtype = x.F.dtype
        kind = "mm" if mod.use_mm else ("convtr" if mod.is_transpose else "conv")
        K = 1 if mod.use_mm else mod.kernel_generator.kernel_volume
        row = self._row(mod, kind, x.F.shape[0], K, mod.in_channels, mod.out_channels)
        st = {"row": row, "dy": None, "mod": mod, "pending": 0}
        xf = tap(x.F, lambda g: self._conv_dx(st, g)) if grad else x.F
        xs = self.ME.SparseTensor(xf, coordinate_map_key=x.coordinate_map_key,
                                  coordinate_manager=x.coordinate_manager)
        tc0 = _lib.tc_launch_count()
        y = forward(xs, coordinates)
        tc = _lib.tc_launch_count() > tc0
        row.route = "mm" if mod.use_mm else ("tc" if tc else "cuda")
        row.expect.update(["fwd", "coords"])
        if grad:
            row.expect.update(["wgrad"] + ["dgrad"] * xf.requires_grad +
                              ["bias_grad"] * (mod.bias is not None))
        st["x"] = xf.detach()
        if mod.use_mm:
            wc = mod.kernel.detach().to(dtype)
            row.put("fwd", self._mm(row, y.F, xf.detach(), wc, bias=mod.bias))
            row.put("coords", (0.0, None) if y.coordinate_map_key == x.coordinate_map_key else
                    (float("inf"), "a K = 1 stride-1 layer changed the coordinate map"))
            st["wc"] = wc
        else:
            assert mod.bias is None, "the float64 restatement covers bias-free convolutions"
            pairs, checks = self._conv_geometry(mod, xs, y)
            for k, v in checks.items():
                row.put(k, v)
            wl = self._weights(mod, dtype, tc)
            ref, A = ref_conv(xf.detach(), wl, pairs, y.F.shape[0])
            acc = self._acc(dtype, tc)
            row.put("fwd", _ratio(y.F, ref, one_rounding_bound(ref, A, dtype, acc)))
            del ref, A
            st.update(pairs=pairs, wl=wl, n_in=x.F.shape[0], n_out=y.F.shape[0])
        self._last_conv = st
        st["y"], st["listeners"] = y.F, []
        if not grad:
            return y
        st["pending"] = int(xf.requires_grad) + 1 + int(mod.bias is not None)
        mod._audit_state = st
        yf = tap(y.F, lambda g: self._conv_dy(st, g))
        st["y"] = yf
        return self.ME.SparseTensor(yf, coordinate_map_key=y.coordinate_map_key,
                                    coordinate_manager=y.coordinate_manager)

    def _mm(self, row, got, a, b, out_dtype=None, bias=None):
        """A K = 1 stride-1 layer is torch's a.mm(b) [+ bias]: bit for bit against the same
        expression recomputed; if cuBLAS does not repeat itself, within float64 of one fp32
        accumulation on the tensor cores (TC_ACC) and one rounding (noted as "fp64")."""
        want = a.mm(b)
        if bias is not None:
            want = want + bias.detach().to(want.dtype)
        if out_dtype is not None:
            want = want.to(out_dtype)
        got = got.detach()
        if torch.equal(got, want):
            if "bitwise" not in row.notes:
                row.notes.append("bitwise")
            return 0.0, None
        row.notes.append("fp64")
        ref, A = a.double().mm(b.double()), a.double().abs().mm(b.double().abs())
        if bias is not None:
            ref = ref + bias.detach().double()
            A = A + bias.detach().double().abs()
        return _ratio(got, ref, one_rounding_bound(ref, A, got.dtype, TC_ACC))

    def _release(self, st):
        st["pending"] -= 1
        if st["pending"] <= 0:
            for k in ("x", "dy", "wc", "wl", "pairs", "y"):
                st.pop(k, None)

    def _conv_dy(self, st, g):
        st["dy"] = g.detach()
        for cb in st["listeners"]:
            cb(g)

    def _conv_dx(self, st, g):
        row, mod, dy = st["row"], st["mod"], st["dy"]
        if mod.use_mm:                                   # torch autograd of x.mm(W.to(dtype))
            row.put("dgrad", self._mm(row, g, dy, st["wc"].t()))
        else:
            tc = self._bwd_tc.get(id(mod.kernel), False)
            row.route += "/" + ("tc" if tc else "cuda")
            pairs = [(o, i) for i, o in st["pairs"]]
            ref, A = ref_conv(dy, st["wl"].transpose(1, 2), pairs, st["n_in"])
            row.put("dgrad", _ratio(g, ref, one_rounding_bound(ref, A, g.dtype,
                                                               self._acc(g.dtype, tc))))
        self._release(st)

    def _kernel_grad(self, p):
        mod = self._owner[id(p)]
        st = getattr(mod, "_audit_state", None)
        if st is None or "x" not in st:
            return
        row, dy = st["row"], st["dy"]
        if mod.use_mm:
            row.put("wgrad", self._mm(row, p.grad, st["x"].t(), dy, p.dtype))
        else:
            tc = self._bwd_tc.get(id(mod.kernel), False)
            ref, A = ref_wgrad(st["x"], dy, st["pairs"])
            acc = self._acc(st["x"].dtype, tc)
            if tc and st["x"].dtype != torch.float32:
                # the error in 2^-20 A units, and how one-signed the worst element's sum is
                unit = ((p.grad.double() - ref).abs() / (A * 2.0 ** -20)).where(A > 0, 0.0)
                j = int(unit.argmax())
                row.notes.append(f"wgrad/2^-20A {float(unit.flatten()[j]):.3g} at "
                                 f"|sum|/A {float(ref.abs().flatten()[j] / A.flatten()[j]):.2f}")
                acc = self._wgrad_acc(mod, st, acc)
            row.put("wgrad", _ratio(p.grad, ref, one_rounding_bound(ref, A, torch.float32, acc)))
        self._release(st)

    def _wgrad_acc(self, mod, st, acc):
        """The bf16 / fp16 tensor-core wgrad's bound in 2^-20 A units, per offset: TC_ACC, or on
        the pair lists WG_STEP · steps · 2^-24 where that is larger (one-signed operands,
        tests/test_gpu_wgrad_accumulation.py)."""
        from minkowskiengine_b200 import _lib, backend
        x, kernel = st["x"], mod.kernel
        K, c_in, c_out = kernel.shape
        if backend._is_stem(kernel, x.dtype) or not (backend._is_master(kernel) and _lib.load(
                ).meb200_conv_wgrad_uses_pairs(_lib.dtype_code(x.dtype), c_in, c_out, K)):
            return acc
        sms = torch.cuda.get_device_properties(x.device).multi_processor_count
        steps = wgrad_share_steps([len(i) for i, _ in st["pairs"]], st["n_in"], st["n_out"],
                                  c_in, sms)
        return torch.tensor([max(acc, WG_STEP * n / 16) for n in steps], dtype=torch.float64,
                            device=x.device).view(-1, 1, 1)

    def _bias_grad(self, p):
        mod = self._owner[id(p)]
        st = getattr(mod, "_audit_state", None)
        if st is None or st.get("dy") is None:
            return
        st["row"].put("bias_grad", _exact(p.grad, st["dy"].sum(0, keepdim=True).to(p.dtype)))
        self._release(st)

    # -- batch norm --
    def bn_call(self, norm, x, residual, relu, call, conv=None):
        """`call(x, residual)` of batch norm module `norm`, audited.  With `conv`, x is None and
        `call` runs that convolution first (fused_conv_bn_relu in training): the norm's input is
        the convolution's output, and the convolution's output tap gives the norm's dx."""
        if not self.enabled:
            return call(x, residual)
        from test_gpu_batchnorm_fp64 import (_dx_bound, _grad_bounds, _stat_bounds, _stored,
                                             _y_bound, bn_geometry)
        bn = norm.bn
        assert float(np.float32(bn.eps)) == float(np.float32(1e-5)) and \
            float(np.float32(bn.momentum)) == float(np.float32(0.1)), \
            "the bounds are those of eps 1e-5 and momentum 0.1"
        training = bn.training
        grad = torch.is_grad_enabled()
        st = {"pending": 0}
        rm0, rv0 = bn.running_mean.detach().clone(), bn.running_var.detach().clone()
        nbt0 = int(bn.num_batches_tracked)
        xs = None
        if x is not None:
            xf = tap(x.F, lambda g: self._bn_dx(st, g)) if grad else x.F
            xs = self.ME.SparseTensor(xf, coordinate_map_key=x.coordinate_map_key,
                                      coordinate_manager=x.coordinate_manager)
        rs = None
        if residual is not None:
            rf = tap(residual.F, lambda g: self._bn_dres(st, g)) if grad else residual.F
            rs = self.ME.SparseTensor(rf, coordinate_map_key=residual.coordinate_map_key,
                                      coordinate_manager=residual.coordinate_manager)
        self._last_conv = None
        out = call(xs, rs)
        if conv is not None:
            cst = self._last_conv
            assert cst is not None and cst["mod"] is conv, "the convolution was not audited"
            xf = cst["y"]
            if grad:
                cst["listeners"].append(lambda g: self._bn_dx(st, g))
        n, C = xf.shape
        row = st["row"] = self._row(norm, "bn" + ("+res" if residual is not None else "") +
                                    ("+relu" if relu else ""), n, 0, C, C)
        row.route = "train" if training else "eval"
        row.expect.update(["y"] + ["relu"] * relu +
                          (["run_mean", "run_var", "nbt"] if training else ["run_stats"]))
        if grad:
            row.expect.update(["dx"] + ["dres"] * (rs is not None and rs.F.requires_grad) +
                              ["dweight", "dbias"] * bn.affine)
        dtype = out.F.dtype
        dev = out.F.device
        x0 = xf.detach().double()
        geom = bn_geometry(n, C)
        st0 = _stat_bounds(x0, geom, training, rm0, rv0)
        one = torch.ones((), dtype=torch.float64, device=dev)
        w64 = bn.weight.detach().double() if bn.affine else one
        b64 = bn.bias.detach().double() if bn.affine else one * 0
        r64 = rs.F.detach().double() if rs is not None else one * 0
        z = (x0 - st0["mu"]) * st0["is_"] * w64 + b64 + r64
        yb = _y_bound(x0, st0["mu"], st0["is_"], w64, b64, r64, st0["e_mu"], st0["rho"])
        yref = z.clamp(min=0) if relu else z
        y = out.F.detach()
        row.put("y", _ratio(y, yref, _stored(yb, yref, dtype)))
        if relu:
            flip = (y > 0) != (z > 0)
            ok = bool((z[flip].abs() <= yb[flip]).all())
            row.put("relu", (0.0, None) if ok else (float("inf"), "a ReLU decision beyond the bound"))
        del yref
        if training:
            mom = float(np.float32(0.1))
            mu, var = st0["mu"], st0["var"]
            rm = (1 - mom) * rm0.double() + mom * mu
            rv = (1 - mom) * rv0.double() + mom * var * n / (n - 1)
            row.put("run_mean", _ratio(bn.running_mean, rm, st0["e_rm"]))
            row.put("run_var", _ratio(bn.running_var, rv, st0["e_rv"]))
            row.put("nbt", (0.0, None) if int(bn.num_batches_tracked) == nbt0 + 1 else
                    (float("inf"), "num_batches_tracked did not count the batch"))
        else:
            ok = torch.equal(bn.running_mean, rm0) and torch.equal(bn.running_var, rv0)
            row.put("run_stats", (0.0, None) if ok else
                    (float("inf"), "eval mode moved the running statistics"))
        if not grad:
            return out
        st.update(x0=x0, st=st0, geom=geom, w64=w64, y=y, relu=relu, training=training,
                  dtype=dtype, grads=(_grad_bounds, _dx_bound, _stored))
        st["pending"] = 1 + int(residual is not None and rs.F.requires_grad) + \
            (2 if bn.affine else 0)
        norm._audit_state = st
        yf = tap(out.F, lambda g: self._bn_dy(st, g))
        return self.ME.SparseTensor(yf, coordinate_map_key=out.coordinate_map_key,
                                    coordinate_manager=out.coordinate_manager)

    def _bn_dy(self, st, g):
        """Every backward reference of the norm, from the gradient of its output."""
        _grad_bounds, _dx_bound, _stored = st["grads"]
        dy = g.detach().double()
        x0, s, geom, n = st["x0"], st["st"], st["geom"], st["x0"].shape[0]
        D = torch.where(st["y"] > 0, dy, 0.0) if st["relu"] else dy
        X, ex, eG1, eG2 = _grad_bounds(D, x0, s, geom, st["training"])
        G1, G2 = D.sum(0), (D * X).sum(0)
        isw = s["is_"] * st["w64"]
        if st["training"]:
            K1, K2 = G1 / n, G2 / n
            ek1 = eG1 / n + (U + 2 * 2.0 ** -53) * (K1.abs() + eG1 / n)
            ek2 = eG2 / n + (U + 2 * 2.0 ** -53) * (K2.abs() + eG2 / n)
        else:
            K1 = K2 = ek1 = ek2 = torch.zeros_like(G1)
        dx = (D - K1 - X * K2) * isw
        st["dx"] = (dx, _stored(_dx_bound(D, X, K1, K2, isw, s["rho"], ex, ek1, ek2), dx, st["dtype"]))
        st["D"] = D.to(st["dtype"])
        st["G"] = (G1, eG1 + U * (G1.abs() + eG1), G2, eG2 + U * (G2.abs() + eG2))
        for k in ("x0", "y"):
            st.pop(k)

    def _bn_release(self, st):
        st["pending"] -= 1
        if st["pending"] <= 0:
            for k in ("dx", "D", "G", "x0", "y"):
                st.pop(k, None)

    def _bn_dx(self, st, g):
        st["row"].put("dx", _ratio(g, *st["dx"]))
        self._bn_release(st)

    def _bn_dres(self, st, g):
        st["row"].put("dres", _exact(g, st["D"]))
        self._bn_release(st)

    def _bn_weight_grad(self, p):
        st = getattr(self._owner[id(p)], "_audit_state", None)
        if st is not None and "G" in st:
            G1, bG1, G2, bG2 = st["G"]
            st["row"].put("dweight", _ratio(p.grad, G2, bG2))
            self._bn_release(st)

    def _bn_bias_grad(self, p):
        st = getattr(self._owner[id(p)], "_audit_state", None)
        if st is not None and "G" in st:
            G1, bG1, G2, bG2 = st["G"]
            st["row"].put("dbias", _ratio(p.grad, G1, bG1))
            self._bn_release(st)

    # -- the package's functions --
    def fused_conv_bn_relu(self, conv, norm, x, residual=None, relu=True):
        ME = self.ME
        if not self.enabled:
            return ME.fused_conv_bn_relu(conv, norm, x, residual, relu)
        if norm.bn.training or torch.is_grad_enabled():
            # the convolution (audited by its subclass), then the batch-norm tail on its output
            return self.bn_call(norm, None, residual, relu,
                                lambda _, rs: ME.fused_conv_bn_relu(conv, norm, x, rs, relu),
                                conv=conv)
        return self._fused_eval(conv, norm, x, residual, relu)

    def _fused_eval(self, conv, norm, x, residual, relu):
        """Eval, no gradient: one convolution with batch norm, residual and ReLU in its epilogue,
        against a float64 convolution followed by the float64 batch norm's affine map."""
        from minkowskiengine_b200 import _lib
        from minkowskiengine_b200.normalization import _bn_tail
        ME = self.ME
        dtype = x.F.dtype
        K = conv.kernel_generator.kernel_volume
        row = self._row(conv, "conv+bn", x.F.shape[0], K, conv.in_channels, conv.out_channels)
        self.calls[(self.step, self._name(norm))] += 1
        row.name = f"{row.name}+{self._name(norm).rsplit('.', 1)[-1]}"
        self._conv_entered = None
        n0, tc0 = _lib.launch_count(), _lib.tc_launch_count()
        out = ME.fused_conv_bn_relu(conv, norm, x, residual, relu)
        n_fused, tc = _lib.launch_count() - n0, _lib.tc_launch_count() > tc0
        row.route = "tc" if tc else "cuda"
        row.expect.update(["one_launch", "coords", "fwd"])
        one_pass = self._conv_entered is None
        self.enabled = False
        try:
            n0 = _lib.launch_count()
            c = conv(x)
            _bn_tail(norm, c, residual, relu) if (residual is not None or relu) else norm(c)
            n_comp = _lib.launch_count() - n0
        finally:
            self.enabled = True
        row.put("one_launch", (0.0, None) if one_pass and n_fused < n_comp else
                (float("inf"), f"{n_fused} launches, the composition {n_comp}"))
        pairs, checks = self._conv_geometry(conv, x, out)
        for k, v in checks.items():
            row.put(k, v)
        ref, A = ref_conv(x.F, self._weights(conv, dtype, tc), pairs, out.F.shape[0])
        bn = norm.bn
        one = torch.ones((), dtype=torch.float64, device=ref.device)
        w64 = bn.weight.detach().double() if bn.affine else one
        b64 = bn.bias.detach().double() if bn.affine else one * 0
        rm, rv = bn.running_mean.double(), bn.running_var.double()
        s = w64 / (rv + float(np.float32(bn.eps))).sqrt()
        cb = conv.bias.detach().double().reshape(-1) if conv.bias is not None else one * 0
        sh = b64 - rm * s + cb * s
        pre = ref * s + sh
        mag = (ref * s).abs() + sh.abs()
        if residual is not None:
            pre = pre + residual.F.double()
            mag = mag + residual.F.double().abs()
        yref = pre.clamp(min=0) if relu else pre
        # tests/test_gpu_conv_epilogue._expected: the accumulator's error scaled by |scale|, the
        # epilogue's fp32 fma and residual add; plus the fp32 folding of the scale (rsqrt 2 ulp,
        # the sum and the product with w: 6u with one spare) and of the shift (its product and
        # two sums, on |rm s|, |b| and |conv bias · s|)
        e_s = 6 * U * s.abs()
        e_sh = (rm.abs() + cb.abs()) * e_s + 3 * U * ((rm * s).abs() + b64.abs() + (cb * s).abs())
        delta = A * (self._acc(dtype, tc) * 2.0 ** -20) * s.abs() + 2.0 ** -22 * mag + \
            ref.abs() * e_s + e_sh
        if dtype != torch.float32:
            delta = half_ulp(yref.abs() + delta, dtype) + delta
        row.put("fwd", _ratio(out.F, yref, delta))
        return out

    def fused_bn_relu(self, norm, x, residual=None):
        ME = self.ME
        return self.bn_call(norm, x, residual, True,
                            lambda xs, rs: ME.fused_bn_relu(norm, xs, rs))

    def cat(self, *tensors):
        ME = self.ME
        if not self.enabled:
            return ME.cat(*tensors)
        grad = torch.is_grad_enabled()
        row = Row(self.step, f"cat{self.cats[self.step]}", "cat", tensors[0].F.shape[0], 0,
                  sum(t.F.shape[1] for t in tensors), sum(t.F.shape[1] for t in tensors))
        row.route = "torch"
        row.expect.update(["fwd"] + ["dx"] * (len(tensors) * grad))
        self.rows.append(row)
        self.cats[self.step] += 1
        st = {"dy": None}
        ins, off = [], 0
        for t in tensors:
            c = t.F.shape[1]
            f = tap(t.F, (lambda lo, hi: lambda g: row.put("dx", _exact(g, st["dy"][:, lo:hi])))(
                off, off + c)) if grad else t.F
            ins.append(ME.SparseTensor(f, coordinate_map_key=t.coordinate_map_key,
                                       coordinate_manager=t.coordinate_manager))
            off += c
        out = ME.cat(*ins)
        row.put("fwd", _exact(out.F.detach(), torch.cat([t.F.detach() for t in ins], 1)))
        if not grad:
            return out

        def dy(g):
            st["dy"] = g.detach()
        return ME.SparseTensor(tap(out.F, dy), coordinate_map_key=out.coordinate_map_key,
                               coordinate_manager=out.coordinate_manager)


def RecordingHandle(ME, audit):
    """A module handle for examples/minkunet.py: the package, but for audited subclasses of its
    convolution and batch-norm modules and audited `fused_conv_bn_relu`, `fused_bn_relu`, `cat`."""

    class MinkowskiConvolution(ME.MinkowskiConvolution):
        def forward(self, input, coordinates=None):
            return audit.conv_call(self, super().forward, input, coordinates)

    class MinkowskiConvolutionTranspose(ME.MinkowskiConvolutionTranspose):
        def forward(self, input, coordinates=None):
            return audit.conv_call(self, super().forward, input, coordinates)

    class MinkowskiBatchNorm(ME.MinkowskiBatchNorm):
        def forward(self, input):
            return audit.bn_call(self, input, None, False, lambda xs, _: super(
                MinkowskiBatchNorm, self).forward(xs))

    class Handle:
        def __getattr__(self, name):
            return getattr(ME, name)

    h = Handle()
    h.MinkowskiConvolution = MinkowskiConvolution
    h.MinkowskiConvolutionTranspose = MinkowskiConvolutionTranspose
    h.MinkowskiBatchNorm = MinkowskiBatchNorm
    h.fused_conv_bn_relu = audit.fused_conv_bn_relu
    h.fused_bn_relu = audit.fused_bn_relu
    h.cat = audit.cat
    return h
