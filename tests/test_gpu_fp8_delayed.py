"""fp8 training with delayed scaling (ME.Fp8DelayedScaling) on the GPU: the convert-and-record and
roll kernels against torch and float64, the batch-norm passes that write fp8 copies (every other
output bit-identical to the passes without them), saturation and the next step's scale, a step
without host synchronisation, and MinkUNet training steps: step 0 bit for bit that of
fp8_training(weight_gradient=True), the shadows read from step 1 on, a checkpoint resumed bit for
bit, and a short fit against bf16."""
import contextlib
import types

import numpy as np
import pytest
import torch

from test_gpu_batchnorm_fp64 import CASES

pytestmark = pytest.mark.gpu

FMTS = {"e4m3": (0, torch.float8_e4m3fn, 448.0), "e5m2": (1, torch.float8_e5m2, 57344.0)}
DTYPES = [torch.float32, torch.bfloat16, torch.float16]
FLT_MAX = float(np.finfo(np.float32).max)


def _expect(v, inv, fmt):
    """The bytes the kernels write of values v at a scale: the product in fp32, saturated."""
    _, dt, M = FMTS[fmt]
    return (v.float() * inv).clamp(-M, M).to(dt).view(torch.uint8)


def _finite_amax(v):
    a = v.float().abs()
    return float(torch.where(torch.isfinite(a), a, torch.zeros_like(a)).max()) if v.numel() else 0.


# ---- convert and record -----------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", list(FMTS))
@pytest.mark.parametrize("dtype", DTYPES, ids=str)
@pytest.mark.parametrize("n,c,offset", [(1000, 64, 0), (1000, 64, 1), (37, 33, 0), (3, 7, 3),
                                        (100_003, 96, 0), (1, 1, 0)])
def test_convert_and_record(ME, cuda, fmt, dtype, n, c, offset):
    B = ME.backend
    g = torch.Generator(device=cuda).manual_seed(n + c)
    base = (torch.randn(n * c + offset, generator=g, device=cuda) * 3).to(dtype)
    x = base[offset:].view(n, c)                      # offset: not 16-byte aligned
    amax = _finite_amax(x)
    inv = torch.tensor(FMTS[fmt][2] / (0.5 * amax), dtype=torch.float32)   # saturates the top half
    scale = torch.stack([1 / inv, inv]).float().to(cuda)
    slot = torch.tensor([0.25], device=cuda)
    q = B.quantize_fp8_record(x, FMTS[fmt][0], scale, slot)
    assert torch.equal(q, _expect(x, scale[1], fmt))
    assert float(slot) == max(amax, 0.25)


@pytest.mark.parametrize("fmt", list(FMTS))
def test_record_ignores_nan_and_inf(ME, cuda, fmt):
    x = torch.randn(4096, 32, device=cuda).bfloat16()
    x[5, 3], x[77, 0], x[1000, 31] = float("nan"), float("inf"), -float("inf")
    scale = torch.tensor([1.0, 1.0], device=cuda)
    for prev in (0.0, 1e3):
        slot = torch.tensor([prev], device=cuda)
        ME.backend.quantize_fp8_record(x, FMTS[fmt][0], scale, slot)
        assert float(slot) == max(prev, _finite_amax(x))


# ---- the roll ----------------------------------------------------------------------------------------
def _scales64(amax, margin, M):
    a = min(float(np.float32(amax)) * 2.0 ** margin, FLT_MAX)
    if a == 0:
        return 1.0, 1.0
    q = M / a
    if q >= FLT_MAX * (1 + 2 ** -25):
        return float(np.float32(1 / FLT_MAX)), FLT_MAX
    return float(np.float32(a / M)), float(np.float32(q))


@pytest.mark.parametrize("H", [1, 2, 16, 1024])
@pytest.mark.parametrize("margin", [0, 3])
def test_roll(ME, cuda, H, margin):
    n4, n5 = 70, 45
    L = n4 + n5
    g = torch.Generator().manual_seed(H + margin)
    hist = (torch.rand(L, H, generator=g) * 10) ** 4
    hist[::7] = 0                                       # never recorded
    hist[3, :] = 1e-45                                  # subnormal
    hist[4, 0] = FLT_MAX
    cur = torch.rand(L, generator=g) * 100
    cur[::5] = 0
    h_dev, c_dev = hist.to(cuda), cur.to(cuda)
    nxt, scales = ME.backend.fp8_roll(c_dev, h_dev, n4, n5, margin)
    want = torch.cat([cur[:, None], hist[:, :H - 1]], 1)
    assert torch.equal(h_dev.cpu(), want)
    assert not nxt.any()
    sc = scales.cpu()
    for i in range(L):
        M = 448.0 if i < n4 else 57344.0
        s, inv = _scales64(float(want[i].max()), margin, M)
        assert (float(sc[i, 0]), float(sc[i, 1])) == (s, inv), i


# ---- batch-norm shadows ----------------------------------------------------------------------------
def _bn_run(ME, x0, res0, relu, fp8, group=None):
    from minkowskiengine_b200.normalization import _BatchNormFunction
    C = x0.shape[1]
    dev = x0.device
    x = x0.clone().requires_grad_(True)
    res = None if res0 is None else res0.clone().requires_grad_(True)
    w = torch.linspace(0.5, 1.5, C, device=dev).requires_grad_(True)
    b = torch.linspace(-0.2, 0.3, C, device=dev).requires_grad_(True)
    rm, rv = torch.zeros(C, device=dev), torch.ones(C, device=dev)
    y = _BatchNormFunction.apply(x, w, b, rm, rv, 0.1, 1e-5, group, relu, res, False, None, fp8)
    dy = torch.randn(x0.shape, generator=torch.Generator(device=dev).manual_seed(1),
                     device=dev).to(x0.dtype)
    y.backward(dy)
    return {"y": y.detach(), "dx": x.grad, "dres": None if res is None else res.grad,
            "gw": w.grad, "gb": b.grad, "rm": rm, "rv": rv}


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
@pytest.mark.parametrize("relu,residual", [(False, False), (True, False), (True, True),
                                           (False, True)])
@pytest.mark.parametrize("n,C", CASES, ids=lambda v: str(v))
def test_bn_shadows(ME, cuda, n, C, dtype, relu, residual):
    from minkowskiengine_b200.fp8_delayed import _BnStep
    g = torch.Generator(device=cuda).manual_seed(n ^ C)
    x0 = (torch.randn(n, C, generator=g, device=cuda) * 2 + 0.5).to(dtype)
    res0 = torch.randn(n, C, generator=g, device=cuda).to(dtype) if residual else None
    plain = _bn_run(ME, x0, res0, relu, None)
    # scales from the plain outputs, halved so that the largest values saturate
    sy = 448.0 / max(0.5 * _finite_amax(plain["y"]), 1e-30)
    sdx = 57344.0 / max(0.5 * _finite_amax(plain["dx"]), 1e-30)
    y_scale = torch.tensor([1 / sy, sy], device=cuda)
    dx_scale = torch.tensor([1 / sdx, sdx], device=cuda)
    qy = torch.empty(n, C, dtype=torch.uint8, device=cuda)
    y_slot, dx_slot = torch.zeros(1, device=cuda), torch.zeros(1, device=cuda)
    grad = types.SimpleNamespace(scale=dx_scale, slot=dx_slot, shadow=None)
    step = _BnStep(None, None, (qy, y_scale, y_slot), grad)
    got = _bn_run(ME, x0, res0, relu, step)
    for k, v in plain.items():
        assert (v is None and got[k] is None) or torch.equal(v, got[k]), k
    assert step.written
    assert torch.equal(qy, _expect(got["y"], y_scale[1], "e4m3"))
    assert float(y_slot) == _finite_amax(got["y"])
    qdx, ptr, shape, version = grad.shadow
    assert ptr == got["dx"].data_ptr() and shape == got["dx"].shape
    assert torch.equal(qdx, _expect(got["dx"], dx_scale[1], "e5m2"))
    assert float(dx_slot) == _finite_amax(got["dx"])


class _OneRankPeer:
    """A one-rank statistics exchange in device memory, laid out as _PeerExchange's symmetric
    buffer: drives the peer entries (meb200_bn_forward_train_peer[_q], ..._backward_reduce_peer) on
    one GPU."""

    def __init__(self, dev):
        from minkowskiengine_b200.normalization import _PeerExchange
        self.SLOTS, self.SLOT_DOUBLES = _PeerExchange.SLOTS, _PeerExchange.SLOT_DOUBLES
        self.buf = torch.zeros(1024 + self.SLOTS * self.SLOT_DOUBLES * 8, dtype=torch.uint8,
                               device=dev)
        self.bases = torch.tensor([self.buf.data_ptr()], dtype=torch.int64, device=dev)
        self.bases_dev, self.rank, self.world, self.seq = self.bases.data_ptr(), 0, 1, 0
        self.next_slot_offset = types.MethodType(_PeerExchange.next_slot_offset, self)


@pytest.fixture(params=["peer", "all_reduce"])
def sync_route(request, cuda, monkeypatch):
    """A synchronised batch norm of one rank on the peer exchange or on the all-reduce fallback
    (meb200_bn_stats_to, _finalize, _apply_fused[_q]); returns the group to pass."""
    from minkowskiengine_b200 import normalization as N
    if request.param == "peer":
        peer = _OneRankPeer(cuda)
        monkeypatch.setattr(N, "_USE_PEER", True)
        monkeypatch.setattr(N._PeerExchange, "get", classmethod(lambda cls, g, d: peer))
    else:
        monkeypatch.setattr(N, "_USE_PEER", False)
        monkeypatch.setattr(torch.distributed, "all_reduce", lambda t, group=None: None)
    return object()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=str)
@pytest.mark.parametrize("n,C", [(0, 32), (1, 8), (12_345, 96), (777, 256), (200_003, 8)],
                         ids=lambda v: str(v))
def test_bn_shadows_synchronised_routes(ME, cuda, sync_route, n, C, dtype):
    """The _q entries of the synchronised routes, a rank without rows included: every output of the
    pass without the copy, bit for bit, and the copies and amaxes as in test_bn_shadows."""
    from minkowskiengine_b200.fp8_delayed import _BnStep
    g = torch.Generator(device=cuda).manual_seed(n + C)
    x0 = (torch.randn(n, C, generator=g, device=cuda) * 2 + 0.5).to(dtype)
    res0 = torch.randn(n, C, generator=g, device=cuda).to(dtype)
    plain = _bn_run(ME, x0, res0, True, None, group=sync_route)
    y_scale = torch.tensor([1 / 64.0, 64.0], device=cuda)
    dx_scale = torch.tensor([1 / 4096.0, 4096.0], device=cuda)
    qy = torch.empty(n, C, dtype=torch.uint8, device=cuda)
    y_slot, dx_slot = torch.zeros(1, device=cuda), torch.zeros(1, device=cuda)
    grad = types.SimpleNamespace(scale=dx_scale, slot=dx_slot, shadow=None)
    step = _BnStep(None, None, (qy, y_scale, y_slot), grad)
    got = _bn_run(ME, x0, res0, True, step, group=sync_route)
    for k, v in plain.items():          # as bytes: a global row count of 0 gives NaN statistics
        assert torch.equal(v.contiguous().view(torch.uint8), got[k].contiguous().view(torch.uint8)), k
    assert step.written
    assert torch.equal(qy, _expect(got["y"], y_scale[1], "e4m3"))
    assert float(y_slot) == _finite_amax(got["y"])
    if n > 0:
        assert torch.equal(grad.shadow[0], _expect(got["dx"], dx_scale[1], "e5m2"))
        assert float(dx_slot) == _finite_amax(got["dx"])


# ---- saturation ---------------------------------------------------------------------------------
@pytest.mark.parametrize("role", ["input", "grad_output"])
@pytest.mark.parametrize("H", [1, 4])
def test_saturation_and_the_next_scale(ME, cuda, H, role):
    """A tensor 16 times the history's amax saturates to +-448 (the e4m3 input) or +-57344 (the
    e5m2 output gradient); the next step's scale covers it."""
    net = torch.nn.Sequential(ME.MinkowskiConvolution(32, 32, kernel_size=3, dimension=3)).to(cuda)
    rec = ME.Fp8DelayedScaling(net, history=H)
    x = torch.randn(1000, 32, device=cuda)
    a = _finite_amax(x)
    _, dt, M = FMTS["e4m3" if role == "input" else "e5m2"]

    def operand(t):
        with ME.fp8_training(scaling=rec):
            layer = rec._conv_begin(net[0], types.SimpleNamespace(F=x))
        return layer.act if role == "input" else layer.grad.operand(t)

    def forward_operand(t):
        with ME.fp8_training(scaling=rec):
            return rec._conv_begin(net[0], types.SimpleNamespace(F=t)).act

    op = forward_operand if role == "input" else operand
    op(x)                                                # step 0: dynamic, records a
    q, s = op(x)                                         # step 1: the scale of a
    assert float(s[1]) == float(np.float32(M) / np.float32(a))
    q, s = op(16 * x)                                    # step 2: saturates
    f = q.view(dt).float()
    assert float(f.abs().max()) == M and int((f.abs() == M).sum()) > 1
    q, s = op(x)                                         # step 3: covers 16 a
    assert float(s[1]) == float(np.float32(M) / np.float32(16 * a))


# ---- empty inputs -----------------------------------------------------------------------------------
def test_empty_input_every_step(ME, cuda):
    """A layer whose input has no rows, over its dynamic first step and the delayed ones after it:
    operands without a launch, an all-zero output on an output map with rows."""
    from minkowskiengine_b200 import backend
    net = torch.nn.Sequential(ME.MinkowskiConvolution(64, 32, kernel_size=3, dimension=3)).to(cuda)
    rec = ME.Fp8DelayedScaling(net)
    none = lambda *s: torch.full(s, -1, dtype=torch.int32, device=cuda)     # noqa: E731
    km = backend._KernelMap(none(27, 40), none(27, 0))                    # no input rows
    w = net[0].kernel.detach()
    for step in range(3):
        x = torch.zeros(0, 64, device=cuda).bfloat16()
        with ME.fp8_training(scaling=rec, weight_gradient=True):
            layer = rec._conv_begin(net[0], types.SimpleNamespace(F=x))
            q, sc = layer.act
            assert q.shape == (0, 64) and sc.shape == (2,)
            y = backend._conv_forward(x, w, km, fp8=True, act=layer.act)
        assert y.shape == (40, 32) and not y.any(), step
        g = torch.zeros(0, 32, device=cuda).bfloat16()
        gq, gs = layer.grad.operand(g)
        assert gq.shape == (0, 32) and gs.shape == (2,)
    torch.cuda.synchronize()


# ---- a step without host synchronisation -----------------------------------------------------------
def test_step_does_not_synchronise(ME, cuda):
    from examples.synthetic import surface_cloud

    class Net(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.c1 = ME.MinkowskiConvolution(32, 64, kernel_size=3, dimension=3)
            self.n1 = ME.MinkowskiBatchNorm(64)
            self.c2 = ME.MinkowskiConvolution(64, 32, kernel_size=3, dimension=3)
            self.n2 = ME.MinkowskiBatchNorm(32)

        def forward(self, x):
            return ME.fused_bn_relu(self.n2, self.c2(ME.fused_bn_relu(self.n1, self.c1(x))))

    torch.manual_seed(0)
    net = Net().to(cuda)
    rec = ME.Fp8DelayedScaling(net)
    coords = surface_cloud(20_000, 0, batch=0).to(cuda)
    x = ME.SparseTensor(torch.randn(len(coords), 32, device=cuda).bfloat16().requires_grad_(True),
                        coords)

    def step():
        with ME.fp8_training(scaling=rec, weight_gradient=True):
            out = net(x)
        out.F.float().square().sum().backward()

    for _ in range(3):                                  # maps and packs built, links recorded
        step()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        step()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()


# ---- layers: the operands and the products of fp8_training() ----------------------------------------
class _Calls:
    """Records the fp8 forward, dgrad and wgrad calls of the layers (arguments and results)."""

    def __init__(self, ME, monkeypatch):
        B = ME.backend
        self.orig = {n: getattr(B, n) for n in ("_conv_forward_fp8", "_conv_dgrad_fp8",
                                                 "_conv_wgrad_fp8")}
        self.calls = []
        for n, fn in self.orig.items():
            monkeypatch.setattr(B, n, self._wrap(n, fn))

    def _wrap(self, name, fn):
        def call(*args, **kw):
            out = fn(*args, **kw)
            self.calls.append((name, args, kw, out))
            return out
        return call


def test_layers_equal_fp8_training_on_their_operands(ME, cuda, monkeypatch):
    """Steps 1-2 of conv -> fused_bn_relu -> conv -> fused_bn_relu under delayed scaling: every
    forward, dgrad and fp8 wgrad receives its operands as (bytes, scale), the bytes are the torch
    expression of the tensor it multiplies at that scale (e4m3 input, e5m2 output gradient, whether
    a batch norm or the layer wrote them), each product equals _conv_forward_fp8 / _conv_dgrad_fp8
    / _conv_wgrad_fp8 on the same operands bit for bit, and the forward and dgrad are within the
    n * 2^-13 * A bounds of fp8_training() against float64 of those operands."""
    from examples.synthetic import surface_cloud
    from helpers import _pairs, half_ulp, ref_conv
    B = ME.backend

    class Net(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.c1 = ME.MinkowskiConvolution(32, 64, kernel_size=3, dimension=3)
            self.n1 = ME.MinkowskiBatchNorm(64)
            self.c2 = ME.MinkowskiConvolution(64, 32, kernel_size=3, stride=2, dimension=3)
            self.n2 = ME.MinkowskiBatchNorm(32)

        def forward(self, x):
            return ME.fused_bn_relu(self.n2, self.c2(ME.fused_bn_relu(self.n1, self.c1(x))))

    torch.manual_seed(0)
    net = Net().to(cuda)
    rec = ME.Fp8DelayedScaling(net)
    coords = surface_cloud(30_000, 1, batch=0).to(cuda)
    feats = torch.randn(len(coords), 32, device=cuda).bfloat16()
    calls = _Calls(ME, monkeypatch)
    worst = 0.0
    for step in range(3):
        calls.calls.clear()
        x = ME.SparseTensor(feats.clone().requires_grad_(True), coords)
        with ME.fp8_training(scaling=rec, weight_gradient=True):
            out = net(x)
        out.F.float().square().sum().backward()
        if step == 0:
            continue
        names = [c[0] for c in calls.calls]
        assert names.count("_conv_forward_fp8") == names.count("_conv_dgrad_fp8") == 2
        assert names.count("_conv_wgrad_fp8") == 2
        for name, args, kw, out_t in calls.calls:
            if name == "_conv_forward_fp8":
                in_feat, kernel, km, epi = args[:4]
                act = kw.get("act", args[4] if len(args) > 4 else None)
                assert act is not None
                assert torch.equal(act[0], _expect(in_feat, act[1][1], "e4m3"))
                assert torch.equal(out_t, calls.orig[name](in_feat, kernel, km, epi, act))
                w_t, w_scale = B._fp8_weights(kernel)
                xd = act[0].view(torch.float8_e4m3fn).double() * act[1][0].double()
                wd = w_t.view(torch.float8_e4m3fn).double().transpose(1, 2) * w_scale.double()
                ref, A = ref_conv(xd, wd, _pairs(km.out_nbr), km.n_out)
                steps = km.K * in_feat.shape[1] // 32
            elif name == "_conv_dgrad_fp8":
                grad_out, kernel, km, dtype = args[:4]
                grad_q = kw.get("grad_q", args[4] if len(args) > 4 else None)
                assert grad_q is not None
                assert torch.equal(grad_q[0], _expect(grad_out, grad_q[1][1], "e5m2"))
                assert torch.equal(out_t, calls.orig[name](grad_out, kernel, km, dtype, grad_q))
                w_c, w_scale = B._fp8_dgrad_weights(kernel)
                gd = grad_q[0].view(torch.float8_e5m2).double() * grad_q[1][0].double()
                wd = w_c.view(torch.float8_e4m3fn).double() * w_scale.double()[None, :, None]
                ref, A = ref_conv(gd, wd.transpose(1, 2), _pairs(km.in_nbr), km.n_in)
                steps = km.K * grad_out.shape[1] // 32
            else:
                act, grad_q, kernel, km = args
                assert torch.equal(out_t, calls.orig[name](act, grad_q, kernel, km))
                continue
            bound = A * (steps * 2.0 ** -13) + 2.0 ** -21 * ref.abs()
            bound = half_ulp(ref.abs() + bound, out_t.dtype) + bound
            err = (out_t.double() - ref).abs()
            ratio = float((err / bound.clamp(min=1e-300)).max())
            assert bool((err <= bound).all()), (name, step, ratio)
            worst = max(worst, ratio)
    print(f"worst err / bound over the forwards and dgrads of steps 1-2: {worst:.3f}")


# ---- MinkUNet training steps ------------------------------------------------------------------------
class _Count:
    """Counts the conversions the layers make, by route, while active."""

    def __init__(self, ME, monkeypatch):
        B = ME.backend
        self.n = {"record_e4m3": 0, "record_e5m2": 0, "dynamic": 0}
        rec_fn, dyn_fn = B.quantize_fp8_record, B._quantize_dynamic

        def record(feat, fmt, scale, slot):
            self.n["record_e5m2" if fmt else "record_e4m3"] += 1
            return rec_fn(feat, fmt, scale, slot)

        def dynamic(feat, entry):
            self.n["dynamic"] += 1
            return dyn_fn(feat, entry)
        monkeypatch.setattr(B, "quantize_fp8_record", record)
        monkeypatch.setattr(B, "_quantize_dynamic", dynamic)

    def take(self):
        out = dict(self.n)
        for k in self.n:
            self.n[k] = 0
        return out


def _cfg3(cuda):
    from examples.synthetic import surface_cloud
    coords = torch.cat([surface_cloud(100_000, j, batch=j) for j in range(8)], 0)
    feats = torch.rand(len(coords), 3, generator=torch.Generator().manual_seed(0))
    labels = torch.zeros(len(coords), dtype=torch.int64)
    return coords.to(cuda), feats.to(cuda).bfloat16(), labels.to(cuda)


def _step(ME, net, opt, batch, scaling=None, fp8=True):
    coords, feats, labels = batch
    opt.zero_grad(set_to_none=True)
    ctx = ME.fp8_training(weight_gradient=True, scaling=scaling) if fp8 else \
        contextlib.nullcontext()
    with ctx:
        out = net(ME.SparseTensor(feats, coords))
        loss = torch.nn.functional.cross_entropy(out.F.float(), labels)
    loss.backward()
    grads = {n: p.grad.detach().clone() for n, p in net.named_parameters() if p.grad is not None}
    opt.step()
    return loss.detach(), grads


class _Structure:
    """Counts, from the layers as they run, the convolutions fp8_training() selects and those whose
    input is the output of a training batch norm (fused_bn_relu or a batch-norm module) that no
    other selected convolution reads."""

    def __init__(self, ME, monkeypatch):
        from minkowskiengine_b200 import convolution as CV
        from minkowskiengine_b200 import normalization as N
        self.bn_out, self.readers = {}, {}     # held until take(): ids are not reused meanwhile
        self.selected = 0
        bn_tail, conv_fwd, bn_fwd = N._bn_tail, CV.MinkowskiConvolutionBase.forward, \
            N.MinkowskiBatchNorm.forward

        def tail(norm, input, residual, relu):
            out = bn_tail(norm, input, residual, relu)
            self.bn_out[id(out.F)] = out.F
            return out

        def bn_module(module, input):
            out = bn_fwd(module, input)
            self.bn_out[id(out.F)] = out.F
            return out

        def conv(layer, input, coordinates=None):
            if CV._fp8_train(layer, input.F):
                self.selected += 1
                if id(input.F) in self.bn_out:
                    self.readers.setdefault(id(input.F), []).append(layer)
            return conv_fwd(layer, input, coordinates)
        for mod in (N, CV):
            monkeypatch.setattr(mod, "_bn_tail", tail)
        monkeypatch.setattr(N.MinkowskiBatchNorm, "forward", bn_module)
        monkeypatch.setattr(CV.MinkowskiConvolutionBase, "forward", conv)

    def take(self):
        fed = sum(1 for r in self.readers.values() if len(r) == 1)
        out = (self.selected, fed)
        self.bn_out, self.readers, self.selected = {}, {}, 0
        return out


def test_minkunet34c_steps(ME, cuda, monkeypatch):
    from examples.minkunet import minkunet
    batch = _cfg3(cuda)
    torch.manual_seed(0)
    net = minkunet("MinkUNet34C", ME, 3, 20, 3).to(cuda)
    state = {k: v.clone() for k, v in net.state_dict().items()}
    opt = torch.optim.SGD(net.parameters(), lr=1e-2)
    dyn = [_step(ME, net, opt, batch) for _ in range(3)]

    net.load_state_dict(state)
    opt = torch.optim.SGD(net.parameters(), lr=1e-2)
    rec = ME.Fp8DelayedScaling(net, history=16)
    count = _Count(ME, monkeypatch)
    structure = _Structure(ME, monkeypatch)
    l0, g0 = _step(ME, net, opt, batch, rec)
    c0 = count.take()
    n_sel, n_fed = structure.take()
    assert torch.equal(l0, dyn[0][0])                            # step 0: fp8_training()'s
    assert g0.keys() == dyn[0][1].keys()
    assert all(torch.equal(g0[k], dyn[0][1][k]) for k in g0)
    assert c0 == {"record_e4m3": 0, "record_e5m2": 0, "dynamic": 2 * n_sel}   # e4m3 + e5m2 each
    l1, _ = _step(ME, net, opt, batch, rec)
    c1 = count.take()
    assert structure.take() == (n_sel, n_fed)
    print(f"selected {n_sel}, fed straight by a batch norm {n_fed}, step-1 conversions {c1}")
    # every layer fed straight by a batch norm reads its forward shadow, every layer reads its
    # gradient shadow, and the others convert their input in one launch
    assert c1 == {"record_e4m3": n_sel - n_fed, "record_e5m2": 0, "dynamic": 0}
    sd_model = {k: v.clone() for k, v in net.state_dict().items()}
    sd_opt = opt.state_dict()
    sd_rec = rec.state_dict()
    l2, g2 = _step(ME, net, opt, batch, rec)
    assert count.take() == c1
    for i, l in enumerate((l0, l1, l2)):
        rel = float((l - dyn[i][0]).abs() / dyn[i][0].abs())
        print(f"step {i} loss delayed {float(l):.6f} dynamic {float(dyn[i][0]):.6f} rel {rel:.2e}")
        assert rel < 2e-3
    # resume after step 1 into a fresh model and recipe: step 2 bit for bit
    torch.manual_seed(1)
    net2 = minkunet("MinkUNet34C", ME, 3, 20, 3).to(cuda)
    net2.load_state_dict(sd_model)
    opt2 = torch.optim.SGD(net2.parameters(), lr=1e-2)
    opt2.load_state_dict(sd_opt)
    rec2 = ME.Fp8DelayedScaling(net2, history=5)
    rec2.load_state_dict(sd_rec)
    l2b, g2b = _step(ME, net2, opt2, batch, rec2)
    assert torch.equal(l2b, l2) and all(torch.equal(g2b[k], g2[k]) for k in g2)


def test_minkunet14_fits_a_batch(ME, cuda):
    """40 SGD steps of MinkUNet14 on one fixed batch with delayed scaling: the loss falls by a fifth
    and ends near bf16's."""
    from examples.minkunet import minkunet
    from examples.synthetic import surface_cloud
    coords = torch.cat([surface_cloud(20_000, 50 + j, batch=j) for j in range(2)], 0).to(cuda)
    g = torch.Generator().manual_seed(3)
    feats = torch.rand(len(coords), 3, generator=g).to(cuda).bfloat16()
    labels = (coords[:, 1] // 8 % 4 + 4 * (feats[:, 0].float() > 0.5).long()).to(cuda)
    finals = {}
    for mode in ("bf16", "delayed"):
        torch.manual_seed(0)
        net = minkunet("MinkUNet14", ME, 3, 8, 3).to(cuda)
        opt = torch.optim.SGD(net.parameters(), lr=1e-2)
        rec = ME.Fp8DelayedScaling(net) if mode == "delayed" else None
        finals[mode] = torch.stack([_step(ME, net, opt, (coords, feats, labels), rec,
                                          fp8=rec is not None)[0] for _ in range(40)])
        print(f"MinkUNet14 {mode} loss: " + " ".join(f"{float(v):.4f}" for v in finals[mode][::5])
              + f" ... step 40: {float(finals[mode][-1]):.4f}")
    ld, lb = finals["delayed"], finals["bf16"]
    assert bool(torch.isfinite(ld).all())
    assert float(ld[-5:].mean()) < 0.8 * float(ld[:5].mean())
    assert float(ld[-1]) < float(lb[-1]) * 1.1 + 0.02
