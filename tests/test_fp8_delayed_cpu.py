"""fp8 training with delayed scaling without a GPU: the context and its steps, the recipe's
binding, arguments and checkpoints, the library calls of a conv -> batch norm -> conv chain over
steps 0-2 (a stub library records every call), the links that break, and the delayed scale formula
against float64 at its edges."""
import threading

import numpy as np
import pytest
import torch

import minkowskiengine_b200 as ME
from minkowskiengine_b200 import _lib
from minkowskiengine_b200 import backend as B
from minkowskiengine_b200 import fp8_delayed as FD
from minkowskiengine_b200.normalization import _BatchNormFunction

E4M3_MAX, E5M2_MAX = 448.0, 57344.0
FLT_MAX = np.finfo(np.float32).max


class _Net(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.conv1 = ME.MinkowskiConvolution(32, 32, kernel_size=3, dimension=3)
        self.norm = ME.MinkowskiBatchNorm(32)
        self.conv2 = ME.MinkowskiConvolution(32, 64, kernel_size=3, dimension=3)
        self.conv3 = ME.MinkowskiConvolution(32, 64, kernel_size=3, dimension=3)


# ---- the context ---------------------------------------------------------------------------------
def test_none_is_todays_path():
    with ME.fp8_training(scaling=None):
        assert B.fp8_training_enabled() and B.fp8_training_scaling() is None
        assert not B.fp8_training_weight_gradient()
    with ME.fp8_training(weight_gradient=True):
        assert B.fp8_training_scaling() is None and B.fp8_training_weight_gradient()
    assert B.fp8_training_scaling() is None and not B.fp8_training_enabled()


def test_blocks_nest_innermost_decides_and_steps_count_outermost_blocks():
    net = _Net()
    a, b = ME.Fp8DelayedScaling(net), ME.Fp8DelayedScaling(net)
    assert a._step == -1
    with ME.fp8_training(scaling=a, weight_gradient=True):
        assert a._step == 0 and B.fp8_training_scaling() is a
        with ME.fp8_training():
            assert B.fp8_training_scaling() is None and not B.fp8_training_weight_gradient()
            with ME.fp8_training(scaling=a):          # nested in a block of a: the same step
                assert a._step == 0 and B.fp8_training_scaling() is a
        with ME.fp8_training(scaling=b):
            assert b._step == 0 and a._step == 0 and B.fp8_training_scaling() is b
        assert B.fp8_training_scaling() is a and B.fp8_training_weight_gradient()
    for step in (1, 2):
        with ME.fp8_training(scaling=a):
            assert a._step == step
    assert b._step == 0 and B.fp8_training_scaling() is None


def test_thread_local_and_survives_exceptions():
    rec = ME.Fp8DelayedScaling(_Net())
    seen = []
    with pytest.raises(KeyError):
        with ME.fp8_training(scaling=rec):
            t = threading.Thread(target=lambda: seen.append(B.fp8_training_scaling()))
            t.start()
            t.join()
            raise KeyError
    assert seen == [None] and B.fp8_training_scaling() is None and not B.fp8_training_enabled()


# ---- the recipe ----------------------------------------------------------------------------------
def test_binds_to_qualified_names():
    net = _Net()
    rec = ME.Fp8DelayedScaling(net, history=4, margin=2)
    assert list(rec._index) == ["conv1", "conv2", "conv3"]
    assert rec._names[id(net.norm)] == "norm" and (rec.history, rec.margin) == (4, 2)
    stranger = ME.MinkowskiConvolution(32, 32, kernel_size=3, dimension=3)
    assert rec._conv_begin(stranger, _St(torch.randn(10, 32))) is None    # the dynamic path


@pytest.mark.parametrize("kw", [{"history": 0}, {"history": _lib.FP8_MAX_HISTORY + 1},
                                {"history": 2.0}, {"history": True}, {"margin": -1},
                                {"margin": 0.5}, {"margin": 128}, {"margin": None}],
                         ids=lambda k: repr(k))
def test_bad_arguments_raise(kw):
    with pytest.raises(ValueError):
        ME.Fp8DelayedScaling(_Net(), **kw)


def test_limits_are_accepted():
    ME.Fp8DelayedScaling(_Net(), history=1, margin=0)
    ME.Fp8DelayedScaling(_Net(), history=_lib.FP8_MAX_HISTORY, margin=127)


# ---- a stub library -------------------------------------------------------------------------------
class _Stub:
    """Records every call and returns success; the dynamic quantisations write fixed scales."""

    def __init__(self, calls):
        self.calls = calls

    def __getattr__(self, name):
        def fn(*args):
            self.calls.append((name, args))
            return 0
        return fn


@pytest.fixture
def stub(monkeypatch):
    calls = []
    monkeypatch.setattr(_lib, "load", lambda: _Stub(calls))
    monkeypatch.setattr(_lib, "current_stream", lambda: None)
    monkeypatch.setattr(B, "_QUANT_WS", {})
    return calls


class _St:
    """The part of a SparseTensor the recipe's hooks read: .F, and attributes set on it."""

    def __init__(self, F):
        self.F = F


def _names(calls):
    return [c[0] for c in calls if not c[0].endswith("_workspace_bytes")]


def _bn(norm, st, rec):
    """A training batch norm on st through the native function, as _bn_tail runs it."""
    fp8 = rec._bn_begin(norm, st)
    bn = norm.bn
    y = _BatchNormFunction.apply(st.F, bn.weight, bn.bias, bn.running_mean, bn.running_var,
                                 bn.momentum, bn.eps, None, False, None, False, None, fp8)
    out = _St(y)
    if fp8 is not None:
        rec._bn_end(fp8, out)
    return out


def _chain(net, rec, x, stub, consumers=("conv2",), between=None):
    """One step of conv1 -> norm -> consumers, backward through norm: the calls of each part."""
    marks = {}
    with ME.fp8_training(scaling=rec, weight_gradient=True):
        n0 = len(stub)
        l1 = rec._conv_begin(net.conv1, _St(x))
        h = _St(torch.randn(10, 32, requires_grad=True))
        rec._tag(h, l1)
        marks["conv1"] = _names(stub[n0:])
        n0 = len(stub)
        y = _bn(net.norm, h, rec)
        marks["bn"] = _names(stub[n0:])
        if between is not None:
            y = between(y)
        for c in consumers:
            n0 = len(stub)
            rec._conv_begin(getattr(net, c), y)
            marks[c] = _names(stub[n0:])
    n0 = len(stub)
    dx = torch.autograd.grad(y.F.sum(), h.F)[0]
    marks["bn_backward"] = _names(stub[n0:])
    n0 = len(stub)
    l1.grad.operand(dx.contiguous())
    marks["conv1_backward"] = _names(stub[n0:])
    return marks


DYN_E4M3 = ["meb200_quantize_e4m3", "meb200_amax_accumulate"]
DYN_E5M2 = ["meb200_quantize_e5m2", "meb200_amax_accumulate"]
ROLL = ["meb200_fp8_roll"]


def test_step0_is_dynamic_then_shadows(stub):
    """Step 0: the dynamic conversions of fp8_training() (each recording its amax), plain batch-norm
    passes.  From step 1: the linked batch norm calls its _q entries forward and backward, and
    neither convolution it feeds or is fed by converts; the first layer converts in one launch."""
    net = _Net()
    rec = ME.Fp8DelayedScaling(net)
    x = torch.randn(10, 32)
    m0 = _chain(net, rec, x, stub)
    assert m0["conv1"] == ROLL + DYN_E4M3
    assert m0["bn"] == ["meb200_bn_forward_train"]
    assert m0["bn_backward"] == ["meb200_bn_backward_reduce_to", "meb200_bn_backward_apply_fused"]
    assert m0["conv2"] == DYN_E4M3 and m0["conv1_backward"] == DYN_E5M2
    for step in (1, 2):
        m = _chain(net, rec, x, stub)
        assert m["conv1"] == ROLL + ["meb200_quantize_fp8_record"]
        assert m["bn"] == ["meb200_bn_forward_train_q"]
        assert m["conv2"] == []                                    # the forward shadow
        assert m["bn_backward"] == ["meb200_bn_backward_reduce_to",
                                    "meb200_bn_backward_apply_fused_q"]
        assert m["conv1_backward"] == []                           # the gradient shadow
    assert len([c for c in stub if c[0] == "meb200_fp8_roll"]) == 3    # one per step and device


def test_unlinked_consumer_converts_once(stub):
    net = _Net()
    rec = ME.Fp8DelayedScaling(net)
    x = torch.randn(10, 32)
    _chain(net, rec, x, stub)
    with ME.fp8_training(scaling=rec):
        n0 = len(stub)
        rec._conv_begin(net.conv3, _St(torch.randn(10, 32)))      # its first step
        assert _names(stub[n0:]) == ROLL + DYN_E4M3
    with ME.fp8_training(scaling=rec):
        n0 = len(stub)
        rec._conv_begin(net.conv3, _St(torch.randn(10, 32)))
        assert _names(stub[n0:]) == ROLL + ["meb200_quantize_fp8_record"]


def _cat(y):
    return _St(torch.cat([y.F[:5], y.F[5:]]))       # a new tensor (ME.cat, an activation module)


def _bump(y):
    with torch.no_grad():
        y.F.add_(0)                                    # modified in place after the shadow
    return y


@pytest.mark.parametrize("what", ["cat", "two_consumers", "stale_version"])
def test_broken_links_fall_back(stub, what):
    net = _Net()
    rec = ME.Fp8DelayedScaling(net)
    x = torch.randn(10, 32)
    kw = {"cat": {"between": _cat}, "two_consumers": {"consumers": ("conv2", "conv3")},
          "stale_version": {}}[what]
    for step in range(3):
        if what == "stale_version" and step == 2:
            kw = {"between": _bump}
        m = _chain(net, rec, x, stub, **kw)
        bn_q = m["bn"] == ["meb200_bn_forward_train_q"]
        if step == 0:
            assert m["conv2"] == DYN_E4M3
        elif what == "stale_version":
            assert bn_q                                  # the link holds ...
            assert m["conv2"] == ([] if step == 1 else ["meb200_quantize_fp8_record"])
        else:
            assert not bn_q and m["conv2"] == ["meb200_quantize_fp8_record"]
        if what == "two_consumers" and step > 0:
            assert m["conv3"] == ["meb200_quantize_fp8_record"]


def test_state_dict_round_trip(stub):
    net = _Net()
    rec = ME.Fp8DelayedScaling(net, history=3, margin=1)
    x = torch.randn(10, 32)
    for _ in range(2):
        _chain(net, rec, x, stub)
    ds = rec._dev[torch.device("cpu")]
    ds.hist.copy_(torch.arange(ds.hist.numel(), dtype=torch.float32).reshape(ds.hist.shape))
    ds.cur.copy_(torch.arange(ds.cur.numel(), dtype=torch.float32) + 0.5)
    sd = rec.state_dict()
    assert sd["history"] == 3 and sd["margin"] == 1 and sd["step"] == 1
    assert sd["links"] == {"norm": ["conv2"]}
    assert sd["entries"]["conv1"]["input"]["first_step"] == 0
    assert sd["entries"]["conv3"]["input"]["first_step"] is None
    assert sd["entries"]["conv2"]["grad_output"]["amax"].shape == (4,)
    net2 = _Net()
    fresh = ME.Fp8DelayedScaling(net2)
    fresh.load_state_dict(sd)
    sd2 = fresh.state_dict()
    assert sd2.keys() == sd.keys() and sd2["links"] == sd["links"] and sd2["step"] == 1
    for name, ent in sd["entries"].items():
        for role in FD.ROLES:
            assert torch.equal(sd2["entries"][name][role]["amax"], ent[role]["amax"])
            assert sd2["entries"][name][role]["first_step"] == ent[role]["first_step"]
    # the next step of the fresh recipe rolls the loaded state and uses the saved link
    m = _chain(net2, fresh, x, stub)
    with pytest.raises(KeyError):
        ME.Fp8DelayedScaling(torch.nn.Sequential(net.conv1)).load_state_dict(sd)
    assert m["conv1"] == ROLL + ["meb200_quantize_fp8_record"]


# ---- the delayed scale formula --------------------------------------------------------------------
def delayed_scales(history, margin, kmax):
    """(scale, inv) of k_fp8_roll in fp32: amax = max of the history, a = min(amax * 2^margin,
    FLT_MAX), then the per-tensor formula (numpy rounds fp32 divisions to nearest)."""
    amax = np.float32(max(history))
    with np.errstate(over="ignore"):
        a = np.float32(min(np.float32(np.ldexp(amax, margin)), FLT_MAX))
        if a == 0:
            return np.float32(1), np.float32(1)
        inv = np.float32(kmax) / a
    if np.isinf(inv):
        return np.float32(1) / FLT_MAX, FLT_MAX
    return a / np.float32(kmax), inv


@pytest.mark.parametrize("kmax", [E4M3_MAX, E5M2_MAX], ids=["e4m3", "e5m2"])
@pytest.mark.parametrize("history,margin", [
    ([0.0] * 16, 0), ([0.0] * 16, 5), ([1e-45], 0), ([1e-45, 0.0], 3), ([1e-40, 2e-41], 0),
    ([3.0, 7.5, 1.0], 0), ([3.0, 7.5, 1.0], 4), ([2.0], 0), ([FLT_MAX], 0), ([FLT_MAX], 1),
    ([1e38, 1.0], 2), ([448.0], 127), ([1e-30] * 4, 0)],
    ids=lambda v: str(v)[:24])
def test_delayed_scales_against_float64(history, margin, kmax):
    """scale and inv are the fp32 roundings of the float64 quotients of kmax and the scaled amax,
    except at amax = 0 (both 1), where amax * 2^margin passes FLT_MAX (FLT_MAX is used) and where
    kmax / amax overflows fp32 (inv = FLT_MAX, scale = 1 / FLT_MAX)."""
    s, inv = delayed_scales([np.float32(h) for h in history], margin, kmax)
    a = max(float(np.float32(h)) for h in history) * 2.0 ** margin
    a = min(a, float(FLT_MAX))
    if a == 0:
        assert (s, inv) == (1, 1)
        return
    q = kmax / a
    if q >= float(FLT_MAX) * (1 + 2 ** -25):
        assert inv == FLT_MAX and s == np.float32(1 / float(FLT_MAX))
        return
    assert inv == np.float32(q) and s == np.float32(a / kmax)
    assert abs(float(s) * float(inv) - 1) <= 2 ** -22


@pytest.mark.parametrize("margin", [-1, 128])
def test_load_state_dict_rejects_a_bad_margin(stub, margin):
    net = _Net()
    rec = ME.Fp8DelayedScaling(net)
    _chain(net, rec, torch.randn(10, 32), stub)
    sd = rec.state_dict()
    sd["margin"] = margin
    with pytest.raises(ValueError):
        ME.Fp8DelayedScaling(_Net()).load_state_dict(sd)


def test_linked_batch_norm_without_rows_writes_no_copy(stub):
    """A rank or batch without rows: the linked batch norm passes no fp8 output (its entries would
    see a NULL buffer), and the consumer's operand needs no launch."""
    net = _Net()
    rec = ME.Fp8DelayedScaling(net)
    x = torch.randn(10, 32)
    _chain(net, rec, x, stub)
    with ME.fp8_training(scaling=rec):
        rec._conv_begin(net.conv1, _St(x))
        bn = rec._bn_begin(net.norm, _St(torch.zeros(0, 32)))
        assert bn is not None and bn.y_out is None
