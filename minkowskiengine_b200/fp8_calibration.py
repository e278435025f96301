"""Static activation scales for fp8 inference (DESIGN.md §3).

Fp8Calibration(model) records, over eval forwards run inside its observe() block, the amax of the
input of every layer fp8_inference() would run on e4m3 operands, and which layers feed one of them
directly (links).  Inside fp8_inference(calibration):
- a calibrated layer quantises its input with the static scale of its amax: one conversion launch,
  no amax pass, and a result for one cloud that does not depend on the clouds batched with it;
- a layer that fed a calibrated one also writes, in the launch that writes its output, the e4m3
  copy of that output at the consumer's scale (the shadow), which the consumer then reads in place
  of converting its input.
"""
import contextlib

import torch

from . import backend as _C

_SHADOW = "_fp8_shadow"        # SparseTensor attribute: (q, scale, features, features' _version)
_PRODUCER = "_fp8_producer"    # SparseTensor attribute while observing: (calibration, name)


def module_names(model):
    """{id(module): qualified name} of every module of `model` (a module reached twice keeps its
    first name): how the fp8 recipes bind to a model's layers."""
    names = {}
    for name, m in model.named_modules():
        names.setdefault(id(m), name)
    return names


class Fp8Calibration:
    """Static e4m3 scales for the convolutions of `model`, keyed by their qualified module names.

        calib = ME.Fp8Calibration(model)
        with torch.no_grad(), calib.observe():
            for x in calibration_batches:
                model(x)
        with torch.no_grad(), ME.fp8_inference(calib):
            y = model(x)

    A consumer is a MinkowskiConvolution, MinkowskiConvolutionTranspose,
    MinkowskiGenerativeConvolutionTranspose or the convolution of fused_conv_bn_relu that
    fp8_inference() would run on e4m3 operands.  A link is a convolution (or fused_conv_bn_relu
    call) whose returned SparseTensor is itself the input of a consumer: anything in between (ME.cat,
    an activation module, a new SparseTensor) breaks it, and the consumer then converts its input
    with its static scale.  The scale of a layer's shadow is that of the largest amax among the
    consumers it fed."""

    def __init__(self, model):
        self._names = module_names(model)
        self._amax = {}          # consumer name -> fp32 [1] amax (on the device it was observed on)
        self._feeds = {}         # producer name -> set of consumer names
        self._scales = {}        # (kind, name, device) -> fp32 [2] (scale, inv) on the device

    # ---- calibration ---------------------------------------------------------------------------
    @contextlib.contextmanager
    def observe(self):
        """Within the block, the forwards of this thread run exactly as they do outside fp8 and
        every consumer adds its input's amax (over the finite values, on the device, no host read)
        to its running amax; links are recorded as they are seen."""
        if _C.fp8_enabled():
            raise RuntimeError("Fp8Calibration.observe() inside fp8_inference(): observe the "
                               "layers as they run outside fp8")
        if _C.fp8_observer() is not None:
            raise RuntimeError("Fp8Calibration.observe() blocks do not nest")
        self._scales.clear()
        _C._FP8_STATE.observing = self
        try:
            yield self
        finally:
            _C._FP8_STATE.observing = None
            self._scales.clear()

    def state_dict(self):
        """{qualified module name: {"amax": fp32 0-d CPU tensor or None, "feeds": [consumer
        names]}} for every calibrated layer and every producer."""
        out = {}
        for name in sorted(set(self._amax) | set(self._feeds)):
            a = self._amax.get(name)
            out[name] = {"amax": None if a is None else a.detach().reshape(()).cpu().clone(),
                         "feeds": sorted(self._feeds.get(name, ()))}
        return out

    def load_state_dict(self, state):
        """Replaces the calibration by `state` (from state_dict()); every name must be a module of
        the bound model."""
        known = set(self._names.values())
        missing = [n for n in state if n not in known]
        if missing:
            raise KeyError(f"Fp8Calibration.load_state_dict: no module named {missing[0]!r}")
        amax, feeds = {}, {}
        for name, ent in state.items():
            if ent.get("amax") is not None:
                amax[name] = torch.as_tensor(ent["amax"], dtype=torch.float32).reshape(1).clone()
            if ent.get("feeds"):
                feeds[name] = set(ent["feeds"])
        self._amax, self._feeds = amax, feeds
        self._scales.clear()

    # ---- hooks of the convolution layers ---------------------------------------------------------
    def _observe(self, conv, input, selected):
        """Before `conv` runs on `input` while observing: a selected consumer's amax and link."""
        name = self._names.get(id(conv))
        if name is None or not selected:
            return
        feats = input.F.contiguous()
        amax = self._amax.get(name)
        if amax is None or amax.device != feats.device:
            amax = torch.zeros(1, dtype=torch.float32, device=feats.device) if amax is None \
                else amax.to(feats.device)
            self._amax[name] = amax
        _C.amax_accumulate(feats, amax)
        tag = getattr(input, _PRODUCER, None)
        if tag is not None and tag[0] is self:
            self._feeds.setdefault(tag[1], set()).add(name)

    def _tag(self, conv, out):
        """After `conv` (a route that can write a shadow) returned `out` while observing."""
        name = self._names.get(id(conv))
        if name is not None:
            setattr(out, _PRODUCER, (self, name))

    def _scale(self, kind, name, amaxes, device):
        key = (kind, name, device)
        s = self._scales.get(key)
        if s is None:
            a = [x.to(device) for x in amaxes]
            s = self._scales[key] = _C.e4m3_scales(a[0] if len(a) == 1 else torch.stack(a).amax(0))
        return s

    def _input_scale(self, conv, device):
        """A calibrated consumer's static scale, or None (uncalibrated: the dynamic path)."""
        name = self._names.get(id(conv))
        amax = self._amax.get(name) if name is not None else None
        return None if amax is None else self._scale("in", name, [amax], device)

    def _shadow_scale(self, conv, device):
        """The scale of the shadow `conv` writes, or None when it fed no calibrated consumer."""
        name = self._names.get(id(conv))
        if name is None or name not in self._feeds:
            return None
        amaxes = [self._amax[c] for c in sorted(self._feeds[name]) if c in self._amax]
        if not amaxes:
            return None
        if len(amaxes) == 1:
            c = next(c for c in sorted(self._feeds[name]) if c in self._amax)
            return self._scale("in", c, amaxes, device)
        return self._scale("shadow", name, amaxes, device)


def fresh_shadow(input):
    """(e4m3 bytes, scale) of `input`'s shadow when its features are those it was written from and
    have not been modified since (their _version has not moved), else None."""
    sh = getattr(input, _SHADOW, None)
    if sh is None:
        return None
    q, scale, feats, version = sh
    if input.F is not feats or feats._version != version:
        return None
    return q, scale


def attach_shadow(out, q, scale):
    setattr(out, _SHADOW, (q, scale, out.F, out.F._version))


def input_operand(calib, conv, input):
    """The e4m3 input of a consumer selected for fp8 inside fp8_inference(calib): (bytes, scale)
    from a fresh shadow or converted at its static scale, or None: uncalibrated, the dynamic path
    (which ignores any shadow)."""
    if calib is None:
        return None
    scale = calib._input_scale(conv, input.F.device)
    if scale is None:
        return None
    sh = fresh_shadow(input)
    if sh is not None:
        return sh
    return _C.quantize_e4m3_static(input.F.contiguous(), scale), scale
