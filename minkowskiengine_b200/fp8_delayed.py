"""Delayed scaling for fp8 training (DESIGN.md §3, "delayed scaling").

Fp8DelayedScaling(model) keeps, for every convolution of `model`, two entries: `input` (its e4m3
operand) and `grad_output` (its e5m2 operand).  An entry holds the amax of its last H steps and a
slot the running step records into.  Inside fp8_training(scaling=recipe):
- step t converts at the scale of the history alone, recording the step's amax in the same pass,
  so no conversion waits on an amax pass;
- a training batch norm whose output went straight into exactly one selected convolution in the
  previous step (a link) writes that consumer's e4m3 input in its apply pass (a shadow);
- a training batch norm fed by a selected convolution writes the e5m2 copy of its input gradient
  for that convolution's backward;
- an entry that has never recorded a step takes the dynamic route of fp8_training() for that step,
  so step 0 equals fp8_training() bit for bit.
"""
import torch

from . import _lib
from . import backend as _C
from .fp8_calibration import attach_shadow, fresh_shadow, module_names
from .normalization import _device_guard

_PRODUCER = "_fp8_delayed_producer"   # SparseTensor attribute: (recipe, batch-norm name)
_GRAD = "_fp8_delayed_grad"           # SparseTensor attribute: the _GradEntry of its producer
ROLES = ("input", "grad_output")


class _DeviceState:
    """The entries of one device: hist [2L, H] (newest first), the running step's slots [2L], the
    step's (scale, inv) [2L, 2], and the step each entry first recorded in."""

    def __init__(self, hist, cur, first):
        self.hist, self.cur, self.scales = hist, cur, None
        self.first = first
        self.step = None            # the step whose roll produced cur and scales


class _GradEntry:
    """A selected layer's grad_output entry as its forward saw it: the slot and scale of that step
    (None while the entry has never recorded), and the e5m2 copy a batch norm wrote of the gradient
    (bytes, data_ptr, shape, _version)."""

    def __init__(self, recipe, ds, idx):
        self.recipe, self.ds, self.idx, self.step = recipe, ds, idx, recipe._step
        self.slot = ds.cur[idx:idx + 1]
        self.scale = ds.scales[idx] if recipe._ready(ds, idx) else None
        self.shadow = None

    def operand(self, grad):
        """(e5m2 bytes, scale) of the contiguous output gradient: the batch norm's copy when `grad`
        is the tensor it was written from, unmodified; else converted at the entry's scale in one
        launch; else (first step) at its own amax, recording the amax."""
        if self.scale is None:
            self.ds.first.setdefault(self.idx, self.step)
            q, s = _C._quantize_dynamic(grad, "meb200_quantize_e5m2")
            _C.amax_accumulate(grad, self.slot)
            return q, s
        sh = self.shadow
        if sh is not None and sh[1:] == (grad.data_ptr(), grad.shape, grad._version):
            return sh[0], self.scale
        return _C.quantize_fp8_record(grad, _lib.FP8_E5M2, self.scale, self.slot), self.scale


class _LayerStep:
    """What a selected layer's forward hands its autograd Function: its e4m3 input (bytes, scale)
    and its grad_output entry."""
    __slots__ = ("act", "grad")

    def __init__(self, act, grad):
        self.act, self.grad = act, grad


class _BnStep:
    """The fp8 outputs of one training batch norm: y_out = (q, scale, slot) of its consumer's input
    (or None), grad = the _GradEntry of the layer that fed it (or None).  `written`: set by the
    native pass that wrote them."""

    def __init__(self, recipe, name, y_out, grad):
        self.recipe, self.name, self.y_out, self.grad = recipe, name, y_out, grad
        self.written = False


class Fp8DelayedScaling:
    """Delayed fp8 scales for the convolutions of `model`, keyed by their qualified module names.

        scaling = ME.Fp8DelayedScaling(model, history=16, margin=0)
        for x, y in loader:
            with ME.fp8_training(scaling=scaling, weight_gradient=True):
                loss = criterion(model(x).F, y)
            loss.backward()
            opt.step()

    history: H >= 1 (at most _lib.FP8_MAX_HISTORY) past steps whose amax max sets a step's scale.
    margin: an integer >= 0; the scale is that of amax * 2^margin.  The layers it scales are those
    fp8_training() selects; selected layers that are not modules of `model` keep dynamic scales."""

    def __init__(self, model, history=16, margin=0):
        from .convolution import MinkowskiConvolutionBase
        if isinstance(history, bool) or not isinstance(history, int) \
                or not 1 <= history <= _lib.FP8_MAX_HISTORY:
            raise ValueError(f"Fp8DelayedScaling: history must be an integer in [1, "
                             f"{_lib.FP8_MAX_HISTORY}] (got {history!r})")
        if isinstance(margin, bool) or not isinstance(margin, int) or not 0 <= margin <= 127:
            raise ValueError(f"Fp8DelayedScaling: margin must be an integer in [0, 127] "
                             f"(got {margin!r})")
        self.history, self.margin = history, margin
        self._names = module_names(model)
        convs = []
        for m in model.modules():
            if isinstance(m, MinkowskiConvolutionBase) and self._names[id(m)] not in convs:
                convs.append(self._names[id(m)])
        self._index = {name: j for j, name in enumerate(convs)}
        self._step = -1                 # the running step (-1: none yet)
        self._dev = {}                  # device -> _DeviceState
        self._loaded = None             # (hist, cur, first) from load_state_dict, until used
        self._observed = {}             # batch-norm name -> consumer names seen this step
        self._links = {}                # batch-norm name -> consumer name, from the last step

    # ---- steps ---------------------------------------------------------------------------------
    def _begin_step(self):
        self._step += 1
        self._links = {bn: next(iter(cs)) for bn, cs in self._observed.items() if len(cs) == 1}
        self._observed = {}

    def _state(self, device):
        """The entries on `device`, rolled into the running step (one launch per step and
        device)."""
        ds = self._dev.get(device)
        if ds is None:
            L = 2 * len(self._index)
            if self._loaded is not None:
                hist, cur, first = self._loaded
                ds = _DeviceState(hist.to(device, copy=True), cur.to(device, copy=True),
                                  dict(first))
                ds.step = self._loaded_step
            else:
                f32 = {"dtype": torch.float32, "device": device}
                ds = _DeviceState(torch.zeros((L, self.history), **f32), torch.zeros(L, **f32), {})
            self._dev[device] = ds
        if ds.step != self._step:
            n = len(self._index)
            with _device_guard(device):
                ds.cur, ds.scales = _C.fp8_roll(ds.cur, ds.hist, n, n, self.margin)
            ds.step = self._step
        return ds

    def _ready(self, ds, idx):
        """Whether the entry has recorded a step before the running one (it has a delayed scale)."""
        first = ds.first.get(idx)
        return first is not None and first < self._step

    # ---- hooks of the layers ---------------------------------------------------------------------
    def _conv_begin(self, conv, input):
        """Before a selected convolution runs on `input`: its operands, or None when it is not a
        module of the bound model (the dynamic path)."""
        name = self._names.get(id(conv))
        j = self._index.get(name)
        if j is None:
            return None
        tag = getattr(input, _PRODUCER, None)
        if tag is not None and tag[0] is self:
            self._observed.setdefault(tag[1], set()).add(name)
        feats = input.F.contiguous()
        ds = self._state(feats.device)
        if not self._ready(ds, j):
            ds.first.setdefault(j, self._step)
            act = _C._quantize_e4m3(feats)
            _C.amax_accumulate(feats, ds.cur[j:j + 1])
        else:
            scale = ds.scales[j]
            act = fresh_shadow(input)
            if act is None or act[1].data_ptr() != scale.data_ptr():
                act = _C.quantize_fp8_record(feats, _lib.FP8_E4M3, scale, ds.cur[j:j + 1]), scale
        return _LayerStep(act, _GradEntry(self, ds, len(self._index) + j))

    def _bn_begin(self, norm, input):
        """Before a training batch norm runs on `input`: its fp8 outputs, or None."""
        name = self._names.get(id(norm))
        grad = getattr(input, _GRAD, None)
        if grad is not None and (grad.recipe is not self or grad.scale is None
                                 or grad.step != self._step):
            grad = None
        y_out = None
        consumer = self._links.get(name) if name is not None else None
        if consumer is not None and input.F.shape[0] > 0:
            j = self._index[consumer]
            ds = self._state(input.F.device)
            if self._ready(ds, j):
                q = torch.empty(input.F.shape, dtype=torch.uint8, device=input.F.device)
                y_out = (q, ds.scales[j], ds.cur[j:j + 1])
        if name is None and grad is None:
            return None
        return _BnStep(self, name, y_out, grad)

    @staticmethod
    def _bn_end(step, out):
        """After the batch norm of `step` returned `out`: its producer tag and shadow."""
        if step.name is not None:
            setattr(out, _PRODUCER, (step.recipe, step.name))
        if step.written and step.y_out is not None:
            attach_shadow(out, step.y_out[0], step.y_out[1])

    @staticmethod
    def _tag(out, layer):
        setattr(out, _GRAD, layer.grad)

    # ---- checkpoints -----------------------------------------------------------------------------
    def state_dict(self):
        """{"history": H, "margin": margin, "step": the running step, "entries": {layer name:
        {role: {"amax": fp32 [H + 1] CPU tensor (the running step's slot, then the H past steps,
        newest first), "first_step": the step it first recorded in, or None}}}, "links":
        {batch-norm name: [consumer names seen in the running step]}}.  Entries held on several
        devices are combined by max."""
        L = 2 * len(self._index)
        amax = torch.zeros((L, self.history + 1), dtype=torch.float32)
        first = {}
        sources = [(ds.cur, ds.hist, ds.first) for ds in self._dev.values()]
        if not sources and self._loaded is not None:
            sources = [(self._loaded[1], self._loaded[0], self._loaded[2])]
        for cur, hist, fs in sources:
            both = torch.cat([cur.reshape(L, 1), hist], 1).cpu()
            amax = torch.maximum(amax, both)
            for i, s in fs.items():
                first[i] = min(s, first.get(i, s))
        n = len(self._index)
        entries = {name: {role: {"amax": amax[j + r * n].clone(),
                                 "first_step": first.get(j + r * n)}
                          for r, role in enumerate(ROLES)}
                   for name, j in self._index.items()}
        return {"history": self.history, "margin": self.margin, "step": self._step,
                "entries": entries, "links": {bn: sorted(cs) for bn, cs in self._observed.items()}}

    def load_state_dict(self, state):
        """Replaces the recipe's state by `state` (from state_dict()); every name must be a module
        of the bound model.  The next step continues from the saved one."""
        known = set(self._names.values())
        names = list(state["entries"]) + list(state["links"]) + [
            c for cs in state["links"].values() for c in cs]
        missing = [n for n in names if n not in known]
        if missing:
            raise KeyError(f"Fp8DelayedScaling.load_state_dict: no module named {missing[0]!r}")
        unbound = [n for n in state["entries"] if n not in self._index]
        if unbound:
            raise KeyError(f"Fp8DelayedScaling.load_state_dict: {unbound[0]!r} is not a "
                           "convolution")
        H = int(state["history"])
        if not 1 <= H <= _lib.FP8_MAX_HISTORY:
            raise ValueError(f"Fp8DelayedScaling.load_state_dict: history {H}")
        margin = int(state["margin"])
        if not 0 <= margin <= 127:
            raise ValueError(f"Fp8DelayedScaling.load_state_dict: margin {margin}")
        self.history, self.margin, self._step = H, margin, int(state["step"])
        n = len(self._index)
        hist = torch.zeros((2 * n, H), dtype=torch.float32)
        cur = torch.zeros(2 * n, dtype=torch.float32)
        first = {}
        for name, ent in state["entries"].items():
            for r, role in enumerate(ROLES):
                i = self._index[name] + r * n
                a = torch.as_tensor(ent[role]["amax"], dtype=torch.float32).reshape(H + 1)
                cur[i], hist[i] = a[0], a[1:]
                if ent[role]["first_step"] is not None:
                    first[i] = int(ent[role]["first_step"])
        self._loaded, self._loaded_step = (hist, cur, first), self._step
        self._dev = {}
        self._observed = {bn: set(cs) for bn, cs in state["links"].items()}
        self._links = {}
