"""Batch normalisation on the feature matrix of a sparse tensor
(reference: MinkowskiNormalization.py:51-192, which wraps torch.nn.BatchNorm1d / SyncBatchNorm).

The modules keep a torch `BatchNorm1d` / `SyncBatchNorm` as the PARAMETER HOLDER (`bn.weight`,
`bn.bias`, `bn.running_mean`, ... — state_dict compatible with the reference) but, for CUDA
features with C % 8 == 0, run the four passes through libmeb200's streaming kernels
(csrc/batchnorm.cu; SURVEY.md §8(f) row 1).  Semantics are torch's: biased variance for
normalisation, unbiased for the running estimate, momentum update, per-channel affine; the
synchronised variant all-reduces (sum, sum of squares, count) forward and (sum dy, sum dy*xhat)
backward over the process group, exactly the exchange torch.nn.SyncBatchNorm performs.
`MEB200_TORCH_BN=1` routes everything through torch's own kernels (A/B comparisons).
The exchange runs over NVLink peer memory by default (csrc/peer.cuh), inside the LAST CTA of the
reduction kernels themselves (`meb200_bn_forward_train_peer`, `meb200_bn_backward_reduce_peer`):
no NCCL launch, no cross-stream hand-off, no extra kernel — a synchronised pass launches exactly
what a local one does.
`MEB200_SYNCBN_PEER=0` (or symmetric memory being unavailable) selects NCCL all-reduces.
"""
import contextlib
import ctypes
import os

import torch
import torch.nn as nn

from . import _lib
from .backend import fp8_out as _fp8_out
from .sparse_tensor import SparseTensor
from .tensor_field import same_kind as _same_kind

_USE_TORCH = os.environ.get("MEB200_TORCH_BN", "0") not in ("", "0")
_USE_PEER = os.environ.get("MEB200_SYNCBN_PEER", "1") not in ("", "0")


class _PeerExchange:
    """Symmetric-memory buffer of one (process group, device) for the statistics exchange.
    Layout (include/meb200.h, csrc/peer.cuh): 1024 bytes of flags, then SLOTS
    rotating slots of SLOT_DOUBLES fp64 each; `seq` counts the exchanges (identical on all ranks
    because every rank runs the same layers in the same order)."""
    SLOTS = 4
    SLOT_DOUBLES = 2 * 2048 + 8
    _cache = {}

    @classmethod
    def get(cls, group, device):
        """The exchange buffer of (group, device), or None when symmetric memory cannot be set
        up here (every rank then takes the NCCL exchange: the failure is a property of the
        installation, not of the rank)."""
        key = (id(group), device.index)
        if key not in cls._cache:
            try:
                cls._cache[key] = cls(group, device)
            except Exception as exc:                  # noqa: BLE001
                import warnings
                warnings.warn(f"MEB200_SYNCBN_PEER: symmetric memory unavailable ({exc!r}); "
                              "using the NCCL exchange")
                cls._cache[key] = None
        return cls._cache[key]

    def __init__(self, group, device):
        import torch.distributed._symmetric_memory as symm_mem
        self.world = torch.distributed.get_world_size(group)
        self.rank = torch.distributed.get_rank(group)
        nbytes = 1024 + self.SLOTS * self.SLOT_DOUBLES * 8
        self.buf = symm_mem.empty(nbytes, dtype=torch.uint8, device=device)
        self.buf.zero_()
        self.handle = symm_mem.rendezvous(self.buf, group)
        torch.cuda.synchronize(device)
        torch.distributed.barrier(group)        # every rank's flags are zero before the first call
        self.bases_dev = int(self.handle.buffer_ptrs_dev)   # device array of the ranks' bases
        self.seq = 0

    def next_slot_offset(self, n):
        """Byte offset of the slot of the next exchange (advances the sequence number)."""
        assert n <= self.SLOT_DOUBLES
        self.seq = self.seq + 1 if self.seq < 0x7FFFFFFF else 1
        return 1024 + (self.seq % self.SLOTS) * self.SLOT_DOUBLES * 8


_WORKSPACES = {}


def _workspace(dev, stream):
    """The zero-filled reduction workspace of (device, stream) — csrc/batchnorm.cu BnTail: the
    last CTA of every reduction leaves it zero again, so all layers of a stream share one."""
    key = (dev.index, stream)
    ws = _WORKSPACES.get(key)
    if ws is None:
        ws = torch.zeros(int(_lib.load().meb200_bn_workspace_bytes()), dtype=torch.uint8, device=dev)
        _WORKSPACES[key] = ws
    return ws


_NULL_GUARD = contextlib.nullcontext()


def _device_guard(dev):
    """Native launches go to the CURRENT device's stream: make the tensor's device current
    (nothing to do — and nothing spent — when it already is, the usual case)."""
    if dev.type != "cuda" or dev.index == torch.cuda.current_device():
        return _NULL_GUARD
    return torch.cuda.device(dev)


def _f32(t):
    """fp32 contiguous view of a parameter without a copy when it already is one."""
    if t is None:
        return None
    t = t.detach()
    return t if (t.dtype == torch.float32 and t.is_contiguous()) else t.float().contiguous()


class _BatchNormFunction(torch.autograd.Function):
    """y = relu?( bn(x) + residual? ) with batch statistics (training) or the running statistics
    (`use_running`, inference under autograd: frozen-BN fine-tuning, attribution)."""

    @staticmethod
    def forward(ctx, x, weight, bias, running_mean, running_var, momentum, eps, group, relu,
                residual, use_running, num_batches_tracked=None, fp8=None):
        """fp8 (training only): a fp8_delayed._BnStep, whose y_out = (q, scale, slot) the apply
        pass writes the e4m3 copy of y into and whose grad entry the backward writes the e5m2 copy
        of dx for (each may be None)."""
        lib = _lib.load()
        x = x.contiguous()
        n, C = x.shape
        code = _lib.dtype_code(x.dtype)
        dev = x.device
        with _device_guard(dev):
            stream = _lib.current_stream()
            w32, b32 = _f32(weight), _f32(bias)
            d_count = None
            if residual is not None:
                residual = residual.contiguous()
            y = torch.empty_like(x)
            if use_running:
                # a copy: backward reads it, and a training forward in between rewrites the
                # buffer from the kernel, unseen by autograd's version counter
                mean = running_mean.detach().clone()
                invstd = torch.rsqrt(running_var.detach().float() + eps)
            else:
                mean = torch.empty(C, dtype=torch.float32, device=dev)
                invstd = torch.empty(C, dtype=torch.float32, device=dev)
                ws = _workspace(dev, stream)
            peer = None
            if not use_running and group is not None and _USE_PEER:
                peer = _PeerExchange.get(group, dev)
            fq = None if fp8 is None or fp8.y_out is None or n == 0 else _fp8_out(*fp8.y_out)

            def call(name, *args):
                """Entry `name`, or with fq its _q twin (the same arguments, fq before the
                stream)."""
                if fq is None:
                    return getattr(lib, name)(*args)
                return getattr(lib, name + "_q")(*args[:-1], ctypes.byref(fq), args[-1])
            if not use_running and group is None and n > 0:
                # statistics + finalize in one launch, then the apply pass
                _lib.check(call("meb200_bn_forward_train",
                    _lib.ptr(x), code, n, C, _lib.ptr(w32), _lib.ptr(b32), _lib.ptr(residual),
                    1 if relu else 0, float(eps), float(momentum), _lib.ptr(running_mean),
                    _lib.ptr(running_var), _lib.ptr(num_batches_tracked), _lib.ptr(ws),
                    _lib.ptr(mean), _lib.ptr(invstd), _lib.ptr(y), stream))
                num_batches_tracked = None
            elif peer is not None:
                # the same two launches: the last CTA of the reduction exchanges the statistics
                # with the other ranks over NVLink peer memory before it finalizes
                off = peer.next_slot_offset(2 * C + 1)
                d_count = torch.empty(1, dtype=torch.float64, device=dev)
                _lib.check(call("meb200_bn_forward_train_peer",
                    _lib.ptr(x), code, n, C, _lib.ptr(w32), _lib.ptr(b32), _lib.ptr(residual),
                    1 if relu else 0, float(eps), float(momentum), _lib.ptr(running_mean),
                    _lib.ptr(running_var), _lib.ptr(num_batches_tracked), _lib.ptr(ws),
                    peer.bases_dev, off, peer.seq, peer.rank, peer.world, _lib.ptr(mean),
                    _lib.ptr(invstd), _lib.ptr(d_count), _lib.ptr(y), stream))
                num_batches_tracked = None
            else:
                if not use_running:
                    sums = torch.empty(2 * C + 1, dtype=torch.float64, device=dev)
                    _lib.check(lib.meb200_bn_stats_to(_lib.ptr(x), code, n, C, _lib.ptr(ws),
                                                      _lib.ptr(sums), stream))
                    if group is not None:
                        sums[2 * C] = float(n)
                        torch.distributed.all_reduce(sums, group=group)
                        d_count = sums[2 * C:]
                    _lib.check(lib.meb200_bn_finalize(
                        _lib.ptr(sums), float(max(n, 1)), _lib.ptr(d_count), C, float(eps),
                        float(momentum), _lib.ptr(running_mean), _lib.ptr(running_var),
                        _lib.ptr(mean), _lib.ptr(invstd), stream))
                _lib.check(call("meb200_bn_apply_fused",
                    _lib.ptr(x), code, n, C, _lib.ptr(mean), _lib.ptr(invstd), _lib.ptr(w32),
                    _lib.ptr(b32), _lib.ptr(residual), 1 if relu else 0, _lib.ptr(y), stream))
            if fp8 is not None:
                fp8.written = not use_running
        if num_batches_tracked is not None and not use_running:
            num_batches_tracked.add_(1)        # paths whose kernels do not count the batch themselves
        ctx.save_for_backward(x, mean, invstd, w32 if w32 is not None else mean.new_empty(0),
                              d_count if d_count is not None else mean.new_empty(0, dtype=torch.float64),
                              y if relu else x.new_empty(0))
        ctx.group = group
        ctx.has_affine = weight is not None
        ctx.param_dtype = None if weight is None else weight.dtype
        ctx.relu, ctx.has_residual, ctx.use_running = bool(relu), residual is not None, use_running
        ctx.grad_entry = None if fp8 is None or use_running else fp8.grad
        return y

    @staticmethod
    def backward(ctx, dy):
        lib = _lib.load()
        x, mean, invstd, w32, d_count, y = ctx.saved_tensors
        dy = dy.contiguous()
        if dy.dtype != x.dtype:
            dy = dy.to(x.dtype)
        n, C = x.shape
        code = _lib.dtype_code(x.dtype)
        ymask = y if ctx.relu else None
        with _device_guard(x.device):
            stream = _lib.current_stream()
            group = None if ctx.use_running else ctx.group
            peer = _PeerExchange.get(group, x.device) if (group is not None and _USE_PEER) else None
            gs = torch.empty(2 * C, dtype=torch.float64, device=x.device)
            grad_w = grad_b = None
            g32 = None
            if ctx.has_affine:   # local sums; DDP averages parameter gradients across ranks
                g32 = torch.empty(2 * C, dtype=torch.float32, device=x.device)
                grad_b, grad_w = g32[:C], g32[C:]
            ws = _workspace(x.device, stream)
            if peer is not None:
                # one launch: reduction, exchange over peer memory by its last CTA (global totals
                # into `gs`), local totals into the fp32 parameter gradients
                off = peer.next_slot_offset(2 * C)
                _lib.check(lib.meb200_bn_backward_reduce_peer(
                    _lib.ptr(dy), _lib.ptr(x), _lib.ptr(ymask), code, n, C, _lib.ptr(mean),
                    _lib.ptr(invstd), _lib.ptr(ws), peer.bases_dev, off, peer.seq, peer.rank,
                    peer.world, _lib.ptr(gs), _lib.ptr(grad_w), _lib.ptr(grad_b), stream))
            else:
                _lib.check(lib.meb200_bn_backward_reduce_to(
                    _lib.ptr(dy), _lib.ptr(x), _lib.ptr(ymask), code, n, C, _lib.ptr(mean),
                    _lib.ptr(invstd), _lib.ptr(ws), _lib.ptr(gs), _lib.ptr(grad_w),
                    _lib.ptr(grad_b), stream))
            if g32 is not None and ctx.param_dtype != torch.float32:
                g32 = g32.to(ctx.param_dtype)
                grad_b, grad_w = g32[:C], g32[C:]
            if ctx.use_running:
                gs = torch.zeros_like(gs)      # statistics are constants: dx = dy' * invstd * w
            elif peer is None and group is not None:
                torch.distributed.all_reduce(gs, group=group)
            dx = torch.empty_like(x)
            dres = torch.empty_like(x) if ctx.has_residual else None
            args = (_lib.ptr(dy), _lib.ptr(x), _lib.ptr(ymask), code, n, C, _lib.ptr(mean),
                    _lib.ptr(invstd), _lib.ptr(w32) if w32.numel() else None, _lib.ptr(gs),
                    float(max(n, 1)), _lib.ptr(d_count) if d_count.numel() else None, _lib.ptr(dx),
                    _lib.ptr(dres))
            g = ctx.grad_entry
            if g is None or n == 0:
                _lib.check(lib.meb200_bn_backward_apply_fused(*args, stream))
            else:
                # the e5m2 copy of dx for the backward of the convolution that produced x
                q = torch.empty(x.shape, dtype=torch.uint8, device=x.device)
                fq = _fp8_out(q, g.scale, g.slot)
                _lib.check(lib.meb200_bn_backward_apply_fused_q(*args, ctypes.byref(fq), stream))
                g.shadow = (q, dx.data_ptr(), dx.shape, dx._version)
        return dx, grad_w, grad_b, None, None, None, None, None, None, dres, None, None, None


def _native_ok(bn, x):
    """Shape/dtype/configuration only (never the row count or per-rank state): every rank of a
    process group must take the same path, or their collectives would not match."""
    def buf_ok(t):
        return (t is not None and t.dtype == torch.float32 and t.is_contiguous()
                and t.device == x.device)
    return (not _USE_TORCH and x.is_cuda and x.dim() == 2 and x.shape[1] % 8 == 0
            and 8 <= x.shape[1] <= 2048
            and x.dtype in (torch.float32, torch.bfloat16, torch.float16)
            and bn.track_running_stats and bn.momentum is not None
            and buf_ok(bn.running_mean) and buf_ok(bn.running_var))


def _batch_norm(bn, x, group=None, relu=False, residual=None, fp8=None):
    """Functional core shared by the modules and fused_bn_relu.  fp8: the delayed-scaling outputs
    of a training batch norm (_BatchNormFunction), written only by the native training pass."""
    if not _native_ok(bn, x) or (residual is not None and (residual.shape != x.shape
                                                           or residual.dtype != x.dtype)):
        y = bn(x)
        if residual is not None:
            y = y + residual
        return torch.relu(y) if relu else y
    if bn.training:
        if x.shape[0] == 0 and group is None:      # nothing to normalise, statistics untouched
            return x.clone() if residual is None else x + residual
        nbt = bn.num_batches_tracked
        if nbt is not None and not (nbt.dtype == torch.int64 and nbt.device == x.device):
            nbt.add_(1)
            nbt = None
        return _BatchNormFunction.apply(x, bn.weight, bn.bias, bn.running_mean, bn.running_var,
                                        bn.momentum, bn.eps, group, relu, residual, False, nbt,
                                        fp8)
    return _BatchNormFunction.apply(x, bn.weight, bn.bias, bn.running_mean, bn.running_var,
                                    bn.momentum, bn.eps, None, relu, residual, True)


def fused_bn_relu(norm, input, residual=None):
    """relu(norm(input) [+ residual]) in one pass over the features — the tail of a residual
    block (reference: MinkowskiEngine/modules/resnet_block.py:52-68 runs norm, `+=` and ReLU as
    three passes).  `norm` is a MinkowskiBatchNorm / MinkowskiSyncBatchNorm module."""
    return _bn_tail(norm, input, residual, relu=True)


def _bn_tail(norm, input, residual, relu):
    """relu?(norm(input) [+ residual]) in one pass over the features (fused_bn_relu)."""
    bn = norm.bn
    group = norm._group() if isinstance(norm, MinkowskiSyncBatchNorm) else None
    res = None
    if residual is not None:
        assert residual.coordinate_map_key == input.coordinate_map_key, \
            "residual and input must live on the same coordinate map"
        res = residual.F
    fp8 = _fp8_begin(norm, input)
    out = _batch_norm(bn, input.F, group, relu=relu, residual=res, fp8=fp8)
    return _fp8_end(fp8, SparseTensor(out, coordinate_map_key=input.coordinate_map_key,
                                      coordinate_manager=input.coordinate_manager))


def _fp8_begin(norm, input):
    """The delayed-scaling fp8 outputs of a training batch norm on `input` inside
    fp8_training(scaling=...) (fp8_delayed.Fp8DelayedScaling._bn_begin), or None."""
    if not norm.bn.training:
        return None
    from . import backend as _C
    scaling = _C.fp8_training_scaling()
    return None if scaling is None else scaling._bn_begin(norm, input)


def _fp8_end(fp8, out):
    """`out`, with the producer tag and the shadow of the fp8 outputs (if any)."""
    if fp8 is not None:
        fp8.recipe._bn_end(fp8, out)
    return out


def _eval_scale_shift(bn, conv_bias=None):
    """fp32 [C] (scale, shift) of eval-mode batch norm as one affine map, y = x * scale + shift,
    by the formula the eval apply pass uses: invstd = rsqrt(running_var + eps), scale = invstd * w,
    shift = b - running_mean * scale (w = 1, b = 0 without affine parameters).  A bias added
    before the norm (a convolution's, [1, C] or [C]) folds in as shift += conv_bias * scale."""
    invstd = torch.rsqrt(bn.running_var.detach().float() + bn.eps)
    scale = invstd if bn.weight is None else invstd * _f32(bn.weight)
    mean = bn.running_mean.detach().float()
    shift = -(mean * scale) if bn.bias is None else _f32(bn.bias) - mean * scale
    if conv_bias is not None:
        shift = shift + conv_bias.detach().float().reshape(-1) * scale
    return scale.contiguous(), shift.contiguous()


class MinkowskiBatchNorm(nn.Module):
    def __init__(self, num_features, eps=1e-5, momentum=0.1, affine=True,
                 track_running_stats=True):
        super().__init__()
        self.bn = torch.nn.BatchNorm1d(num_features, eps=eps, momentum=momentum, affine=affine,
                                       track_running_stats=track_running_stats)

    def forward(self, input):
        fp8 = _fp8_begin(self, input)
        output = _batch_norm(self.bn, input.F, fp8=fp8)
        return _fp8_end(fp8, _same_kind(input, output))

    def __repr__(self):
        s = "({}, eps={}, momentum={}, affine={}, track_running_stats={})".format(
            self.bn.num_features, self.bn.eps, self.bn.momentum, self.bn.affine,
            self.bn.track_running_stats)
        return self.__class__.__name__ + s


class MinkowskiSyncBatchNorm(MinkowskiBatchNorm):
    def __init__(self, num_features, eps=1e-5, momentum=0.1, affine=True,
                 track_running_stats=True, process_group=None):
        nn.Module.__init__(self)
        self.bn = torch.nn.SyncBatchNorm(num_features, eps=eps, momentum=momentum,
                                         affine=affine,
                                         track_running_stats=track_running_stats,
                                         process_group=process_group)

    def _group(self):
        bn = self.bn
        if bn.training and torch.distributed.is_available() and torch.distributed.is_initialized():
            group = getattr(bn, "process_group", None) or torch.distributed.group.WORLD
            if torch.distributed.get_world_size(group) > 1:
                return group
        return None

    def forward(self, input):
        fp8 = _fp8_begin(self, input)
        output = _batch_norm(self.bn, input.F, self._group(), fp8=fp8)
        return _fp8_end(fp8, _same_kind(input, output))

    @classmethod
    def convert_sync_batchnorm(cls, module, process_group=None):
        """Recursively swaps MinkowskiBatchNorm for MinkowskiSyncBatchNorm
        (reference: MinkowskiNormalization.py:123-192)."""
        module_output = module
        if isinstance(module, MinkowskiBatchNorm) and not isinstance(module, MinkowskiSyncBatchNorm):
            module_output = MinkowskiSyncBatchNorm(
                module.bn.num_features, module.bn.eps, module.bn.momentum, module.bn.affine,
                module.bn.track_running_stats, process_group)
            if module.bn.affine:
                with torch.no_grad():
                    module_output.bn.weight = module.bn.weight
                    module_output.bn.bias = module.bn.bias
            module_output.bn.running_mean = module.bn.running_mean
            module_output.bn.running_var = module.bn.running_var
            module_output.bn.num_batches_tracked = module.bn.num_batches_tracked
            return module_output         # its only child is the parameter holder just rebuilt
        for name, child in module.named_children():
            module_output.add_module(name, cls.convert_sync_batchnorm(child, process_group))
        del module
        return module_output


class MinkowskiInstanceNormFunction(torch.autograd.Function):
    """Per-cloud normalisation (reference: MinkowskiNormalization.py:194-310), composed from the
    native per-cloud reduction and broadcast as the reference composes global average pooling and
    broadcast.  Statistics stay fp32 and the centred features are kept in fp32, so a bf16 / fp16
    output carries one rounding:
        mean = avg(x),  var = avg((x - mean)^2),  inv_std = 1 / sqrt(var + 1e-8),
        y = x * inv_std - mean * inv_std
    backward (reference :254-310):
        dx = (dy - y * avg(dy * y) - avg(dy)) * inv_std"""

    @staticmethod
    def forward(ctx, in_feat, in_coords_key, glob_coords_key=None, coords_manager=None,
                gpooling_mode=None):
        from . import backend as _C
        mgr = coords_manager._manager
        in_feat = in_feat.contiguous()
        _C._check_feats(in_feat, mgr, in_coords_key)
        grp = mgr._origin_grouping(in_coords_key)
        mean = _C._segment_reduce(in_feat, grp, _lib.SEG_AVG)
        centered = _C._broadcast(in_feat, (-mean).contiguous(), grp, _lib.BCAST_ADD, torch.float32)
        var = _C._segment_reduce(centered, grp, _lib.SEG_AVG, b=centered)
        del centered
        inv_std = torch.rsqrt(var + 1e-8)
        norm_feat = _C._broadcast_fma(in_feat, inv_std, grp, k32=(-mean * inv_std).contiguous())
        ctx.grp = grp
        ctx.save_for_backward(inv_std, norm_feat)
        return norm_feat

    @staticmethod
    def backward(ctx, out_grad):
        from . import backend as _C
        inv_std, norm_feat = ctx.saved_tensors
        grp = ctx.grp
        dy = out_grad.contiguous()
        if dy.dtype != norm_feat.dtype:
            dy = dy.to(norm_feat.dtype)
        mean_dout = _C._segment_reduce(dy, grp, _lib.SEG_AVG)
        mean_dout_feat = _C._segment_reduce(dy, grp, _lib.SEG_AVG, b=norm_feat)
        din = _C._broadcast_fma(dy, inv_std, grp, z=norm_feat,
                                h32=(-mean_dout_feat * inv_std).contiguous(),
                                k32=(-mean_dout * inv_std).contiguous())
        return din, None, None, None, None


class MinkowskiInstanceNorm(nn.Module):
    """Instance normalisation of a sparse tensor: every cloud normalised by its own per-channel
    statistics, then `* weight + bias` ([1, C] parameters; reference MinkowskiNormalization.py:
    357-400).  The affine step keeps the feature dtype."""

    def __init__(self, num_features):
        nn.Module.__init__(self)
        self.num_features = num_features
        self.weight = nn.Parameter(torch.ones(1, num_features))
        self.bias = nn.Parameter(torch.zeros(1, num_features))
        self.reset_parameters()
        self.inst_norm = MinkowskiInstanceNormFunction

    def __repr__(self):
        return self.__class__.__name__ + f"(nchannels={self.num_features})"

    def reset_parameters(self):
        self.weight.data.fill_(1)
        self.bias.data.zero_()

    def forward(self, input: SparseTensor):
        assert isinstance(input, SparseTensor)
        output = self.inst_norm.apply(input.F, input.coordinate_map_key, None,
                                      input.coordinate_manager)
        w, b = self.weight, self.bias
        if w.dtype != output.dtype:
            w, b = w.to(output.dtype), b.to(output.dtype)
        output = output * w + b
        return SparseTensor(output, coordinate_map_key=input.coordinate_map_key,
                            coordinate_manager=input.coordinate_manager)
