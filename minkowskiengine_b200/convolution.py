"""Sparse (transposed) convolution layers and their autograd functions
(reference: MinkowskiConvolution.py:42-634)."""
import math
from typing import Union

import torch
from torch.autograd import Function
from torch.nn import Parameter

from . import backend as _C
from .backend import CoordinateMapKey
from .common import MinkowskiModuleBase
from .coordinate_manager import CoordinateManager
from .enums import ConvolutionMode, RegionType
from .fp8_calibration import attach_shadow, input_operand
from .kernel_generator import KernelGenerator
from .normalization import MinkowskiBatchNorm, _bn_tail, _eval_scale_shift, _native_ok
from .sparse_tensor import SparseTensor, _get_coordinate_map_key


def _fp8_input(ctx, input_features, fp8_wgrad):
    """Saves what the backward reads of the input: with fp8_wgrad (fp8_training(weight_gradient=
    True)) its e4m3 bytes and scale, which the forward multiplies (returned, for its `act`) and the
    weight gradient reads, in place of the features; else the features (returns None)."""
    if not fp8_wgrad:
        ctx.input_features, ctx.act = input_features, None
        return None
    q, a_scale = _C._quantize_e4m3(input_features)
    ctx.input_features, ctx.act = None, (q, a_scale, input_features.dtype)
    return q, a_scale


class MinkowskiConvolutionFunction(Function):
    @staticmethod
    def forward(ctx, input_features: torch.Tensor, kernel_weights: torch.Tensor,
                kernel_generator: KernelGenerator, convolution_mode: ConvolutionMode,
                in_coordinate_map_key: CoordinateMapKey,
                out_coordinate_map_key: CoordinateMapKey = None,
                coordinate_manager: CoordinateManager = None, fp8: bool = False,
                fp8_wgrad: bool = False):
        if out_coordinate_map_key is None:
            out_coordinate_map_key = CoordinateMapKey(
                in_coordinate_map_key.get_coordinate_size())
        input_features = input_features.contiguous()
        act = _fp8_input(ctx, input_features, fp8_wgrad)
        ctx.kernel_weights = kernel_weights
        ctx.misc = (kernel_generator, convolution_mode, in_coordinate_map_key,
                    out_coordinate_map_key, coordinate_manager)
        ctx.fp8 = fp8
        return _C.ConvolutionForwardGPU(
            input_features, kernel_weights, kernel_generator.kernel_size,
            kernel_generator.kernel_stride, kernel_generator.kernel_dilation,
            kernel_generator.region_type, kernel_generator.region_offsets,
            kernel_generator.expand_coordinates, convolution_mode, in_coordinate_map_key,
            out_coordinate_map_key, coordinate_manager._manager, fp8=fp8, act=act)

    @staticmethod
    def backward(ctx, grad_out_feat: torch.Tensor):
        grad_out_feat = grad_out_feat.contiguous()
        kgen, mode, in_key, out_key, manager = ctx.misc
        grad_in_feat, grad_kernel = _C.ConvolutionBackwardGPU(
            ctx.input_features, grad_out_feat, ctx.kernel_weights, kgen.kernel_size,
            kgen.kernel_stride, kgen.kernel_dilation, kgen.region_type, kgen.region_offsets,
            mode, in_key, out_key, manager._manager,
            need_in=ctx.needs_input_grad[0], need_w=ctx.needs_input_grad[1], fp8=ctx.fp8,
            act=ctx.act)
        return grad_in_feat, grad_kernel, None, None, None, None, None, None, None


class MinkowskiConvolutionTransposeFunction(Function):
    @staticmethod
    def forward(ctx, input_features: torch.Tensor, kernel_weights: torch.Tensor,
                kernel_generator: KernelGenerator, convolution_mode: ConvolutionMode,
                in_coordinate_map_key: CoordinateMapKey,
                out_coordinate_map_key: CoordinateMapKey = None,
                coordinate_manager: CoordinateManager = None, fp8: bool = False,
                fp8_wgrad: bool = False):
        if out_coordinate_map_key is None:
            out_coordinate_map_key = CoordinateMapKey(
                in_coordinate_map_key.get_coordinate_size())
        input_features = input_features.contiguous()
        act = _fp8_input(ctx, input_features, fp8_wgrad)
        ctx.kernel_weights = kernel_weights
        ctx.misc = (kernel_generator, convolution_mode, in_coordinate_map_key,
                    out_coordinate_map_key, coordinate_manager)
        ctx.fp8 = fp8
        return _C.ConvolutionTransposeForwardGPU(
            input_features, kernel_weights, kernel_generator.kernel_size,
            kernel_generator.kernel_stride, kernel_generator.kernel_dilation,
            kernel_generator.region_type, kernel_generator.region_offsets,
            kernel_generator.expand_coordinates, convolution_mode, in_coordinate_map_key,
            out_coordinate_map_key, coordinate_manager._manager, fp8=fp8, act=act)

    @staticmethod
    def backward(ctx, grad_out_feat: torch.Tensor):
        grad_out_feat = grad_out_feat.contiguous()
        kgen, mode, in_key, out_key, manager = ctx.misc
        grad_in_feat, grad_kernel = _C.ConvolutionTransposeBackwardGPU(
            ctx.input_features, grad_out_feat, ctx.kernel_weights, kgen.kernel_size,
            kgen.kernel_stride, kgen.kernel_dilation, kgen.region_type, kgen.region_offsets,
            mode, in_key, out_key, manager._manager,
            need_in=ctx.needs_input_grad[0], need_w=ctx.needs_input_grad[1], fp8=ctx.fp8,
            act=ctx.act)
        return grad_in_feat, grad_kernel, None, None, None, None, None, None, None


class MinkowskiConvolutionBase(MinkowskiModuleBase):
    def __init__(self, in_channels, out_channels, kernel_size=-1, stride=1, dilation=1,
                 bias=False, kernel_generator=None, is_transpose=False,
                 expand_coordinates=False, convolution_mode=ConvolutionMode.DEFAULT,
                 dimension=-1):
        super().__init__()
        assert dimension > 0, \
            f"Invalid dimension. Please provide a valid dimension argument. dimension={dimension}"
        if kernel_generator is None:
            kernel_generator = KernelGenerator(kernel_size=kernel_size, stride=stride,
                                               dilation=dilation,
                                               expand_coordinates=expand_coordinates,
                                               dimension=dimension)
        else:
            kernel_generator.expand_coordinates = expand_coordinates
        self.is_transpose = is_transpose
        self.in_channels = in_channels
        self.out_channels = out_channels
        self.kernel_generator = kernel_generator
        self.dimension = dimension
        # kernel volume 1 and stride 1: plain matrix product (MinkowskiConvolution.py:265-270)
        self.use_mm = (kernel_generator.kernel_volume == 1
                       and kernel_generator.requires_strided_coordinates)
        if self.use_mm:
            kernel_shape = (in_channels, out_channels)
        else:
            kernel_shape = (kernel_generator.kernel_volume, in_channels, out_channels)
        self.kernel = Parameter(torch.empty(*kernel_shape, dtype=torch.float32))
        self.bias = Parameter(torch.empty(1, out_channels, dtype=torch.float32)) if bias else None
        self.convolution_mode = convolution_mode
        self.conv = (MinkowskiConvolutionTransposeFunction if is_transpose
                     else MinkowskiConvolutionFunction)

    def forward(self, input: SparseTensor,
                coordinates: Union[torch.Tensor, CoordinateMapKey, SparseTensor] = None):
        assert isinstance(input, SparseTensor)
        assert input.D == self.dimension
        observer = selected = None
        if self.use_mm:
            out_coordinate_map_key = input.coordinate_map_key
            kernel = self.kernel if self.kernel.dtype == input.F.dtype else self.kernel.to(input.F.dtype)
            outfeat = input.F.mm(kernel)
        else:
            out_coordinate_map_key = _get_coordinate_map_key(
                input, coordinates, expand_coordinates=self.kernel_generator.expand_coordinates)
            if _fp8(self, input.F):
                # the bias is the epilogue's shift: one rounding of the biased output
                shift = None if self.bias is None else self.bias.detach().float().reshape(-1)
                return _run(self, input, out_coordinate_map_key, (None, shift, None, False),
                            fp8=True)
            observer = _C.fp8_observer()
            if observer is not None:
                selected = _fp8_rule(self, input.F)
                observer._observe(self, input, selected)
            fp8 = _fp8_train(self, input.F)
            outfeat = self.conv.apply(input.F, self.kernel, self.kernel_generator,
                                      self.convolution_mode, input.coordinate_map_key,
                                      out_coordinate_map_key, input._manager, fp8,
                                      fp8 and _fp8_train_wgrad(self))
        if self.bias is not None:
            outfeat = outfeat + self.bias.to(outfeat.dtype)
        out = SparseTensor(outfeat, coordinate_map_key=out_coordinate_map_key,
                           coordinate_manager=input._manager)
        if selected:        # in fp8 it runs the e4m3 route, which writes shadows
            observer._tag(self, out)
        return out

    def reset_parameters(self, is_transpose=False):
        with torch.no_grad():
            n = (self.out_channels if is_transpose else self.in_channels) \
                * self.kernel_generator.kernel_volume
            stdv = 1.0 / math.sqrt(n)
            self.kernel.data.uniform_(-stdv, stdv)
            if self.bias is not None:
                self.bias.data.uniform_(-stdv, stdv)

    def __repr__(self):
        s = f"(in={self.in_channels}, out={self.out_channels}, "
        if self.kernel_generator.region_type in [RegionType.CUSTOM]:
            s += (f"region_type={self.kernel_generator.region_type}, "
                  f"kernel_volume={self.kernel_generator.kernel_volume}, ")
        else:
            s += f"kernel_size={self.kernel_generator.kernel_size}, "
        s += (f"stride={self.kernel_generator.kernel_stride}, "
              f"dilation={self.kernel_generator.kernel_dilation})")
        return self.__class__.__name__ + s


class MinkowskiConvolution(MinkowskiConvolutionBase):
    """Sparse convolution layer (reference: MinkowskiConvolution.py:360-451)."""

    def __init__(self, in_channels, out_channels, kernel_size=-1, stride=1, dilation=1,
                 bias=False, kernel_generator=None, expand_coordinates=False,
                 convolution_mode=ConvolutionMode.DEFAULT, dimension=None):
        MinkowskiConvolutionBase.__init__(
            self, in_channels, out_channels, kernel_size, stride, dilation, bias,
            kernel_generator, is_transpose=False, expand_coordinates=expand_coordinates,
            convolution_mode=convolution_mode, dimension=dimension)
        self.reset_parameters()


class MinkowskiConvolutionTranspose(MinkowskiConvolutionBase):
    """Sparse transposed convolution layer (reference: MinkowskiConvolution.py:454-543)."""

    def __init__(self, in_channels, out_channels, kernel_size=-1, stride=1, dilation=1,
                 bias=False, kernel_generator=None, expand_coordinates=False,
                 convolution_mode=ConvolutionMode.DEFAULT, dimension=None):
        if kernel_generator is None:
            kernel_generator = KernelGenerator(kernel_size=kernel_size, stride=stride,
                                               dilation=dilation, dimension=dimension)
        MinkowskiConvolutionBase.__init__(
            self, in_channels, out_channels, kernel_size, stride, dilation, bias,
            kernel_generator, is_transpose=True, expand_coordinates=expand_coordinates,
            convolution_mode=convolution_mode, dimension=dimension)
        self.reset_parameters(True)


class MinkowskiGenerativeConvolutionTranspose(MinkowskiConvolutionBase):
    """Transposed convolution that always generates new output coordinates
    (reference: MinkowskiConvolution.py:546-634)."""

    def __init__(self, in_channels, out_channels, kernel_size=-1, stride=1, dilation=1,
                 bias=False, kernel_generator=None,
                 convolution_mode=ConvolutionMode.DEFAULT, dimension=None):
        if kernel_generator is None:
            kernel_generator = KernelGenerator(kernel_size=kernel_size, stride=stride,
                                               dilation=dilation, expand_coordinates=True,
                                               dimension=dimension)
        else:
            kernel_generator.expand_coordinates = True
        MinkowskiConvolutionBase.__init__(
            self, in_channels, out_channels, kernel_size, stride, dilation, bias,
            kernel_generator, is_transpose=True, expand_coordinates=True,
            convolution_mode=convolution_mode, dimension=dimension)
        self.reset_parameters(True)


_FUSED_CONVS = (MinkowskiConvolution, MinkowskiConvolutionTranspose,
                MinkowskiGenerativeConvolutionTranspose)


def _fuses(conv, norm, feats, res):
    """Whether conv -> norm [+ res] can run as one convolution with an epilogue, from everything
    but the residual's coordinate map: norm in eval mode with running statistics (and a shape and
    dtype the native batch norm takes), no gradient needed, a conv that is not a plain matrix
    product (kernel volume 1, stride 1), a residual in the output dtype."""
    bn = norm.bn
    if bn.training or conv.use_mm:
        return False
    if torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in (
            feats, conv.kernel, conv.bias, bn.weight, bn.bias, res)):
        return False
    if res is not None and res.dtype != feats.dtype:
        return False
    return _native_ok(bn, feats.new_empty((0, conv.out_channels)))


def _fp8(conv, feats):
    """Whether `conv` runs its forward on e4m3 operands (backend.fp8_inference): inside the
    context, when _fp8_rule holds."""
    return _C.fp8_enabled() and _fp8_rule(conv, feats)


def _fp8_rule(conv, feats):
    """The layers fp8 inference selects (and Fp8Calibration observes): one that needs no gradient
    (feats, kernel or bias requiring one with grad mode on; fused_conv_bn_relu checks the norm and
    the residual in _fuses), is not a plain matrix product (kernel volume 1, stride 1), has fp32 /
    bf16 / fp16 features and c_in -> c_out on the e4m3 grid (which leaves out the stem, c_in <= 4)."""
    if conv.use_mm or feats.dtype not in _C._FP8_DTYPES:
        return False
    if torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in (
            feats, conv.kernel, conv.bias)):
        return False
    return _C.fp8_supported(conv.in_channels, conv.out_channels)


def _fp8_train(conv, feats):
    """Whether `conv` runs its forward on e4m3 and its input gradient on e5m2 x e4m3 operands
    (backend.fp8_training): inside the context, when _fp8_train_rule holds."""
    return _C.fp8_training_enabled() and _fp8_train_rule(conv, feats)


def _fp8_train_wgrad(conv):
    """Whether a layer fp8 training selected also runs its weight gradient on fp8: inside
    fp8_training(weight_gradient=True) (the innermost block), when the fp8 wgrad takes its shape
    (K <= 1023: the pair lists' limit; c_in and c_out are on the grid already)."""
    return (_C.fp8_training_weight_gradient() and _C.fp8_wgrad_supported(
        conv.in_channels, conv.out_channels, conv.kernel_generator.kernel_volume))


def _fp8_train_rule(conv, feats):
    """The layers fp8 training selects: one that needs a gradient (grad mode on and feats, kernel
    or bias requiring one: the negation of _fp8_rule's check), is not a plain matrix product (kernel
    volume 1, stride 1), has fp32 / bf16 / fp16 features, and is on the e4m3 grid both ways,
    c_in -> c_out for the forward and c_out -> c_in for the dgrad (whether or not the input needs a
    gradient; this leaves out the stem, c_in <= 4)."""
    if conv.use_mm or feats.dtype not in _C._FP8_DTYPES:
        return False
    if not (torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in (
            feats, conv.kernel, conv.bias))):
        return False
    return (_C.fp8_supported(conv.in_channels, conv.out_channels)
            and _C.fp8_supported(conv.out_channels, conv.in_channels))


def _forward_with(conv, input, out_key, epilogue, fp8=False, act=None, shadow=None):
    """conv's native forward onto `out_key` with `epilogue` (no autograd)."""
    kg = conv.kernel_generator
    forward = _C.ConvolutionTransposeForwardGPU if conv.is_transpose else _C.ConvolutionForwardGPU
    return forward(input.F.contiguous(), conv.kernel, kg.kernel_size, kg.kernel_stride,
                   kg.kernel_dilation, kg.region_type, kg.region_offsets, kg.expand_coordinates,
                   conv.convolution_mode, input.coordinate_map_key, out_key,
                   input._manager._manager, epilogue=epilogue, fp8=fp8, act=act, shadow=shadow)


def _run(conv, input, out_key, epilogue, fp8):
    """conv(input) onto `out_key` with `epilogue`, as a SparseTensor (no autograd).  Inside
    fp8_inference(calibration) a calibrated e4m3 layer takes its static-scale input
    (fp8_calibration.input_operand), and a layer that fed a calibrated one also writes the shadow
    of its output.  While observing, records the input's amax and tags the output."""
    observer = _C.fp8_observer()
    if observer is not None:
        observer._observe(conv, input, _fp8_rule(conv, input.F))
    calib = _C.fp8_calibration() if _C.fp8_enabled() else None
    act = input_operand(calib, conv, input) if fp8 else None
    shadow = calib._shadow_scale(conv, input.F.device) if calib is not None else None
    feats = _forward_with(conv, input, out_key, epilogue, fp8=fp8, act=act, shadow=shadow)
    q = None
    if shadow is not None:
        feats, q = feats
    out = SparseTensor(feats, coordinate_map_key=out_key, coordinate_manager=input._manager)
    if q is not None:
        attach_shadow(out, q, shadow)
    if observer is not None:
        observer._tag(conv, out)
    return out


def _output_key(conv, input):
    """The key of conv(input)'s output map, made as the forward makes it."""
    kg = conv.kernel_generator
    manager = input._manager._manager
    out_key = _get_coordinate_map_key(input, None, expand_coordinates=kg.expand_coordinates)
    region = (kg.region_type, kg.kernel_size, kg.kernel_dilation, kg.region_offsets)
    if conv.is_transpose:
        _C._set_transposed_key(manager, input.coordinate_map_key, out_key, kg.kernel_stride,
                               region, kg.expand_coordinates)
    else:
        _C._set_strided_key(manager, input.coordinate_map_key, out_key, kg.kernel_stride,
                            region if kg.expand_coordinates else None)
    return out_key


def fused_conv_bn_relu(conv, norm, input, residual=None, relu=True):
    """relu?(norm(conv(input)) [+ residual]) on the convolution's output map.

    `conv`: a MinkowskiConvolution, MinkowskiConvolutionTranspose or
    MinkowskiGenerativeConvolutionTranspose; `norm`: a MinkowskiBatchNorm or MinkowskiSyncBatchNorm.
    When `norm` is in eval mode with running statistics and no gradient is needed, eval batch norm
    is one affine map per channel, and the convolution applies it (with its own bias folded in),
    the residual and the ReLU to its fp32 accumulator before its one rounding to the output dtype:
    the normalised tensor is written once instead of written, read back and written again.  In
    every other case (training, a K = 1 stride-1 layer, a shape the native batch norm does not
    take, a residual on another map or in another dtype) this is exactly
    fused_bn_relu(norm, conv(input), residual), or norm(conv(input)) when relu is False and there
    is no residual."""
    if not isinstance(conv, _FUSED_CONVS):
        raise TypeError(f"fused_conv_bn_relu: {type(conv).__name__} is not a MinkowskiConvolution, "
                        "MinkowskiConvolutionTranspose or MinkowskiGenerativeConvolutionTranspose")
    if not isinstance(norm, MinkowskiBatchNorm):
        raise TypeError(f"fused_conv_bn_relu: {type(norm).__name__} is not a MinkowskiBatchNorm "
                        "or MinkowskiSyncBatchNorm")
    assert isinstance(input, SparseTensor)
    res = residual.F if residual is not None else None
    out_key = _output_key(conv, input) if _fuses(conv, norm, input.F, res) else None
    if res is not None and out_key is not None and residual.coordinate_map_key != out_key:
        out_key = None
    if out_key is None:
        out = conv(input)
        if residual is None and not relu:
            return norm(out)
        return _bn_tail(norm, out, residual, relu)
    assert input.D == conv.dimension
    scale, shift = _eval_scale_shift(norm.bn, conv.bias)
    return _run(conv, input, out_key, (scale, shift, None if res is None else res.contiguous(), relu),
                fp8=_fp8(conv, input.F))
