"""Channel-wise (depthwise) sparse convolution and its autograd function
(reference: MinkowskiChannelwiseConvolution.py:37-212)."""
import math
from typing import Union

import torch
from torch.autograd import Function
from torch.nn import Parameter

from . import backend as _C
from .backend import CoordinateMapKey
from .common import MinkowskiModuleBase
from .coordinate_manager import CoordinateManager
from .enums import RegionType
from .kernel_generator import KernelGenerator
from .sparse_tensor import SparseTensor, _get_coordinate_map_key


class MinkowskiChannelwiseConvolutionFunction(Function):
    """y[o, c] = sum_k kernel[k, c] * x[i_k(o), c] over the convolution's kernel map; forward,
    input gradient and weight gradient each run one native kernel (csrc/chwise.cu)."""

    @staticmethod
    def forward(ctx, input_features: torch.Tensor, kernel_weights: torch.Tensor,
                kernel_generator: KernelGenerator, in_coordinate_map_key: CoordinateMapKey,
                out_coordinate_map_key: CoordinateMapKey = None,
                coordinate_manager: CoordinateManager = None):
        if out_coordinate_map_key is None:
            out_coordinate_map_key = CoordinateMapKey(
                in_coordinate_map_key.get_coordinate_size())
        input_features = input_features.contiguous()
        ctx.input_features = input_features
        ctx.kernel_weights = kernel_weights
        ctx.misc = (kernel_generator, in_coordinate_map_key, out_coordinate_map_key,
                    coordinate_manager)
        return _C.ChannelwiseConvolutionForwardGPU(
            input_features, kernel_weights, kernel_generator.kernel_size,
            kernel_generator.kernel_stride, kernel_generator.kernel_dilation,
            kernel_generator.region_type, kernel_generator.region_offsets, in_coordinate_map_key,
            out_coordinate_map_key, coordinate_manager._manager)

    @staticmethod
    def backward(ctx, grad_out_feat: torch.Tensor):
        kgen, in_key, out_key, manager = ctx.misc
        grad_in_feat, grad_kernel = _C.ChannelwiseConvolutionBackwardGPU(
            ctx.input_features, grad_out_feat, ctx.kernel_weights, kgen.kernel_size,
            kgen.kernel_stride, kgen.kernel_dilation, kgen.region_type, kgen.region_offsets,
            in_key, out_key, manager._manager, need_in=ctx.needs_input_grad[0],
            need_w=ctx.needs_input_grad[1])
        return grad_in_feat, grad_kernel, None, None, None, None


class MinkowskiChannelwiseConvolution(MinkowskiModuleBase):
    """Depthwise sparse convolution: every channel is convolved with its own kernel,
    y[u, c] = sum over offsets i with u + i in the input of W[i, c] * x[u + i, c]
    (reference: MinkowskiChannelwiseConvolution.py:37-212).  `kernel` is fp32 [K, C] and `bias`
    [1, C], as in the reference, so its state_dict loads unchanged.

    Unlike the reference, `coordinates` (a key, a SparseTensor or a coordinate tensor) is honoured:
    the output rows are the given map's, as MinkowskiConvolution does.  Without it the output is
    on the input map strided by `stride`."""

    def __init__(self, in_channels, kernel_size=-1, stride=1, dilation=1, bias=False,
                 kernel_generator=None, dimension=-1):
        super().__init__()
        assert dimension > 0, \
            f"Invalid dimension. Please provide a valid dimension argument. dimension={dimension}"
        if kernel_generator is None:
            kernel_generator = KernelGenerator(kernel_size=kernel_size, stride=stride,
                                               dilation=dilation, dimension=dimension)
        self.kernel_generator = kernel_generator
        self.in_channels = in_channels
        self.dimension = dimension
        self.kernel_shape = (kernel_generator.kernel_volume, self.in_channels)
        self.kernel = Parameter(torch.empty(*self.kernel_shape, dtype=torch.float32))
        self.bias = Parameter(torch.empty(1, in_channels, dtype=torch.float32)) if bias else None
        self.conv = MinkowskiChannelwiseConvolutionFunction
        self.reset_parameters()

    def forward(self, input: SparseTensor,
                coordinates: Union[torch.Tensor, CoordinateMapKey, SparseTensor] = None):
        assert isinstance(input, SparseTensor)
        assert input.D == self.dimension
        assert self.in_channels == input.shape[1], \
            f"Channel size mismatch {self.in_channels} != {input.shape[1]}"
        out_key = _get_coordinate_map_key(input, coordinates)
        outfeat = self.conv.apply(input.F, self.kernel, self.kernel_generator,
                                  input.coordinate_map_key, out_key, input._manager)
        if self.bias is not None:
            outfeat = outfeat + self.bias.to(outfeat.dtype)
        return SparseTensor(outfeat, coordinate_map_key=out_key,
                            coordinate_manager=input._manager)

    def reset_parameters(self, is_transpose=False):
        with torch.no_grad():
            n = self.in_channels * self.kernel_generator.kernel_volume
            stdv = 1.0 / math.sqrt(n)
            self.kernel.data.uniform_(-stdv, stdv)
            if self.bias is not None:
                self.bias.data.uniform_(-stdv, stdv)

    def __repr__(self):
        s = f"(in={self.in_channels}, region_type={self.kernel_generator.region_type}, "
        if self.kernel_generator.region_type in [RegionType.CUSTOM]:
            s += f"kernel_volume={self.kernel_generator.kernel_volume}, "
        else:
            s += f"kernel_size={self.kernel_generator.kernel_size}, "
        s += (f"stride={self.kernel_generator.kernel_stride}, "
              f"dilation={self.kernel_generator.kernel_dilation})")
        return self.__class__.__name__ + s
