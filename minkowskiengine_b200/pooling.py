"""Local pooling layers (reference: MinkowskiPooling.py:42-440)."""
import torch
from torch.autograd import Function

from . import backend as _C
from .backend import CoordinateMapKey
from .common import MinkowskiModuleBase
from .coordinate_manager import CoordinateManager
from .enums import PoolingMode
from .kernel_generator import KernelGenerator
from .sparse_tensor import SparseTensor, _get_coordinate_map_key


class MinkowskiLocalPoolingFunction(Function):
    @staticmethod
    def forward(ctx, input_features: torch.Tensor, pooling_mode: PoolingMode,
                kernel_generator: KernelGenerator, in_coordinate_map_key: CoordinateMapKey,
                out_coordinate_map_key: CoordinateMapKey = None,
                coordinate_manager: CoordinateManager = None):
        if out_coordinate_map_key is None:
            out_coordinate_map_key = CoordinateMapKey(
                in_coordinate_map_key.get_coordinate_size())
        input_features = input_features.contiguous()
        ctx.input_features = input_features
        ctx.pooling_mode = pooling_mode
        ctx.kernel_generator = kernel_generator
        ctx.in_coordinate_map_key = in_coordinate_map_key
        ctx.out_coordinate_map_key = out_coordinate_map_key
        ctx.coordinate_manager = coordinate_manager
        out_feat, num_nonzero = _C.LocalPoolingForwardGPU(
            input_features, kernel_generator.kernel_size, kernel_generator.kernel_stride,
            kernel_generator.kernel_dilation, kernel_generator.region_type,
            kernel_generator.region_offsets, pooling_mode, in_coordinate_map_key,
            out_coordinate_map_key, coordinate_manager._manager)
        ctx.num_nonzero = num_nonzero
        return out_feat

    @staticmethod
    def backward(ctx, grad_out_feat):
        grad_out_feat = grad_out_feat.contiguous()
        kgen = ctx.kernel_generator
        grad_in_feat = _C.LocalPoolingBackwardGPU(
            ctx.input_features, grad_out_feat, ctx.num_nonzero, kgen.kernel_size,
            kgen.kernel_stride, kgen.kernel_dilation, kgen.region_type, kgen.region_offsets,
            ctx.pooling_mode, ctx.in_coordinate_map_key, ctx.out_coordinate_map_key,
            ctx.coordinate_manager._manager)
        return grad_in_feat, None, None, None, None, None


class MinkowskiPoolingBase(MinkowskiModuleBase):
    def __init__(self, kernel_size, stride=1, dilation=1, kernel_generator=None,
                 is_transpose=False, pooling_mode=PoolingMode.LOCAL_AVG_POOLING, dimension=-1):
        super().__init__()
        assert dimension > 0, \
            f"Invalid dimension. Please provide a valid dimension argument. dimension={dimension}"
        if stride == 1 and not is_transpose:
            pass  # the reference warns that stride 1 pooling keeps the coordinates
        if kernel_generator is None:
            kernel_generator = KernelGenerator(kernel_size=kernel_size, stride=stride,
                                               dilation=dilation, dimension=dimension)
        self.is_transpose = is_transpose
        self.kernel_generator = kernel_generator
        self.pooling_mode = pooling_mode
        self.dimension = dimension
        self.pooling = MinkowskiLocalPoolingFunction

    def forward(self, input: SparseTensor, coordinates=None):
        assert isinstance(input, SparseTensor)
        assert input.D == self.dimension
        out_key = _get_coordinate_map_key(input, coordinates)
        outfeat = self.pooling.apply(input.F, self.pooling_mode, self.kernel_generator,
                                     input.coordinate_map_key, out_key, input._manager)
        return SparseTensor(outfeat, coordinate_map_key=out_key,
                            coordinate_manager=input.coordinate_manager)

    def __repr__(self):
        return (f"{self.__class__.__name__}(kernel_size={self.kernel_generator.kernel_size}, "
                f"stride={self.kernel_generator.kernel_stride}, "
                f"dilation={self.kernel_generator.kernel_dilation})")


class MinkowskiAvgPooling(MinkowskiPoolingBase):
    """Average over the NON-ZERO members of each window (MinkowskiPooling.py:187-260)."""

    def __init__(self, kernel_size=-1, stride=1, dilation=1, kernel_generator=None,
                 dimension=None):
        MinkowskiPoolingBase.__init__(self, kernel_size, stride, dilation, kernel_generator,
                                      is_transpose=False,
                                      pooling_mode=PoolingMode.LOCAL_AVG_POOLING,
                                      dimension=dimension)


class MinkowskiSumPooling(MinkowskiPoolingBase):
    def __init__(self, kernel_size, stride=1, dilation=1, kernel_generator=None,
                 dimension=None):
        MinkowskiPoolingBase.__init__(self, kernel_size, stride, dilation, kernel_generator,
                                      is_transpose=False,
                                      pooling_mode=PoolingMode.LOCAL_SUM_POOLING,
                                      dimension=dimension)


class MinkowskiMaxPooling(MinkowskiPoolingBase):
    def __init__(self, kernel_size, stride=1, dilation=1, kernel_generator=None,
                 dimension=None):
        MinkowskiPoolingBase.__init__(self, kernel_size, stride, dilation, kernel_generator,
                                      is_transpose=False,
                                      pooling_mode=PoolingMode.LOCAL_MAX_POOLING,
                                      dimension=dimension)


class MinkowskiLocalPoolingTransposeFunction(Function):
    """Unpooling (reference: MinkowskiPooling.py:441-510): the sum over the transposed pooling map,
    whatever `pooling_mode` says, as both reference backends compute it."""

    @staticmethod
    def forward(ctx, input_features: torch.Tensor, pooling_mode: PoolingMode,
                kernel_generator: KernelGenerator, in_coordinate_map_key: CoordinateMapKey,
                out_coordinate_map_key: CoordinateMapKey = None,
                coordinate_manager: CoordinateManager = None):
        if out_coordinate_map_key is None:
            out_coordinate_map_key = CoordinateMapKey(
                in_coordinate_map_key.get_coordinate_size())
        input_features = input_features.contiguous()
        ctx.input_features = input_features
        ctx.pooling_mode = pooling_mode
        ctx.kernel_generator = kernel_generator
        ctx.in_coordinate_map_key = in_coordinate_map_key
        ctx.out_coordinate_map_key = out_coordinate_map_key
        ctx.coordinate_manager = coordinate_manager
        kgen = kernel_generator
        out_feat, num_nonzero = _C.LocalPoolingTransposeForwardGPU(
            input_features, kgen.kernel_size, kgen.kernel_stride, kgen.kernel_dilation,
            kgen.region_type, kgen.region_offsets, kgen.expand_coordinates, pooling_mode,
            in_coordinate_map_key, out_coordinate_map_key, coordinate_manager._manager)
        ctx.num_nonzero = num_nonzero
        return out_feat

    @staticmethod
    def backward(ctx, grad_out_feat):
        grad_out_feat = grad_out_feat.contiguous()
        kgen = ctx.kernel_generator
        grad_in_feat = _C.LocalPoolingTransposeBackwardGPU(
            ctx.input_features, grad_out_feat, ctx.num_nonzero, kgen.kernel_size,
            kgen.kernel_stride, kgen.kernel_dilation, kgen.region_type, kgen.region_offsets,
            ctx.pooling_mode, ctx.in_coordinate_map_key, ctx.out_coordinate_map_key,
            ctx.coordinate_manager._manager)
        return grad_in_feat, None, None, None, None, None


class MinkowskiPoolingTranspose(MinkowskiPoolingBase):
    """Unpooling to the finer tensor stride `tensor_stride / stride` (reference:
    MinkowskiPooling.py:513-580): out[o] = the SUM of the input rows that reach o through the
    transposed pooling map.  (The reference's docstring says the sum is divided by the number of
    contributors; its code does not divide, and neither does this.)  The finer map is reused when
    it exists; `expand_coordinates=True` generates new coordinates around every input row."""

    def __init__(self, kernel_size, stride, dilation=1, kernel_generator=None,
                 expand_coordinates=False, dimension=None):
        if kernel_generator is None:
            kernel_generator = KernelGenerator(kernel_size=kernel_size, stride=stride,
                                               dilation=dilation,
                                               expand_coordinates=expand_coordinates,
                                               dimension=dimension)
        MinkowskiPoolingBase.__init__(self, kernel_size, stride, dilation, kernel_generator,
                                      is_transpose=True, dimension=dimension)
        self.pooling = MinkowskiLocalPoolingTransposeFunction


class MinkowskiGlobalPoolingFunction(Function):
    """Per-cloud reduction to the origin map (reference: MinkowskiPooling.py:583-630)."""

    @staticmethod
    def forward(ctx, input_features: torch.Tensor, pooling_mode: PoolingMode,
                in_coordinate_map_key: CoordinateMapKey,
                out_coordinate_map_key: CoordinateMapKey = None,
                coordinate_manager: CoordinateManager = None):
        if out_coordinate_map_key is None:
            out_coordinate_map_key = CoordinateMapKey(
                in_coordinate_map_key.get_coordinate_size())
        input_features = input_features.contiguous()
        ctx.input_features = input_features
        ctx.in_coords_key = in_coordinate_map_key
        ctx.out_coords_key = out_coordinate_map_key
        ctx.coordinate_manager = coordinate_manager
        ctx.pooling_mode = pooling_mode
        out_feat, num_nonzero = _C.GlobalPoolingForwardGPU(
            input_features, pooling_mode, in_coordinate_map_key, out_coordinate_map_key,
            coordinate_manager._manager)
        ctx.num_nonzero = num_nonzero
        return out_feat

    @staticmethod
    def backward(ctx, grad_out_feat):
        grad_out_feat = grad_out_feat.contiguous()
        grad_in_feat = _C.GlobalPoolingBackwardGPU(
            ctx.input_features, grad_out_feat, ctx.num_nonzero, ctx.pooling_mode,
            ctx.in_coords_key, ctx.out_coords_key, ctx.coordinate_manager._manager)
        return grad_in_feat, None, None, None, None, None


class MinkowskiGlobalPooling(MinkowskiModuleBase):
    """Reduces every cloud to one row at its origin (b, 0, ..., 0); output row s is the cloud
    with the s-th smallest batch index (reference: MinkowskiPooling.py:633-677)."""

    def __init__(self, mode: PoolingMode = PoolingMode.GLOBAL_AVG_POOLING_PYTORCH_INDEX):
        super().__init__()
        assert isinstance(mode, PoolingMode), f"Mode must be an instance of PoolingMode. mode={mode}"
        self.pooling_mode = mode
        self.pooling = MinkowskiGlobalPoolingFunction

    def forward(self, input: SparseTensor, coordinates=None):
        out_key = _get_coordinate_map_key(input, coordinates)
        output = self.pooling.apply(input.F, self.pooling_mode, input.coordinate_map_key, out_key,
                                    input._manager)
        return SparseTensor(output, coordinate_map_key=out_key,
                            coordinate_manager=input.coordinate_manager)

    def __repr__(self):
        return self.__class__.__name__ + f"(mode={str(self.pooling_mode)})"


class MinkowskiGlobalSumPooling(MinkowskiGlobalPooling):
    def __init__(self, mode=PoolingMode.GLOBAL_SUM_POOLING_PYTORCH_INDEX):
        MinkowskiGlobalPooling.__init__(self, mode=mode)


class MinkowskiGlobalAvgPooling(MinkowskiGlobalPooling):
    def __init__(self, mode=PoolingMode.GLOBAL_AVG_POOLING_PYTORCH_INDEX):
        MinkowskiGlobalPooling.__init__(self, mode=mode)


class MinkowskiGlobalMaxPooling(MinkowskiGlobalPooling):
    """Per-cloud, per-channel maximum; the gradient goes to the lowest row holding it."""

    def __init__(self, mode=PoolingMode.GLOBAL_MAX_POOLING_PYTORCH_INDEX):
        MinkowskiGlobalPooling.__init__(self, mode=mode)


class MinkowskiDirectMaxPoolingFunction(Function):
    """Max pooling over an explicit pair list (reference: MinkowskiPooling.py:752-780):
    out[o, c] = the maximum of in_feat[i, c] over the pairs (in_map[p], out_map[p]) = (i, o).
    The first pair in list order wins a tie; an output row without pairs is 0 and sends no
    gradient; a repeated pair counts once.  The backward walks the winning pairs rather than the
    reference's flat mask, which the forward does not build.  Maps may be int32, int64 or float;
    out-of-range maps raise RuntimeError (one host synchronisation); `is_sorted` is ignored."""

    @staticmethod
    def forward(ctx, in_map: torch.Tensor, out_map: torch.Tensor, in_feat: torch.Tensor,
                out_nrows: int, is_sorted: bool = False):
        out_feat, _, winner, out_rows, in_rows = _C._direct_max_pool(in_map, out_map, in_feat,
                                                                     out_nrows, False)
        ctx.in_nrows = in_feat.size(0)
        ctx.save_for_backward(winner, out_rows, in_rows)
        return out_feat

    @staticmethod
    def backward(ctx, grad_out_feat):
        winner, out_rows, in_rows = ctx.saved_tensors
        grad = _C.direct_max_pool_pairs_bw(grad_out_feat, winner, out_rows, in_rows, ctx.in_nrows)
        return None, None, grad, None, None
