"""Broadcast of per-cloud rows back to the rows of each cloud (reference: MinkowskiBroadcast.py).
Row s of the global tensor belongs to the cloud with the s-th smallest batch index (the origin
map's order)."""
import torch
from torch.autograd import Function
from torch.nn import Module

from . import backend as _C
from .backend import CoordinateMapKey
from .common import MinkowskiModuleBase
from .coordinate_manager import CoordinateManager
from .enums import BroadcastMode
from .sparse_tensor import SparseTensor


class MinkowskiBroadcastFunction(Function):
    @staticmethod
    def forward(ctx, input_features: torch.Tensor, input_features_global: torch.Tensor,
                operation_type: BroadcastMode, in_coords_key: CoordinateMapKey,
                glob_coords_key: CoordinateMapKey, coords_manager: CoordinateManager):
        assert isinstance(operation_type, BroadcastMode)
        input_features = input_features.contiguous()
        input_features_global = input_features_global.contiguous()
        ctx.saved_vars = (input_features, input_features_global, operation_type, in_coords_key,
                          glob_coords_key, coords_manager)
        return _C.BroadcastForwardGPU(input_features, input_features_global, operation_type,
                                      in_coords_key, glob_coords_key, coords_manager._manager)

    @staticmethod
    def backward(ctx, grad_out_feat):
        x, g, op, in_key, glob_key, manager = ctx.saved_vars
        grad_in, grad_glob = _C.BroadcastBackwardGPU(x, g, grad_out_feat.contiguous(), op, in_key,
                                                     glob_key, manager._manager)
        return grad_in, grad_glob, None, None, None, None


class MinkowskiBroadcastBase(MinkowskiModuleBase):
    def __init__(self, operation_type):
        MinkowskiModuleBase.__init__(self)
        assert isinstance(operation_type, BroadcastMode)
        self.operation_type = operation_type
        self.broadcast = MinkowskiBroadcastFunction

    def forward(self, input: SparseTensor, input_glob: SparseTensor):
        assert isinstance(input, SparseTensor)
        output = self.broadcast.apply(input.F, input_glob.F, self.operation_type,
                                      input.coordinate_map_key, input_glob.coordinate_map_key,
                                      input.coordinate_manager)
        return SparseTensor(output, coordinate_map_key=input.coordinate_map_key,
                            coordinate_manager=input.coordinate_manager)

    def __repr__(self):
        return self.__class__.__name__


class MinkowskiBroadcastAddition(MinkowskiBroadcastBase):
    """y_u = x1_u + x2[cloud of u]."""

    def __init__(self):
        MinkowskiBroadcastBase.__init__(self, BroadcastMode.ELEMENTWISE_ADDITON)


class MinkowskiBroadcastMultiplication(MinkowskiBroadcastBase):
    """y_u = x1_u * x2[cloud of u]."""

    def __init__(self):
        MinkowskiBroadcastBase.__init__(self, BroadcastMode.ELEMENTWISE_MULTIPLICATION)


class _BroadcastCopy(Function):
    """y[i] = g[cloud of i]; dg[s] = sum of dy over cloud s (the native broadcast / reduction)."""

    @staticmethod
    def forward(ctx, glob_features, in_key, manager, n):
        grp = manager._origin_grouping(in_key)
        ctx.grp = grp
        ctx.dtype = glob_features.dtype
        return _C._broadcast(None, _C._f32c(glob_features), grp, _C._lib.BCAST_COPY,
                             glob_features.dtype, n=n, C=glob_features.size(1))

    @staticmethod
    def backward(ctx, grad_out):
        g = _C._segment_reduce(grad_out.contiguous(), ctx.grp, _C._lib.SEG_SUM)
        return g.to(ctx.dtype), None, None, None


def _broadcast_copy(input, input_glob):
    mgr = input.coordinate_manager._manager
    _C._check_feats(input.F, mgr, input.coordinate_map_key)
    _C._check_glob(mgr, input.F, input_glob.F, input_glob.coordinate_map_key)
    return _BroadcastCopy.apply(input_glob.F.contiguous(), input.coordinate_map_key, mgr,
                                len(input))


class MinkowskiBroadcast(Module):
    """y_u = x2[cloud of u]; x1 only supplies the output coordinates."""

    def __repr__(self):
        return self.__class__.__name__

    def forward(self, input: SparseTensor, input_glob: SparseTensor):
        assert isinstance(input, SparseTensor)
        assert isinstance(input_glob, SparseTensor)
        return SparseTensor(_broadcast_copy(input, input_glob),
                            coordinate_map_key=input.coordinate_map_key,
                            coordinate_manager=input.coordinate_manager)


class MinkowskiBroadcastConcatenation(MinkowskiBroadcast):
    """y_u = [x1_u, x2[cloud of u]]."""

    def forward(self, input: SparseTensor, input_glob: SparseTensor):
        assert isinstance(input, SparseTensor)
        assert isinstance(input_glob, SparseTensor)
        cat = torch.cat((input.F, _broadcast_copy(input, input_glob)), dim=1)
        return SparseTensor(cat, coordinate_map_key=input.coordinate_map_key,
                            coordinate_manager=input.coordinate_manager)
