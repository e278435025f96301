"""Removing rows from a sparse tensor (reference: MinkowskiPruning.py).  The pruned coordinate map
holds the kept rows in ascending input order; forward and backward are one row gather each
(meb200_gather_rows)."""
import torch
from torch.autograd import Function

from . import backend as _C
from .backend import CoordinateMapKey
from .common import MinkowskiModuleBase
from .coordinate_manager import CoordinateManager
from .sparse_tensor import SparseTensor


class MinkowskiPruningFunction(Function):
    @staticmethod
    def forward(ctx, in_feat: torch.Tensor, mask: torch.Tensor, in_coords_key: CoordinateMapKey,
                out_coords_key: CoordinateMapKey = None, coords_manager: CoordinateManager = None):
        ctx.in_coords_key = in_coords_key
        ctx.out_coords_key = out_coords_key
        ctx.coords_manager = coords_manager
        return _C.PruningForwardGPU(in_feat.contiguous(), mask, in_coords_key, out_coords_key,
                                    coords_manager._manager)

    @staticmethod
    def backward(ctx, grad_out_feat: torch.Tensor):
        grad_in_feat = _C.PruningBackwardGPU(grad_out_feat.contiguous(), ctx.in_coords_key,
                                             ctx.out_coords_key, ctx.coords_manager._manager)
        return grad_in_feat, None, None, None, None


class MinkowskiPruning(MinkowskiModuleBase):
    r"""Removes the rows of a :attr:`SparseTensor` where `mask` is False.

    `mask` is a bool or uint8 tensor with one entry per row, on the tensor's device.  The result
    lives on a new coordinate map at the input's tensor stride whose rows are the kept rows in
    input order.
    """

    def __init__(self):
        super().__init__()
        self.pruning = MinkowskiPruningFunction

    def forward(self, input: SparseTensor, mask: torch.Tensor):
        assert isinstance(input, SparseTensor)
        out_coords_key = CoordinateMapKey(input.coordinate_map_key.get_coordinate_size())
        output = self.pruning.apply(input.F, mask, input.coordinate_map_key, out_coords_key,
                                    input._manager)
        return SparseTensor(output, coordinate_map_key=out_coords_key,
                            coordinate_manager=input._manager)

    def __repr__(self):
        return self.__class__.__name__ + "()"
