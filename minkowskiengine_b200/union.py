"""Union of sparse tensors (reference: MinkowskiUnion.py) and the autograd function behind
arithmetic between sparse tensors on different coordinate maps (MinkowskiTensor.py:522-540).  Both
run the union fold of csrc/union.cu over the manager's cached union map."""
import torch
from torch.autograd import Function
from torch.nn import Module

from . import _lib
from . import backend as _C
from .backend import CoordinateMapKey
from .coordinate_manager import CoordinateManager
from .sparse_tensor import SparseTensor


class MinkowskiUnionFunction(Function):
    @staticmethod
    def forward(ctx, in_coords_keys: list, out_coords_key: CoordinateMapKey,
                coordinate_manager: CoordinateManager, *in_feats):
        assert isinstance(in_feats, (list, tuple)), "Input must be a collection of Tensors"
        assert len(in_feats) > 1, "input must be a set with at least 2 Tensors"
        assert len(in_feats) == len(in_coords_keys), \
            "The input features and keys must have the same length"
        return _union_apply(ctx, in_coords_keys, out_coords_key, coordinate_manager,
                            _lib.UNION_ADD, in_feats)

    @staticmethod
    def backward(ctx, grad_out_feat):
        return (None, None, None, *_union_grads(ctx, grad_out_feat))


class MinkowskiBinaryFunction(Function):
    """op(a, b) between two sparse tensors on different maps: rows only in `a` keep a, rows only in
    `b` give op(0, b), rows in both give op(a, b) (the reference's piecewise semantics)."""

    @staticmethod
    def forward(ctx, op, in_coords_keys, out_coords_key, coordinate_manager, a, b):
        return _union_apply(ctx, in_coords_keys, out_coords_key, coordinate_manager, op, (a, b))

    @staticmethod
    def backward(ctx, grad_out_feat):
        return (None, None, None, None, *_union_grads(ctx, grad_out_feat))


def _union_apply(ctx, in_keys, out_key, manager, op, feats):
    mgr = manager._manager
    um = mgr._union(in_keys)
    out_key.set_key(list(um.key[0]), um.key[1])
    ctx.um, ctx.op = um, op
    ctx.save_for_backward(*feats)
    return _C.union_fold_forward(feats, um, op)


def _union_grads(ctx, grad_out_feat):
    feats = ctx.saved_tensors
    needs = ctx.needs_input_grad[-len(feats):]
    return _C.union_fold_backward(grad_out_feat, feats, ctx.um, ctx.op, needs)


class MinkowskiUnion(Module):
    r"""Union of the coordinates of all input sparse tensors, features of shared coordinates
    added.  Rows of the result: the rows of the first input in order, then the new rows of each
    following input in order.  All inputs must share one coordinate manager and tensor stride."""

    def __init__(self):
        super().__init__()
        self.union = MinkowskiUnionFunction

    def forward(self, *inputs):
        assert isinstance(inputs, (list, tuple)), "The input must be a list or tuple"
        for s in inputs:
            assert isinstance(s, SparseTensor), "Inputs must be sparse tensors."
        assert len(inputs) > 1, "input must be a set with at least 2 SparseTensors"
        ref_coordinate_manager = inputs[0].coordinate_manager
        for s in inputs:
            assert ref_coordinate_manager == s.coordinate_manager, \
                "Invalid coordinate manager. All inputs must have the same coordinate manager."
        coordinate_manager = inputs[0].coordinate_manager
        out_key = CoordinateMapKey(inputs[0].coordinate_map_key.get_coordinate_size())
        # mixed dtypes: summed in their promoted dtype, the result in the first input's dtype (the
        # reference adds into a tensor of that dtype)
        dt = inputs[0].F.dtype
        for s in inputs[1:]:
            dt = torch.promote_types(dt, s.F.dtype)
        output = self.union.apply([s.coordinate_map_key for s in inputs], out_key,
                                  coordinate_manager, *[s.F.to(dt) for s in inputs])
        return SparseTensor(output.to(inputs[0].F.dtype), coordinate_map_key=out_key,
                            coordinate_manager=coordinate_manager)

    def __repr__(self):
        return self.__class__.__name__ + "()"
