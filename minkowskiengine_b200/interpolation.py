"""Multilinear interpolation of sparse-tensor features at float points (reference:
MinkowskiInterpolation.py, src/interpolation_cpu.cpp).  The map (corner rows and weights per point)
is built by `meb200_interp_map`; the forward is point-stationary (`meb200_interp_forward`) and the
backward groups the (point, corner) pairs by row and adds them in pair order
(`meb200_group_by_row` + `meb200_field_reduce`), so both are bit-identical run to run."""
import torch
from torch.autograd import Function

from . import _lib
from . import backend as _C
from .backend import CoordinateMapKey
from .common import MinkowskiModuleBase
from .coordinate_manager import CoordinateManager


def _query(tfield, feats):
    assert tfield.dtype in (torch.float32, torch.float64), \
        f"query coordinates must be float32 or float64, got {tfield.dtype}"
    assert tfield.device == feats.device, \
        f"query coordinates device ({tfield.device}) does not match the features ({feats.device})"
    return tfield.float().contiguous()


class MinkowskiInterpolationFunction(Function):
    """(features [n, C], corner rows int32 [n, 2^D], weights fp32 [n, 2^D]) of the points `tfield`
    (float32 or float64 [n, D+1]) in map `in_coordinate_map_key`; a corner absent from the map has
    row -1 and weight 0.  Differentiable in the features."""

    @staticmethod
    def forward(ctx, input_features: torch.Tensor, tfield: torch.Tensor,
                in_coordinate_map_key: CoordinateMapKey, coordinate_manager: CoordinateManager = None):
        feats = input_features.contiguous()
        mgr = coordinate_manager._manager
        _C._check_feats(feats, mgr, in_coordinate_map_key)
        rows, w = mgr._interp_map(in_coordinate_map_key, _query(tfield, feats))
        out = _C.interp_forward(feats, rows, w)
        ctx.mark_non_differentiable(rows, w)
        ctx.save_for_backward(rows, w)
        ctx.M = feats.size(0)
        return out, rows, w

    @staticmethod
    def backward(ctx, grad_out_feat=None, grad_rows=None, grad_weights=None):
        rows, w = ctx.saved_tensors
        K = rows.size(1)
        group = _C.group_by_row(rows.view(-1), ctx.M)
        grad, _ = _C.field_reduce(grad_out_feat.contiguous(), group, ctx.M, _lib.FIELD_SUM,
                                  weight=w.view(-1), src_div=K)
        return grad, None, None, None


def _pairs(rows, w):
    hit = rows >= 0
    return (rows[hit], torch.nonzero(hit)[:, 0].int()), w[hit]


class MinkowskiInterpolation(MinkowskiModuleBase):
    """Samples linearly interpolated features at float points: out = sum over the 2^D corners
    present in the map of prod_j (1 - |x_j - corner_j| / s_j) * F[corner] (not normalised)."""

    def __init__(self, return_kernel_map=False, return_weights=False):
        super().__init__()
        self.return_kernel_map = return_kernel_map
        self.return_weights = return_weights

    def forward(self, input, tfield: torch.Tensor):
        out, rows, w = MinkowskiInterpolationFunction.apply(input.F, tfield, input.coordinate_map_key,
                                                            input.coordinate_manager)
        ret = [out]
        if self.return_kernel_map or self.return_weights:
            kmap, weights = _pairs(rows, w)    # (in rows, out rows) of the present corners
            if self.return_kernel_map:
                ret.append(kmap)
            if self.return_weights:
                ret.append(weights)
        return tuple(ret) if len(ret) > 1 else out

    def __repr__(self):
        return self.__class__.__name__ + "()"
