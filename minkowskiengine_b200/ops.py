"""Feature-level helpers used by the networks on the path: `cat`, `MinkowskiLinear`,
`MinkowskiToSparseTensor` (reference: MinkowskiOps.py:40-160, :276-352)."""
import torch
from torch.nn import Module

from .sparse_tensor import (COORDINATE_KEY_DIFFERENT_ERROR, COORDINATE_MANAGER_DIFFERENT_ERROR,
                            SparseTensor)
from .tensor_field import TensorField
from .tensor_field import same_kind as _same_kind


class MinkowskiLinear(Module):
    def __init__(self, in_features, out_features, bias=True):
        super().__init__()
        self.linear = torch.nn.Linear(in_features, out_features, bias=bias)

    def forward(self, input):
        output = self.linear(input.F)
        return _same_kind(input, output)

    def __repr__(self):
        return (f"{self.__class__.__name__}(in_features={self.linear.in_features}, "
                f"out_features={self.linear.out_features}, bias={self.linear.bias is not None})")


def cat(*sparse_tensors):
    """Concatenate features of tensors living on the SAME coordinate map, or of TensorFields on the
    same field key (reference: MinkowskiOps.py:70-110)."""
    assert len(sparse_tensors) > 1, f"Invalid number of inputs. The input must be at least two len(sparse_tensors) > 1"
    first = sparse_tensors[0]
    assert isinstance(first, (SparseTensor, TensorField)), \
        "Inputs must be either SparseTensors or TensorFields."
    for s in sparse_tensors:
        assert isinstance(s, type(first)), "Inputs must be either SparseTensors or TensorFields."
        assert first.coordinate_manager == s.coordinate_manager, COORDINATE_MANAGER_DIFFERENT_ERROR
        assert first.coordinate_map_key == s.coordinate_map_key, \
            COORDINATE_KEY_DIFFERENT_ERROR + str(first.coordinate_map_key) + " != " + str(s.coordinate_map_key)
    feats = torch.cat([s.F for s in sparse_tensors], dim=1)
    return _same_kind(first, feats)


class MinkowskiToSparseTensor(Module):
    """TensorField -> SparseTensor through `TensorField.sparse()` (a SparseTensor passes through)
    (reference: MinkowskiOps.py:276-352)."""

    def forward(self, input):
        if isinstance(input, TensorField):
            return input.sparse()
        assert isinstance(input, SparseTensor), "Input must be a TensorField or a SparseTensor"
        return input

    def __repr__(self):
        return self.__class__.__name__ + "()"
