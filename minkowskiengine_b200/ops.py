"""Feature-level helpers used by the networks on the path: `cat`, `sum` / `mean` / `var`,
`MinkowskiLinear`, `MinkowskiToSparseTensor`, `MinkowskiToFeature` and the stack containers
(reference: MinkowskiOps.py:40-245, :276-352, :460-497).  Plain torch on `.F`."""
import torch
from torch.nn import Module

from .dense import to_sparse, to_sparse_all
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


def _tuple_operator(tensors, operator):
    """`operator` over the features of tensors on one coordinate map (or of TensorFields on one field
    key), as a tensor of their kind (reference: MinkowskiOps.py:70-140).  Accepts the tensors as
    arguments or as one list / tuple."""
    if len(tensors) == 1:
        assert isinstance(tensors[0], (tuple, list))
        tensors = tensors[0]
    assert len(tensors) > 1, \
        "Invalid number of inputs. The input must be at least two len(sparse_tensors) > 1"
    first = tensors[0]
    if not isinstance(first, (SparseTensor, TensorField)):
        raise ValueError("Invalid data type. The input must be either a list of sparse tensors or "
                         "a list of tensor fields.")
    for s in tensors:
        assert isinstance(s, type(first)), "Inputs must be either SparseTensors or TensorFields."
        assert first.device == s.device, f"Device must be the same. {first.device} != {s.device}"
        assert first.coordinate_manager == s.coordinate_manager, COORDINATE_MANAGER_DIFFERENT_ERROR
        assert first.coordinate_map_key == s.coordinate_map_key, \
            COORDINATE_KEY_DIFFERENT_ERROR + str(first.coordinate_map_key) + " != " + \
            str(s.coordinate_map_key)
    return _same_kind(first, operator([s.F for s in tensors]))


def _add_all(xs):
    acc = xs[0] + xs[1]
    for x in xs[2:]:
        acc = acc + x
    return acc


def _var(xs):
    mean = _add_all(xs) / len(xs)
    acc = (xs[0] - mean) ** 2
    for x in xs[1:]:
        acc = acc + (x - mean) ** 2
    return acc / len(xs)


def sum(*sparse_tensors):  # noqa: A001 -- the reference's public name (ME.sum)
    """Element-wise sum of the features of tensors on the same coordinates (MinkowskiOps.py:143)."""
    return _tuple_operator(sparse_tensors, _add_all)


def mean(*sparse_tensors):
    """Element-wise mean of the features of tensors on the same coordinates (MinkowskiOps.py:171)."""
    return _tuple_operator(sparse_tensors, lambda xs: _add_all(xs) / len(xs))


def var(*sparse_tensors):
    """Element-wise (biased) variance of the features of tensors on the same coordinates
    (MinkowskiOps.py:199)."""
    return _tuple_operator(sparse_tensors, _var)


class MinkowskiToFeature(Module):
    """SparseTensor / TensorField -> its feature matrix `.F` (MinkowskiOps.py:460-477)."""

    def forward(self, x):
        assert isinstance(x, (SparseTensor, TensorField)), "Invalid input type for MinkowskiToFeature"
        return x.F

    def __repr__(self):
        return self.__class__.__name__ + "()"


class MinkowskiStackCat(torch.nn.Sequential):
    """Runs every module on the same input and concatenates the outputs' features."""

    def forward(self, x):
        return _tuple_operator([module(x) for module in self], lambda xs: torch.cat(xs, dim=-1))


class MinkowskiStackSum(torch.nn.Sequential):
    def forward(self, x):
        return sum([module(x) for module in self])


class MinkowskiStackMean(torch.nn.Sequential):
    def forward(self, x):
        return mean([module(x) for module in self])


class MinkowskiStackVar(torch.nn.Sequential):
    def forward(self, x):
        return var([module(x) for module in self])


class MinkowskiToSparseTensor(Module):
    """TensorField -> SparseTensor through `TensorField.sparse()` (a SparseTensor passes through);
    a dense [B, C, X1..XD] torch.Tensor -> `to_sparse_all(input, coordinates)` when `coordinates`
    are given (cache them with `dense_coordinates` for a fixed shape), else `to_sparse(input)`
    when `remove_zeros`, else `to_sparse_all(input)` (reference: MinkowskiOps.py:351-411, as its
    docstring has it)."""

    def __init__(self, remove_zeros=True, coordinates=None):
        super().__init__()
        self.remove_zeros = remove_zeros
        self.coordinates = coordinates

    def forward(self, input):
        if isinstance(input, TensorField):
            return input.sparse()
        if isinstance(input, torch.Tensor):
            if self.coordinates is not None:
                return to_sparse_all(input, self.coordinates)
            return to_sparse(input) if self.remove_zeros else to_sparse_all(input)
        assert isinstance(input, SparseTensor), \
            "Input must be a TensorField, a SparseTensor or a torch.Tensor"
        return input

    def __repr__(self):
        return self.__class__.__name__ + "()"
