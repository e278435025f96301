"""Pointwise non-linearities: torch modules applied to `.F`
(reference: MinkowskiNonlinearity.py:41-200)."""
import torch

from .common import MinkowskiModuleBase
from .tensor_field import same_kind as _same_kind


class MinkowskiNonlinearityBase(MinkowskiModuleBase):
    MODULE = None

    def __init__(self, *args, **kwargs):
        super().__init__()
        self.module = self.MODULE(*args, **kwargs)

    def forward(self, input):
        output = self.module(input.F)
        return _same_kind(input, output)

    def __repr__(self):
        return self.__class__.__name__ + "()"


def _wrap(name, mod):
    return type(name, (MinkowskiNonlinearityBase,), {"MODULE": mod})


MinkowskiReLU = _wrap("MinkowskiReLU", torch.nn.ReLU)
MinkowskiReLU6 = _wrap("MinkowskiReLU6", torch.nn.ReLU6)
MinkowskiLeakyReLU = _wrap("MinkowskiLeakyReLU", torch.nn.LeakyReLU)
MinkowskiPReLU = _wrap("MinkowskiPReLU", torch.nn.PReLU)
MinkowskiELU = _wrap("MinkowskiELU", torch.nn.ELU)
MinkowskiSELU = _wrap("MinkowskiSELU", torch.nn.SELU)
MinkowskiCELU = _wrap("MinkowskiCELU", torch.nn.CELU)
MinkowskiGELU = _wrap("MinkowskiGELU", torch.nn.GELU)
MinkowskiSiLU = _wrap("MinkowskiSiLU", torch.nn.SiLU)
MinkowskiSigmoid = _wrap("MinkowskiSigmoid", torch.nn.Sigmoid)
MinkowskiTanh = _wrap("MinkowskiTanh", torch.nn.Tanh)
MinkowskiSoftplus = _wrap("MinkowskiSoftplus", torch.nn.Softplus)
MinkowskiSoftmax = _wrap("MinkowskiSoftmax", torch.nn.Softmax)
MinkowskiLogSoftmax = _wrap("MinkowskiLogSoftmax", torch.nn.LogSoftmax)
MinkowskiDropout = _wrap("MinkowskiDropout", torch.nn.Dropout)
MinkowskiHardtanh = _wrap("MinkowskiHardtanh", torch.nn.Hardtanh)
MinkowskiHardswish = _wrap("MinkowskiHardswish", torch.nn.Hardswish)
