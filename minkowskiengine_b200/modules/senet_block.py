"""Squeeze-excitation blocks (reference: MinkowskiEngine/modules/senet_block.py): a per-cloud
average, two linear layers and a sigmoid give one gate per cloud and channel, multiplied back into
every row of the cloud (global pooling + broadcast multiplication)."""
import torch.nn as nn

from ..broadcast import MinkowskiBroadcastMultiplication
from ..nonlinearity import MinkowskiReLU, MinkowskiSigmoid
from ..ops import MinkowskiLinear
from ..pooling import MinkowskiGlobalPooling
from .resnet_block import BasicBlock


class SELayer(nn.Module):
    def __init__(self, channel, reduction=16, D=-1):
        super().__init__()
        self.fc = nn.Sequential(
            MinkowskiLinear(channel, channel // reduction),
            MinkowskiReLU(inplace=True),
            MinkowskiLinear(channel // reduction, channel),
            MinkowskiSigmoid())
        self.pooling = MinkowskiGlobalPooling()
        self.broadcast_mul = MinkowskiBroadcastMultiplication()

    def forward(self, x):
        return self.broadcast_mul(x, self.fc(self.pooling(x)))


class SEBasicBlock(BasicBlock):
    def __init__(self, inplanes, planes, stride=1, dilation=1, downsample=None, reduction=16,
                 D=-1, dimension=None):
        super().__init__(inplanes, planes, stride=stride, dilation=dilation,
                         downsample=downsample, dimension=dimension if dimension else D)
        self.se = SELayer(planes, reduction=reduction, D=D)

    def forward(self, x):
        residual = x
        out = self.relu(self.norm1(self.conv1(x)))
        out = self.se(self.norm2(self.conv2(out)))
        if self.downsample is not None:
            residual = self.downsample(x)
        out += residual
        return self.relu(out)
