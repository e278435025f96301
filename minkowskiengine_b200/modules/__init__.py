from .resnet_block import BasicBlock, Bottleneck  # noqa: F401
from .senet_block import SEBasicBlock, SELayer  # noqa: F401
