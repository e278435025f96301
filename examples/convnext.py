"""A small depthwise-separable (ConvNeXt-style) sparse classifier, written against a *module handle*
as examples/resnet.py is, so the identical definition runs on this package and on the compiled
reference (`oracle/_ref`, CPU):

    import minkowskiengine_b200 as ME
    from examples.convnext import convnext
    net = convnext(ME, in_channels=3, out_channels=10, D=3).cuda()
    logits = net(x).F            # [number of clouds, out_channels], row s = s-th smallest batch index

Stem convolution, then stages of blocks
    channel-wise k = 7 -> BatchNorm -> Linear(C, 4C) -> GELU -> Linear(4C, C) -> + residual
joined by stride-2 convolutions, global average pooling and a linear head.
"""
import torch.nn as nn


def convnext_block(ME, channels, kernel_size=7, D=3):
    """One depthwise-separable block with its residual connection."""

    class Block(nn.Module):
        def __init__(self):
            super().__init__()
            self.dwconv = ME.MinkowskiChannelwiseConvolution(channels, kernel_size=kernel_size,
                                                             dimension=D)
            self.norm = ME.MinkowskiBatchNorm(channels)
            self.pwconv1 = ME.MinkowskiLinear(channels, 4 * channels)
            self.act = ME.MinkowskiGELU()
            self.pwconv2 = ME.MinkowskiLinear(4 * channels, channels)

        def forward(self, x):
            return x + self.pwconv2(self.act(self.pwconv1(self.norm(self.dwconv(x)))))

    return Block()


def convnext(ME, in_channels=3, out_channels=10, D=3, channels=(32, 64), depths=(1, 1),
             kernel_size=7):
    """Instantiate the classifier on module handle `ME`: stage i has `depths[i]` blocks of
    `channels[i]` channels."""

    class ConvNeXt(nn.Module):
        def __init__(self):
            super().__init__()
            self.stem = nn.Sequential(
                ME.MinkowskiConvolution(in_channels, channels[0], kernel_size=3, stride=2,
                                        dimension=D),
                ME.MinkowskiBatchNorm(channels[0]))
            stages = []
            for i, (c, n) in enumerate(zip(channels, depths)):
                mods = []
                if i > 0:
                    mods += [ME.MinkowskiBatchNorm(channels[i - 1]),
                             ME.MinkowskiConvolution(channels[i - 1], c, kernel_size=2, stride=2,
                                                     dimension=D)]
                mods += [convnext_block(ME, c, kernel_size, D) for _ in range(n)]
                stages.append(nn.Sequential(*mods))
            self.stages = nn.Sequential(*stages)
            # the _KERNEL mode writes cloud s to row s on both packages (the reference's default
            # _PYTORCH_INDEX mode is right only for some origin orders)
            self.pool = ME.MinkowskiGlobalPooling(ME.PoolingMode.GLOBAL_AVG_POOLING_KERNEL)
            self.head = ME.MinkowskiLinear(channels[-1], out_channels, bias=True)

        def forward(self, x):
            return self.head(self.pool(self.stages(self.stem(x))))

    return ConvNeXt()
