"""ResNet classifiers (reference: examples/resnet.py:53-156) and the squeeze-excitation block
(reference: MinkowskiEngine/modules/senet_block.py), written against a *module handle* as
examples/minkunet.py is, so the identical definition runs on this package and on the compiled
reference (`oracle/_ref`, CPU):

    import minkowskiengine_b200 as ME
    from examples.resnet import resnet
    net = resnet("ResNet14", ME, in_channels=3, out_channels=40, D=3).cuda()
    logits = net(x).F            # [number of clouds, out_channels], row s = s-th smallest batch index
"""
import torch.nn as nn

from examples.minkunet import _basic_block, _bn_relu

_LAYERS = {"ResNet14": (1, 1, 1, 1), "ResNet18": (2, 2, 2, 2), "ResNet34": (3, 4, 6, 3)}


def se_layer(ME, channel, reduction=16):
    """Squeeze-excitation: per-cloud average -> two linear layers -> sigmoid gate, multiplied back
    into every row of the cloud (reference senet_block.py SELayer)."""

    class SELayer(nn.Module):
        def __init__(self):
            super().__init__()
            self.fc = nn.Sequential(
                ME.MinkowskiLinear(channel, channel // reduction),
                ME.MinkowskiReLU(inplace=True),
                ME.MinkowskiLinear(channel // reduction, channel),
                ME.MinkowskiSigmoid())
            # the reference's _PYTORCH_INDEX default writes cloud b to row batch_index[b], right
            # only for some origin orders; the _KERNEL mode gives the same result everywhere
            self.pooling = ME.MinkowskiGlobalPooling(ME.PoolingMode.GLOBAL_AVG_POOLING_KERNEL)
            self.broadcast_mul = ME.MinkowskiBroadcastMultiplication()

        def forward(self, x):
            return self.broadcast_mul(x, self.fc(self.pooling(x)))

    return SELayer()


def se_basic_block(ME, inplanes, planes, stride=1, dilation=1, downsample=None, reduction=16,
                   dimension=3):
    """BasicBlock with the squeeze-excitation gate before the residual add (reference
    senet_block.py SEBasicBlock)."""
    BasicBlock = _basic_block(ME)
    bn_relu = _bn_relu(ME)

    class SEBasicBlock(BasicBlock):
        def __init__(self):
            super().__init__(inplanes, planes, stride=stride, dilation=dilation,
                             downsample=downsample, dimension=dimension)
            self.se = se_layer(ME, planes, reduction)

        def forward(self, x):
            residual = x
            out = bn_relu(self.norm1, self.relu, self.conv1(x))
            out = self.se(self.norm2(self.conv2(out)))
            if self.downsample is not None:
                residual = self.downsample(x)
            out += residual
            return self.relu(out)

    return SEBasicBlock()


def resnet(name, ME, in_channels=3, out_channels=40, D=3, dropout=0.5):
    """Instantiate `name` ("ResNet14", "ResNet18", "ResNet34") on module handle `ME`.  `dropout`
    is the probability of the dropout before the last convolution (the reference's 0.5)."""
    layers = _LAYERS[name]
    block = _basic_block(ME)
    planes = (64, 128, 256, 512)

    class ResNet(nn.Module):
        def __init__(self):
            super().__init__()
            self.D = D
            self.inplanes = 64
            self.conv1 = nn.Sequential(
                ME.MinkowskiConvolution(in_channels, self.inplanes, kernel_size=3, stride=2,
                                        dimension=D),
                ME.MinkowskiInstanceNorm(self.inplanes),
                ME.MinkowskiReLU(inplace=True),
                ME.MinkowskiMaxPooling(kernel_size=2, stride=2, dimension=D))
            self.layer1 = self._make_layer(planes[0], layers[0], stride=2)
            self.layer2 = self._make_layer(planes[1], layers[1], stride=2)
            self.layer3 = self._make_layer(planes[2], layers[2], stride=2)
            self.layer4 = self._make_layer(planes[3], layers[3], stride=2)
            self.conv5 = nn.Sequential(
                ME.MinkowskiDropout(p=dropout),
                ME.MinkowskiConvolution(self.inplanes, self.inplanes, kernel_size=3, stride=3,
                                        dimension=D),
                ME.MinkowskiInstanceNorm(self.inplanes),
                ME.MinkowskiGELU())
            self.glob_pool = ME.MinkowskiGlobalMaxPooling()
            self.final = ME.MinkowskiLinear(self.inplanes, out_channels, bias=True)
            for m in self.modules():
                if isinstance(m, ME.MinkowskiConvolution):
                    ME.utils.kaiming_normal_(m.kernel, mode="fan_out", nonlinearity="relu")
                if isinstance(m, ME.MinkowskiBatchNorm):
                    nn.init.constant_(m.bn.weight, 1)
                    nn.init.constant_(m.bn.bias, 0)

        def _make_layer(self, planes_, blocks, stride=1):
            downsample = None
            if stride != 1 or self.inplanes != planes_ * block.expansion:
                downsample = nn.Sequential(
                    ME.MinkowskiConvolution(self.inplanes, planes_ * block.expansion,
                                            kernel_size=1, stride=stride, dimension=D),
                    ME.MinkowskiBatchNorm(planes_ * block.expansion))
            mods = [block(self.inplanes, planes_, stride=stride, downsample=downsample,
                          dimension=D)]
            self.inplanes = planes_ * block.expansion
            for _ in range(1, blocks):
                mods.append(block(self.inplanes, planes_, stride=1, dimension=D))
            return nn.Sequential(*mods)

        def forward(self, x):
            x = self.conv1(x)
            x = self.layer1(x)
            x = self.layer2(x)
            x = self.layer3(x)
            x = self.layer4(x)
            x = self.conv5(x)
            x = self.glob_pool(x)
            return self.final(x)

    ResNet.__name__ = name
    return ResNet()
