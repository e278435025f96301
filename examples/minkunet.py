"""MinkUNet family (reference: examples/minkunet.py:35-245, examples/resnet.py:53-156),
written against a *module handle* so the identical definition runs on this package
(`minkowskiengine_b200`) and on the compiled reference (`oracle/_ref`, CPU) for baselines:

    import minkowskiengine_b200 as ME
    from examples.minkunet import minkunet
    net = minkunet("MinkUNet34C", ME, in_channels=3, out_channels=20, D=3).cuda()
"""
import torch.nn as nn

_LAYERS = {
    "MinkUNet14": (1, 1, 1, 1, 1, 1, 1, 1),
    "MinkUNet18": (2, 2, 2, 2, 2, 2, 2, 2),
    "MinkUNet34": (2, 3, 4, 6, 2, 2, 2, 2),
}
_PLANES = {
    "": (32, 64, 128, 256, 256, 128, 96, 96),
    "A": (32, 64, 128, 256, 128, 128, 96, 96),
    "B": (32, 64, 128, 256, 128, 128, 128, 128),
    "C": (32, 64, 128, 256, 192, 192, 128, 128),
    "D": (32, 64, 128, 256, 384, 384, 384, 384),
}
# the 34 family re-defines A/B/C (examples/minkunet.py:233-245)
_PLANES_34 = {
    "": (32, 64, 128, 256, 256, 128, 96, 96),
    "A": (32, 64, 128, 256, 256, 128, 64, 64),
    "B": (32, 64, 128, 256, 256, 128, 64, 32),
    "C": (32, 64, 128, 256, 256, 128, 96, 96),
}


def _bn_relu(ME):
    """relu(norm(x) [+ residual]): one fused pass on module handles that provide it
    (minkowskiengine_b200.fused_bn_relu), the reference's three separate ops otherwise."""
    fused = getattr(ME, "fused_bn_relu", None)

    def bn_relu(norm, relu, x, residual=None):
        if fused is not None:
            return fused(norm, x, residual)
        out = norm(x)
        if residual is not None:
            out += residual
        return relu(out)
    return bn_relu


def _conv_bn_relu(ME):
    """relu(norm(conv(x)) [+ residual]) on module handles that provide it
    (minkowskiengine_b200.fused_conv_bn_relu: one pass in eval mode under no_grad, the convolution
    then fused_bn_relu otherwise), the reference's separate ops otherwise."""
    fused = getattr(ME, "fused_conv_bn_relu", None)
    bn_relu = _bn_relu(ME)

    def conv_bn_relu(conv, norm, relu, x, residual=None):
        if fused is not None:
            return fused(conv, norm, x, residual)
        return bn_relu(norm, relu, conv(x), residual)
    return conv_bn_relu


def _basic_block(ME):
    bn_relu = _bn_relu(ME)
    conv_bn_relu = _conv_bn_relu(ME)

    class BasicBlock(nn.Module):
        expansion = 1

        def __init__(self, inplanes, planes, stride=1, dilation=1, downsample=None,
                     bn_momentum=0.1, dimension=-1):
            super().__init__()
            self.conv1 = ME.MinkowskiConvolution(inplanes, planes, kernel_size=3, stride=stride,
                                                 dilation=dilation, dimension=dimension)
            self.norm1 = ME.MinkowskiBatchNorm(planes, momentum=bn_momentum)
            self.conv2 = ME.MinkowskiConvolution(planes, planes, kernel_size=3, stride=1,
                                                 dilation=dilation, dimension=dimension)
            self.norm2 = ME.MinkowskiBatchNorm(planes, momentum=bn_momentum)
            self.relu = ME.MinkowskiReLU(inplace=True)
            self.downsample = downsample

        def forward(self, x):
            out = conv_bn_relu(self.conv1, self.norm1, self.relu, x)
            if self.downsample is None:
                return conv_bn_relu(self.conv2, self.norm2, self.relu, out, x)
            if self.training:
                # training fuses nothing here: keep conv2 ahead of the downsample, the order in
                # which the block has always launched its layers
                out = self.conv2(out)
                return bn_relu(self.norm2, self.relu, out, self.downsample(x))
            return conv_bn_relu(self.conv2, self.norm2, self.relu, out, self.downsample(x))

    return BasicBlock


def minkunet(name, ME, in_channels=3, out_channels=20, D=3):
    """Instantiate `name` (e.g. "MinkUNet14", "MinkUNet34C") on module handle `ME`."""
    base = name.rstrip("ABCD")
    variant = name[len(base):]
    layers = _LAYERS[base]
    planes = (_PLANES_34 if base == "MinkUNet34" else _PLANES)[variant]
    block = _basic_block(ME)
    conv_bn_relu = _conv_bn_relu(ME)
    init_dim = 32

    class MinkUNet(nn.Module):
        def __init__(self):
            super().__init__()
            self.D = D
            self.inplanes = init_dim
            conv, convtr, bn = ME.MinkowskiConvolution, ME.MinkowskiConvolutionTranspose, \
                ME.MinkowskiBatchNorm
            self.conv0p1s1 = conv(in_channels, self.inplanes, kernel_size=5, dimension=D)
            self.bn0 = bn(self.inplanes)
            self.conv1p1s2 = conv(self.inplanes, self.inplanes, kernel_size=2, stride=2, dimension=D)
            self.bn1 = bn(self.inplanes)
            self.block1 = self._make_layer(planes[0], layers[0])
            self.conv2p2s2 = conv(self.inplanes, self.inplanes, kernel_size=2, stride=2, dimension=D)
            self.bn2 = bn(self.inplanes)
            self.block2 = self._make_layer(planes[1], layers[1])
            self.conv3p4s2 = conv(self.inplanes, self.inplanes, kernel_size=2, stride=2, dimension=D)
            self.bn3 = bn(self.inplanes)
            self.block3 = self._make_layer(planes[2], layers[2])
            self.conv4p8s2 = conv(self.inplanes, self.inplanes, kernel_size=2, stride=2, dimension=D)
            self.bn4 = bn(self.inplanes)
            self.block4 = self._make_layer(planes[3], layers[3])
            self.convtr4p16s2 = convtr(self.inplanes, planes[4], kernel_size=2, stride=2, dimension=D)
            self.bntr4 = bn(planes[4])
            self.inplanes = planes[4] + planes[2] * block.expansion
            self.block5 = self._make_layer(planes[4], layers[4])
            self.convtr5p8s2 = convtr(self.inplanes, planes[5], kernel_size=2, stride=2, dimension=D)
            self.bntr5 = bn(planes[5])
            self.inplanes = planes[5] + planes[1] * block.expansion
            self.block6 = self._make_layer(planes[5], layers[5])
            self.convtr6p4s2 = convtr(self.inplanes, planes[6], kernel_size=2, stride=2, dimension=D)
            self.bntr6 = bn(planes[6])
            self.inplanes = planes[6] + planes[0] * block.expansion
            self.block7 = self._make_layer(planes[6], layers[6])
            self.convtr7p2s2 = convtr(self.inplanes, planes[7], kernel_size=2, stride=2, dimension=D)
            self.bntr7 = bn(planes[7])
            self.inplanes = planes[7] + init_dim
            self.block8 = self._make_layer(planes[7], layers[7])
            self.final = conv(planes[7] * block.expansion, out_channels, kernel_size=1, bias=True,
                              dimension=D)
            self.relu = ME.MinkowskiReLU(inplace=True)
            self._init_weights()

        def _init_weights(self):
            for m in self.modules():
                if isinstance(m, ME.MinkowskiConvolution):
                    ME.utils.kaiming_normal_(m.kernel, mode="fan_out", nonlinearity="relu")
                if isinstance(m, ME.MinkowskiBatchNorm):
                    nn.init.constant_(m.bn.weight, 1)
                    nn.init.constant_(m.bn.bias, 0)

        def _make_layer(self, planes_, blocks, stride=1, dilation=1):
            downsample = None
            if stride != 1 or self.inplanes != planes_ * block.expansion:
                downsample = nn.Sequential(
                    ME.MinkowskiConvolution(self.inplanes, planes_ * block.expansion,
                                            kernel_size=1, stride=stride, dimension=D),
                    ME.MinkowskiBatchNorm(planes_ * block.expansion))
            mods = [block(self.inplanes, planes_, stride=stride, dilation=dilation,
                          downsample=downsample, dimension=D)]
            self.inplanes = planes_ * block.expansion
            for _ in range(1, blocks):
                mods.append(block(self.inplanes, planes_, stride=1, dilation=dilation, dimension=D))
            return nn.Sequential(*mods)

        def forward(self, x):
            relu = self.relu
            out = conv_bn_relu(self.conv0p1s1, self.bn0, relu, x)
            out_p1 = out
            out = conv_bn_relu(self.conv1p1s2, self.bn1, relu, out_p1)
            out_b1p2 = self.block1(out)
            out = conv_bn_relu(self.conv2p2s2, self.bn2, relu, out_b1p2)
            out_b2p4 = self.block2(out)
            out = conv_bn_relu(self.conv3p4s2, self.bn3, relu, out_b2p4)
            out_b3p8 = self.block3(out)
            out = conv_bn_relu(self.conv4p8s2, self.bn4, relu, out_b3p8)
            out = self.block4(out)
            out = conv_bn_relu(self.convtr4p16s2, self.bntr4, relu, out)
            out = ME.cat(out, out_b3p8)
            out = self.block5(out)
            out = conv_bn_relu(self.convtr5p8s2, self.bntr5, relu, out)
            out = ME.cat(out, out_b2p4)
            out = self.block6(out)
            out = conv_bn_relu(self.convtr6p4s2, self.bntr6, relu, out)
            out = ME.cat(out, out_b1p2)
            out = self.block7(out)
            out = conv_bn_relu(self.convtr7p2s2, self.bntr7, relu, out)
            out = ME.cat(out, out_p1)
            out = self.block8(out)
            return self.final(out)

    MinkUNet.__name__ = name
    return MinkUNet()
