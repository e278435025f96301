"""The fully convolutional point classifier of the reference's ModelNet40 example
(MinkowskiFCNN, examples/classification_modelnet40.py), written from its architecture against a
*module handle* as examples/resnet.py is, so the identical definition runs on this package and on
the compiled reference (`oracle/_ref`, CPU):

    import minkowskiengine_b200 as ME
    from examples.fcnn import fcnn
    net = fcnn(ME, in_channel=3, out_channel=40).cuda()
    x = ME.TensorField(features, coordinates, device="cuda")   # float coordinates
    logits = net(x)     # SparseTensor on the origin map: row s = the s-th smallest batch index

A point MLP on the TensorField, `.sparse()`, four convolution + max-pool levels, the pooled maps of
all four levels sliced back onto the points and concatenated, a second `.sparse()` of that
concatenation, three strided convolutions, global max and average pooling and an MLP head.

`splat=True` builds MinkowskiSplatFCNN of the same example: `x.splat()` in place of the first
`.sparse()`, and the four pooled levels brought back to the points with `interpolate` in place of
`slice`.  The parameters are the same.
"""
import torch.nn as nn

CHANNELS = (32, 48, 64, 96, 128)


def fcnn(ME, in_channel, out_channel, embedding_channel=1024, channels=CHANNELS, hidden=512,
         dropout=0.5, D=3, splat=False):
    """MinkowskiFCNN (MinkowskiSplatFCNN with `splat=True`); `hidden` is the width of the head's
    MLP (the reference's 512), `dropout` the probability of its dropout (the reference's 0.5)."""

    def mlp(c_in, c_out):
        return nn.Sequential(ME.MinkowskiLinear(c_in, c_out, bias=False),
                             ME.MinkowskiBatchNorm(c_out), ME.MinkowskiLeakyReLU())

    def conv(c_in, c_out, stride):
        return nn.Sequential(ME.MinkowskiConvolution(c_in, c_out, kernel_size=3, stride=stride,
                                                     dimension=D),
                             ME.MinkowskiBatchNorm(c_out), ME.MinkowskiLeakyReLU())

    class MinkowskiFCNN(nn.Module):
        def __init__(self):
            super().__init__()
            self.D = D
            self.mlp1 = mlp(in_channel, channels[0])
            self.conv1 = conv(channels[0], channels[1], 1)
            self.conv2 = conv(channels[1], channels[2], 2)
            self.conv3 = conv(channels[2], channels[3], 2)
            self.conv4 = conv(channels[3], channels[4], 2)
            self.conv5 = nn.Sequential(conv(sum(channels[1:]), embedding_channel // 4, 2),
                                       conv(embedding_channel // 4, embedding_channel // 2, 2),
                                       conv(embedding_channel // 2, embedding_channel, 2))
            self.pool = ME.MinkowskiMaxPooling(kernel_size=3, stride=2, dimension=D)
            # the reference's default _PYTORCH_INDEX modes write cloud b to row batch_index[b],
            # right only for some origin orders, so the max and average rows of a cloud can land
            # on different rows of ME.cat; the _KERNEL modes give the same result everywhere
            self.global_max_pool = ME.MinkowskiGlobalPooling(
                ME.PoolingMode.GLOBAL_MAX_POOLING_KERNEL)
            self.global_avg_pool = ME.MinkowskiGlobalPooling(
                ME.PoolingMode.GLOBAL_AVG_POOLING_KERNEL)
            self.final = nn.Sequential(mlp(embedding_channel * 2, hidden),
                                       ME.MinkowskiDropout(p=dropout), mlp(hidden, hidden),
                                       ME.MinkowskiLinear(hidden, out_channel, bias=True))
            for m in self.modules():
                if isinstance(m, ME.MinkowskiConvolution):
                    ME.utils.kaiming_normal_(m.kernel, mode="fan_out", nonlinearity="relu")
                if isinstance(m, ME.MinkowskiBatchNorm):
                    nn.init.constant_(m.bn.weight, 1)
                    nn.init.constant_(m.bn.bias, 0)

        def forward(self, x):
            x = self.mlp1(x)
            y = x.splat() if splat else x.sparse()
            ys = []
            for layer in (self.conv1, self.conv2, self.conv3, self.conv4):
                y = self.pool(layer(y))
                ys.append(y)
            if splat:
                x = ME.cat(*[yi.interpolate(x) for yi in ys])
            else:
                x = ME.cat(*[yi.slice(x) for yi in ys])
            y = self.conv5(x.sparse())
            return self.final(ME.cat(self.global_max_pool(y), self.global_avg_pool(y)))

    return MinkowskiFCNN()
