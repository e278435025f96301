"""The point classifier of the reference's ModelNet40 example (MinkowskiPointNet,
examples/pointnet.py and classification_modelnet40.py), written from its architecture against a
*module handle* as examples/fcnn.py is, so the identical definition runs on this package and on
the compiled reference (`oracle/_ref`, CPU):

    import minkowskiengine_b200 as ME
    from examples.pointnet import pointnet
    net = pointnet(ME, in_channel=3, out_channel=40).cuda()
    x = ME.TensorField(features, coordinates, device="cuda")   # float coordinates
    logits = net(x)     # SparseTensor on the origin map: row s = the s-th smallest batch index

A shared point MLP on the TensorField (five linear + batch norm + ReLU layers), a global max
pooling of every cloud's points with no voxelisation, and a two-layer head.  The reference's
forward returns `.F`; this returns the SparseTensor, whose coordinates name the cloud of each row.
"""
import torch.nn as nn

CHANNELS = (64, 64, 64, 128)


def pointnet(ME, in_channel, out_channel, embedding_channel=1024, channels=CHANNELS, hidden=512,
             dropout=0.5):
    """MinkowskiPointNet; `channels` are the widths of the first four point layers (the
    reference's 64, 64, 64, 128), `hidden` the width of the head (its 512), `dropout` the
    probability of the head's dropout (its 0.5)."""

    def mlp(c_in, c_out):
        return nn.Sequential(ME.MinkowskiLinear(c_in, c_out, bias=False),
                             ME.MinkowskiBatchNorm(c_out), ME.MinkowskiReLU())

    class MinkowskiPointNet(nn.Module):
        def __init__(self):
            super().__init__()
            widths = (in_channel, *channels, embedding_channel)
            self.conv1 = mlp(widths[0], widths[1])
            self.conv2 = mlp(widths[1], widths[2])
            self.conv3 = mlp(widths[2], widths[3])
            self.conv4 = mlp(widths[3], widths[4])
            self.conv5 = mlp(widths[4], widths[5])
            self.max_pool = ME.MinkowskiGlobalMaxPooling()
            self.linear1 = mlp(embedding_channel, hidden)
            self.dp1 = ME.MinkowskiDropout(p=dropout)
            self.linear2 = ME.MinkowskiLinear(hidden, out_channel, bias=True)

        def forward(self, x):
            for layer in (self.conv1, self.conv2, self.conv3, self.conv4, self.conv5):
                x = layer(x)
            return self.linear2(self.dp1(self.linear1(self.max_pool(x))))

    return MinkowskiPointNet()
