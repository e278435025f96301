"""The reference's StackUNet example (examples/stack_unet.py), written from its architecture against
a *module handle* as examples/resnet.py is, so the identical definition runs on this package and on
the compiled reference (`oracle/_ref`, CPU):

    import minkowskiengine_b200 as ME
    from examples.stack_unet import stack_unet
    net = stack_unet(ME, in_nchannel=3, out_nchannel=5, D=2).cuda()
    logits = net(ME.SparseTensor(features, coordinates, device="cuda"))   # a torch.Tensor [N, 5]

Two branches summed on the input's coordinates (MinkowskiStackSum): a stride-1 convolution, and a
stride-2 convolution whose output is summed with a stride-4 convolution, a transposed convolution
and a k2s2 unpooling back to stride 2, then unpooled (k2s2) back to stride 1.  MinkowskiToFeature
and a Linear layer give per-voxel logits.
"""
import torch.nn as nn


def stack_unet(ME, in_nchannel, out_nchannel, D, channels=(16, 32)):
    c1, c2 = channels
    return nn.Sequential(
        ME.MinkowskiStackSum(
            ME.MinkowskiConvolution(in_nchannel, c1, kernel_size=3, stride=1, dimension=D),
            nn.Sequential(
                ME.MinkowskiConvolution(in_nchannel, c1, kernel_size=3, stride=2, dimension=D),
                ME.MinkowskiStackSum(
                    nn.Identity(),
                    nn.Sequential(
                        ME.MinkowskiConvolution(c1, c2, kernel_size=3, stride=2, dimension=D),
                        ME.MinkowskiConvolutionTranspose(c2, c1, kernel_size=3, stride=1,
                                                         dimension=D),
                        ME.MinkowskiPoolingTranspose(kernel_size=2, stride=2, dimension=D),
                    ),
                ),
                ME.MinkowskiPoolingTranspose(kernel_size=2, stride=2, dimension=D),
            ),
        ),
        ME.MinkowskiToFeature(),
        nn.Linear(c1, out_nchannel, bias=True),
    )
