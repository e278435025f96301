"""A sparse encoder between dense tensors, written against a *module handle* as examples/convnext.py
is, so the identical definition runs on this package and on the compiled reference (`oracle/_ref`,
CPU):

    import minkowskiengine_b200 as ME
    from examples.dense_head import dense_head
    net = dense_head(ME, in_channels=2, D=3).cuda()
    out = net(volume)            # volume [B, in_channels, X, Y, Z] -> [B, out_channels, X/2, Y/2, Z/2]

Dense volume (an occupancy grid, a CT scan) -> `to_sparse` (its non-zero cells) -> two strided
convolutions with BatchNorm and ReLU -> a transposed convolution back to tensor stride 2 ->
`MinkowskiToDenseTensor` -> a dense `torch.nn.Conv3d` head: the shape of a detection or occupancy
network whose head works on a regular grid.

`MinkowskiToDenseTensor` anchors the grid on the smallest coordinate of the sparse tensor; the grid
is anchored on the volume's origin when a voxel of cell (0, .., 0) is occupied in some batch (call
`SparseTensor.dense(shape, min_coordinate)` where that cannot be assumed).
"""
import torch
import torch.nn as nn


def dense_head(ME, in_channels=2, out_channels=4, channels=(8, 16), D=3):
    """Instantiate the network on module handle `ME`."""
    assert D == 3, "the dense head is a Conv3d"

    class DenseHead(nn.Module):
        def __init__(self):
            super().__init__()
            c0, c1 = channels
            self.encoder = nn.Sequential(
                ME.MinkowskiConvolution(in_channels, c0, kernel_size=3, stride=2, dimension=D),
                ME.MinkowskiBatchNorm(c0),
                ME.MinkowskiReLU(),
                ME.MinkowskiConvolution(c0, c1, kernel_size=3, stride=2, dimension=D),
                ME.MinkowskiBatchNorm(c1),
                ME.MinkowskiReLU(),
                ME.MinkowskiConvolutionTranspose(c1, c0, kernel_size=2, stride=2, dimension=D))
            self.head = nn.Conv3d(c0, out_channels, kernel_size=3, padding=1)

        def forward(self, volume):
            y = self.encoder(ME.to_sparse(volume))          # tensor stride 2
            shape = torch.Size([volume.shape[0], channels[0]] +
                               [(s + 1) // 2 for s in volume.shape[2:]])
            return self.head(ME.MinkowskiToDenseTensor(shape)(y))

    return DenseHead()
