"""Generative shape completion (reference: examples/completion.py:150-513), written against a
*module handle* as examples/resnet.py is, so the identical definition runs on this package and on
the compiled reference (`oracle/_ref`, CPU):

    import minkowskiengine_b200 as ME
    from examples.completion import completion_net, shell_pair
    net = completion_net(ME).cuda()
    x = ME.SparseTensor(torch.ones(len(partial), 1), partial, device="cuda")
    target_key, _ = x.coordinate_manager.insert_and_map(full.cuda(), string_id="target")
    out_cls, targets, completed = net(x, target_key)

The encoder halves the resolution `levels` times; every decoder level up-samples with a generative
transposed convolution, adds the encoder tensor of its level (a union of two coordinate maps),
classifies every voxel and prunes those with a negative logit (in training, the voxels of the
target are kept as well).  The reference network is `levels = 6` with channels
ENC_CHANNELS / DEC_CHANNELS.
"""
import torch
import torch.nn as nn

ENC_CHANNELS = (16, 32, 64, 128, 256, 512, 1024)
DEC_CHANNELS = (16, 32, 64, 128, 256, 512, 1024)


def completion_net(ME, enc_channels=ENC_CHANNELS, dec_channels=DEC_CHANNELS, in_channels=1):
    """CompletionNet with len(enc_channels) - 1 levels; enc_channels[l] / dec_channels[l] are the
    widths at tensor stride 2^l."""
    enc_ch, dec_ch = list(enc_channels), list(dec_channels)
    levels = len(enc_ch) - 1
    assert levels >= 1 and len(dec_ch) == len(enc_ch)

    def conv_bn_elu(cin, cout, **kw):
        return [ME.MinkowskiConvolution(cin, cout, dimension=3, **kw), ME.MinkowskiBatchNorm(cout),
                ME.MinkowskiELU()]

    class CompletionNet(nn.Module):
        def __init__(self):
            super().__init__()
            self.enc_block_s1 = nn.Sequential(*conv_bn_elu(in_channels, enc_ch[0], kernel_size=3,
                                                           stride=1))
            self.enc_blocks = nn.ModuleList([
                nn.Sequential(*conv_bn_elu(enc_ch[l - 1], enc_ch[l], kernel_size=2, stride=2),
                              *conv_bn_elu(enc_ch[l], enc_ch[l], kernel_size=3))
                for l in range(1, levels + 1)])
            # decoder level l: stride 2^(l+1) -> 2^l, deepest first
            self.dec_blocks = nn.ModuleList()
            self.dec_cls = nn.ModuleList()
            for l in reversed(range(levels)):
                cin = enc_ch[levels] if l == levels - 1 else dec_ch[l + 1]
                self.dec_blocks.append(nn.Sequential(
                    ME.MinkowskiGenerativeConvolutionTranspose(
                        cin, dec_ch[l], kernel_size=4 if l == levels - 1 else 2, stride=2,
                        dimension=3),
                    ME.MinkowskiBatchNorm(dec_ch[l]), ME.MinkowskiELU(),
                    *conv_bn_elu(dec_ch[l], dec_ch[l], kernel_size=3)))
                self.dec_cls.append(ME.MinkowskiConvolution(dec_ch[l], 1, kernel_size=1, bias=True,
                                                            dimension=3))
            self.pruning = ME.MinkowskiPruning()

        def get_target(self, out, target_key, kernel_size=1):
            """Rows of `out` whose coordinate is in the target map strided to out's stride."""
            with torch.no_grad():
                target = torch.zeros(len(out), dtype=torch.bool, device=out.device)
                cm = out.coordinate_manager
                strided_target_key = cm.stride(target_key, out.tensor_stride[0])
                kernel_map = cm.kernel_map(out.coordinate_map_key, strided_target_key,
                                           kernel_size=kernel_size, region_type=1)
                for k, curr_in in kernel_map.items():
                    target[curr_in[0].long()] = 1
            return target

        def forward(self, partial_in, target_key):
            out_cls, targets = [], []
            enc = [self.enc_block_s1(partial_in)]
            for blk in self.enc_blocks:
                enc.append(blk(enc[-1]))
            dec = enc[levels]
            for j, l in enumerate(reversed(range(levels))):
                dec = self.dec_blocks[j](dec)
                dec = dec + enc[l]                      # union with the encoder tensor
                dec_cls = self.dec_cls[j](dec)
                keep = (dec_cls.F > 0).squeeze()
                target = self.get_target(dec, target_key)
                targets.append(target)
                out_cls.append(dec_cls)
                if self.training and l > 0:             # the last level keeps predictions only
                    keep += target
                dec = self.pruning(dec, keep)
            return out_cls, targets, dec

    return CompletionNet()


def completion_loss(out_cls, targets):
    """Per-level binary cross-entropy, averaged over the levels (reference completion.py:551-560)."""
    crit = nn.BCEWithLogitsLoss()
    loss = 0
    for out, target in zip(out_cls, targets):
        loss = loss + crit(out.F.squeeze(1).float(), target.type(out.F.dtype).float()) / len(out_cls)
    return loss


def shell_pair(radius, seed, batch=0, cut=0.3):
    """Synthetic completion pair: (partial, full) int32 [n, 4] coordinates of one voxelised
    sphere shell of `radius`, the partial one missing the cap above z > cut * radius of a randomly
    rotated frame."""
    g = torch.Generator().manual_seed(seed)
    r = int(radius) + 2
    ax = torch.arange(-r, r + 1)
    xyz = torch.stack(torch.meshgrid(ax, ax, ax, indexing="ij"), -1).reshape(-1, 3)
    d = xyz.double().norm(dim=1)
    full = xyz[(d - radius).abs() < 0.5]
    q, _ = torch.linalg.qr(torch.randn(3, 3, generator=g, dtype=torch.float64))
    z = full.double() @ q[:, 2]
    partial = full[z <= cut * radius]
    b = lambda c: torch.cat([torch.full((len(c), 1), batch, dtype=torch.int32), c.int()], 1)
    return b(partial), b(full)
