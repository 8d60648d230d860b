"""Shrink header of the fused map: `DownsampleConv` / `DoubleConv` (reference: opencood/models/sub_modules/downsample_conv.py:7-49).

Only the parameter containers keep the reference's shape -- the checkpoint keys are `layers.<i>.double_conv.{0,2}.{weight,bias}`, so
the two convolutions must sit at indices 0 and 2 of a Sequential called `double_conv`.  Nothing in that Sequential is ever called:
both 3x3 convolutions (bias + ReLU folded) go through `engine.conv_bn_act`, i.e. the wgmma implicit-GEMM kernel on channels-last
split-bf16 activations; these two launches are the MMA-bound ones of the frame (384->256 and 256->256 on the 256 x 256 fused map).  `forward_nhwc` is the engine-internal entry (Act in, Act out); `forward` keeps the reference's
NCHW tensor signature for callers outside the engine."""
import torch.nn as nn

from ... import ops
from ...engine import conv_bn_act


class DoubleConv(nn.Module):
    """conv(k, stride, padding) + ReLU, conv(3, pad 1) + ReLU; holds the parameters, computes through the conv engine."""

    def __init__(self, in_channels, out_channels, kernel_size, stride, padding):
        super().__init__()
        self.double_conv = nn.Sequential(
            nn.Conv2d(in_channels, out_channels, kernel_size=kernel_size, stride=stride, padding=padding),
            nn.ReLU(inplace=True),
            nn.Conv2d(out_channels, out_channels, kernel_size=3, padding=1),
            nn.ReLU(inplace=True))

    def forward_nhwc(self, x):
        x = conv_bn_act(x, self.double_conv[0], None, relu=True)
        return conv_bn_act(x, self.double_conv[2], None, relu=True)

    def forward(self, x):
        return ops.act_to_nchw(self.forward_nhwc(ops.to_act(x)))


class DownsampleConv(nn.Module):
    """`config` = hypes `shrink_header`: lists `kernal_size` (sic, the reference's key), `dim`, `stride`, `padding` + `input_dim`."""

    def __init__(self, config):
        super().__init__()
        self.layers = nn.ModuleList([])
        input_dim = config['input_dim']
        for (ksize, dim, stride, padding) in zip(config['kernal_size'], config['dim'], config['stride'], config['padding']):
            self.layers.append(DoubleConv(input_dim, dim, kernel_size=ksize, stride=stride, padding=padding))
            input_dim = dim

    def forward_nhwc(self, x):
        for layer in self.layers:
            x = layer.forward_nhwc(x)
        return x

    def forward(self, x):
        return ops.act_to_nchw(self.forward_nhwc(ops.to_act(x)))
