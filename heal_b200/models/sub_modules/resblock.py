"""ResNet / ResNeXt blocks mirror (opencood/models/sub_modules/resblock.py:18-219).

nn.Conv2d / nn.BatchNorm2d modules are kept only as parameter containers with the reference's
state-dict names; forward runs each conv+BN(+residual)+ReLU as ONE kernel on channels-last `Act`s."""
from typing import List

import torch.nn as nn

from ... import ops
from ...engine import conv_bn_act


def conv3x3(inp, out, stride=1, groups=1):
    return nn.Conv2d(inp, out, 3, stride=stride, padding=1, groups=groups, bias=False)


def conv1x1(inp, out, stride=1):
    return nn.Conv2d(inp, out, 1, stride=stride, bias=False)


class BasicBlock(nn.Module):
    expansion = 1

    def __init__(self, inplanes, planes, stride=1, downsample=None, groups=1, base_width=64, dilation=1, norm_layer=None):
        super().__init__()
        if groups != 1 or base_width != 64:
            raise ValueError('BasicBlock only supports groups=1 and base_width=64')
        self.conv1 = conv3x3(inplanes, planes, stride)
        self.bn1 = nn.BatchNorm2d(planes)
        self.relu = nn.ReLU(inplace=True)
        self.conv2 = conv3x3(planes, planes)
        self.bn2 = nn.BatchNorm2d(planes)
        self.downsample = downsample
        self.stride = stride

    out_channels = property(lambda self: self.conv2.out_channels)

    def _stem_eligible(self):
        d = self.downsample
        return (d is not None and self.conv1.in_channels == 64 and self.conv1.out_channels == 64 and self.conv1.stride == (2, 2)
                and self.conv1.padding == (1, 1) and d[0].kernel_size == (1, 1) and d[0].stride == (2, 2) and d[0].out_channels == 64)

    def forward_nhwc(self, x, out=None):
        if isinstance(x, ops.SparseCanvas):
            from ... import engine
            if engine.SPARSE_STEM and self._stem_eligible() and x.H % 2 == 0 and x.W % 2 == 0:
                # scatter + conv1/bn1/ReLU + downsample/bn in one kernel, straight from the pillar list
                y, idt = ops.sparse_stem(x, engine.packed(self.conv1, self.bn1, True, kind="simt"),
                                         engine.packed(self.downsample[0], self.downsample[1], False, kind="simt"), engine.act_fmt(),
                                         tensor_cores=(engine.STEM_TC and engine.PRECISION != "fp32"))
                return conv_bn_act(y, self.conv2, self.bn2, relu=True, residual=idt, out=out)
            from ...engine import act_fmt
            x = x.dense(act_fmt())
        idt = x
        if self.downsample is not None:
            idt = conv_bn_act(x, self.downsample[0], self.downsample[1], relu=False)
        y = conv_bn_act(x, self.conv1, self.bn1, relu=True)
        return conv_bn_act(y, self.conv2, self.bn2, relu=True, residual=idt, out=out)


class Bottleneck(nn.Module):
    expansion = 4   # PyramidFusion sets Bottleneck.expansion = 1 (pyramid_fuse.py:72)

    def __init__(self, inplanes, planes, stride=1, downsample=None, groups=1, base_width=64, dilation=1, norm_layer=None):
        super().__init__()
        width = int(planes * (base_width / 64.)) * groups
        self.conv1 = conv1x1(inplanes, width)
        self.bn1 = nn.BatchNorm2d(width)
        self.conv2 = conv3x3(width, width, stride, groups)
        self.bn2 = nn.BatchNorm2d(width)
        self.conv3 = conv1x1(width, planes * self.expansion)
        self.bn3 = nn.BatchNorm2d(planes * self.expansion)
        self.relu = nn.ReLU(inplace=True)
        self.downsample = downsample
        self.stride = stride

    out_channels = property(lambda self: self.conv3.out_channels)

    def _fused_eligible(self, x) -> bool:
        """The shapes ops.bottleneck_tc runs: PyramidFusion's level-0 blocks (64 -> 128 -> 64, 32 groups, stride 1)."""
        from ... import engine
        c1, c2, c3 = self.conv1, self.conv2, self.conv3
        return (isinstance(x, ops.Act) and x.fmt == engine.act_fmt() and engine.PRECISION in ("tc32", "bf16")
                and not engine.BF16_WEIGHTS and self.downsample is None and c2.stride == (1, 1) and c2.groups == 32
                and c1.in_channels == x.C == c3.out_channels == 64 and c1.out_channels == c2.out_channels == c3.in_channels == 128
                and c2.in_channels == 128)

    def _gconv_reduce_eligible(self, x) -> bool:
        """The shapes ops.gconv_reduce_tc runs after the expand: PyramidFusion's stride-1 level-1 and level-2 blocks
        (C -> 2 C -> C with C = 128 or 256, 32 groups, no downsample)."""
        from ... import engine
        c1, c2, c3 = self.conv1, self.conv2, self.conv3
        return (isinstance(x, ops.Act) and x.fmt == engine.act_fmt() and engine.PRECISION in ("tc32", "bf16")
                and not engine.BF16_WEIGHTS and self.downsample is None and c2.stride == (1, 1) and c2.groups == 32
                and x.C == c1.in_channels == c3.out_channels and x.C in (128, 256)
                and c1.out_channels == c2.in_channels == c2.out_channels == c3.in_channels == 2 * x.C)

    def forward_nhwc(self, x, out=None):
        if self._fused_eligible(x) and (out is None or out.fmt == x.fmt):
            from ... import engine
            pcs = [engine.packed(c, b, True, kind="tc2") for c, b in ((self.conv1, self.bn1), (self.conv2, self.bn2), (self.conv3, self.bn3))]
            return ops.bottleneck_tc(x, *pcs, out=out)
        if self._gconv_reduce_eligible(x) and (out is None or out.fmt == x.fmt):
            from ... import engine
            y = conv_bn_act(x, self.conv1, self.bn1, relu=True)
            pc2, pc3 = (engine.packed(c, b, True, kind="tc2") for c, b in ((self.conv2, self.bn2), (self.conv3, self.bn3)))
            return ops.gconv_reduce_tc(y, pc2, pc3, x, out=out)
        idt = x
        if self.downsample is not None:
            idt = conv_bn_act(x, self.downsample[0], self.downsample[1], relu=False)
        y = conv_bn_act(x, self.conv1, self.bn1, relu=True)
        y = conv_bn_act(y, self.conv2, self.bn2, relu=True)
        return conv_bn_act(y, self.conv3, self.bn3, relu=True, residual=idt, out=out)


class ResNetModified(nn.Module):
    def __init__(self, block, layers: List[int], layer_strides: List[int], num_filters: List[int],
                 zero_init_residual=False, groups=1, width_per_group=64, replace_stride_with_dilation=None,
                 norm_layer=None, inplanes=64):
        super().__init__()
        self.inplanes = inplanes
        self.groups = groups
        self.base_width = width_per_group
        self.layernum = len(num_filters)
        for i in range(self.layernum):
            setattr(self, f"layer{i}", self._make_layer(block, num_filters[i], layers[i], layer_strides[i]))
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode='fan_out', nonlinearity='relu')
            elif isinstance(m, nn.BatchNorm2d):
                nn.init.constant_(m.weight, 1)
                nn.init.constant_(m.bias, 0)

    def _make_layer(self, block, planes, blocks, stride):
        downsample = None
        if stride != 1 or self.inplanes != planes * block.expansion:
            downsample = nn.Sequential(conv1x1(self.inplanes, planes * block.expansion, stride),
                                       nn.BatchNorm2d(planes * block.expansion))
        seq = [block(self.inplanes, planes, stride, downsample, self.groups, self.base_width)]
        self.inplanes = planes * block.expansion
        for _ in range(1, blocks):
            seq.append(block(self.inplanes, planes, groups=self.groups, base_width=self.base_width))
        return nn.Sequential(*seq)

    # A level whose largest per-layer tensor (all images) exceeds this is run image by image ("agent-major"): each agent
    # goes through the whole level before the next one starts, so that its intermediates (<= 34 MB at 256x256) stay
    # resident in L2 (50 MB on the H100) between producer and consumer instead of round-tripping HBM.
    # Off by default: on the B200 build it was first tried on, the extra launches cost more than the L2 residency saved; it has
    # not been measured on the H100.  Set HEAL_AGENT_MAJOR_MB to experiment.
    AGENT_MAJOR_BYTES = (int(__import__('os').environ.get('HEAL_AGENT_MAJOR_MB', '0')) << 20) or (1 << 62)

    def _run_level(self, layer, x, out=None):
        blocks = list(layer)
        stride = blocks[0].stride
        Ho, Wo = (x.H - 1) // stride + 1, (x.W - 1) // stride + 1
        widest = max(max(getattr(b, "conv1").out_channels, b.out_channels) for b in blocks)
        biggest = x.N * max(x.H * x.W * max(x.C, blocks[0].conv1.out_channels), Ho * Wo * widest) * 4
        if x.N == 1 or biggest <= self.AGENT_MAJOR_BYTES or isinstance(x, ops.SparseCanvas):
            for j, blk in enumerate(blocks):
                x = blk.forward_nhwc(x, out=out if j == len(blocks) - 1 else None)
            return x
        from ...engine import act_fmt
        if out is None:
            out = ops.act_empty(x.N, Ho, Wo, blocks[-1].out_channels, act_fmt(), x.device)
        for a in range(x.N):
            xi = x.image(a)
            for j, blk in enumerate(blocks):
                xi = blk.forward_nhwc(xi, out=out.image(a) if j == len(blocks) - 1 else None)
        return out

    def forward_nhwc(self, x, outs=None):
        """`outs[i]` (optional): caller-owned Act the LAST block of level i writes into (e.g. a slot of the all-gather buffer)."""
        feats = []
        for i in range(self.layernum):
            x = self._run_level(getattr(self, f"layer{i}"), x, out=outs[i] if outs is not None else None)
            feats.append(x)
        return feats

    def forward(self, x):
        return [ops.act_to_nchw(f) for f in self.forward_nhwc(ops.to_act(x))]
