"""EfficientNet-B0 with the attribute names of efficientnet_pytorch's `EfficientNet` ("efficientnet-b0"), the trunk of the
reference's CamEncode (opencood/models/sub_modules/lss_submodule.py:53, :87-111), so HEAL checkpoints load by key.

A parameter container with two forwards: `endpoints` (plain torch, CPU-capable) and `endpoints_nhwc` (csrc/mbconv.cu).
Nothing is downloaded: the weights are whatever the checkpoint holds.  `_conv_head`, `_bn1` and `_fc` exist for the keys only.

Padding follows the package's `Conv2dStaticSamePadding` built for its nominal 224 x 224 image: fixed at construction, independent of
the real input.  Stride-1 convs pad (k-1)/2 on every side; the five stride-2 convs (all at even nominal sizes) pad k-2 in total,
the smaller half first: k=3 -> (0, 1), k=5 -> (1, 2).  SURVEY.md 8c records what pins this restatement.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from ... import ops

# (kernel, stride, expand ratio, Cin, Cout, repeats)
B0_STAGES = ((3, 1, 1, 32, 16, 1), (3, 2, 6, 16, 24, 2), (5, 2, 6, 24, 40, 2), (3, 2, 6, 40, 80, 3),
             (5, 1, 6, 80, 112, 3), (5, 2, 6, 112, 192, 4), (3, 1, 6, 192, 320, 1))
BN_EPS = 1e-3
# blocks whose output is reduction_3 (40 ch, /8), reduction_4 (112 ch, /16), reduction_5 (320 ch, /32) when every stride-2
# block halves the height: the ones before the next reduction, and the last
ENDPOINT_BLOCKS = (4, 10, 15)


def same_pads(k, stride):
    """(before, after) zeros per axis of the static "same" padding at an even nominal size."""
    total = k - 1 if stride == 1 else k - 2
    return total // 2, total - total // 2


def swish(x):
    return x * torch.sigmoid(x)


def _cached(owner, name, mods, make):
    """`make()` moved to the parameters' device, rebuilt when a source tensor changes (engine._sig), kept out of the state dict."""
    from ...engine import _sig
    sig = _sig(*mods)
    hit = owner.__dict__.get(name)
    if hit is not None and hit[0] == sig:
        return hit[1]
    dev = next(mods[0].parameters()).device
    val = tuple(t.to(dev) for t in make())
    owner.__dict__[name] = (sig, val)
    return val


class MBConvBlock(nn.Module):
    def __init__(self, k, stride, expand, cin, cout):
        super().__init__()
        mid = cin * expand
        self.k, self.stride, self.skip = k, stride, stride == 1 and cin == cout
        if expand != 1:
            self._expand_conv = nn.Conv2d(cin, mid, 1, bias=False)
            self._bn0 = nn.BatchNorm2d(mid, eps=BN_EPS)
        self._depthwise_conv = nn.Conv2d(mid, mid, k, stride=stride, groups=mid, bias=False)
        self._bn1 = nn.BatchNorm2d(mid, eps=BN_EPS)
        sq = max(1, int(cin * 0.25))
        self._se_reduce = nn.Conv2d(mid, sq, 1)
        self._se_expand = nn.Conv2d(sq, mid, 1)
        self._project_conv = nn.Conv2d(mid, cout, 1, bias=False)
        self._bn2 = nn.BatchNorm2d(cout, eps=BN_EPS)

    def forward(self, x):
        y = x
        if hasattr(self, "_expand_conv"):
            y = swish(self._bn0(self._expand_conv(y)))
        p = same_pads(self.k, self.stride)
        y = swish(self._bn1(self._depthwise_conv(F.pad(y, (p[0], p[1], p[0], p[1])))))
        s = self._se_expand(swish(self._se_reduce(y.mean((2, 3), keepdim=True))))
        y = self._bn2(self._project_conv(torch.sigmoid(s) * y))
        return y + x if self.skip else y              # drop-connect is the identity in eval mode

    def forward_nhwc(self, x: ops.Act) -> ops.Act:
        y = x
        if hasattr(self, "_expand_conv"):
            w, b = _cached(self, "_pk_expand", (self._expand_conv, self._bn0), lambda: ops.pack_pwconv(self._expand_conv, self._bn0))
            y = ops.pwconv(y, w, b, swish=True)
        w, b = _cached(self, "_pk_dw", (self._depthwise_conv, self._bn1), lambda: ops.pack_dwconv(self._depthwise_conv, self._bn1))
        p = same_pads(self.k, self.stride)
        y, sums = ops.dwconv_bn_swish(y, w, b, self.k, self.stride, (p[0], p[1], p[0], p[1]))
        se = _cached(self, "_pk_se", (self._se_reduce, self._se_expand), lambda: ops.pack_se(self._se_reduce, self._se_expand))
        gate = ops.se_gate(sums, y.H * y.W, *se)
        w, b = _cached(self, "_pk_project", (self._project_conv, self._bn2), lambda: ops.pack_pwconv(self._project_conv, self._bn2))
        return ops.pwconv(y, w, b, gate=gate, residual=x if self.skip else None)


class EfficientNetB0(nn.Module):
    def __init__(self):
        super().__init__()
        self._conv_stem = nn.Conv2d(3, 32, 3, stride=2, bias=False)
        self._bn0 = nn.BatchNorm2d(32, eps=BN_EPS)
        blocks = []
        for k, stride, expand, cin, cout, repeats in B0_STAGES:
            for r in range(repeats):
                blocks.append(MBConvBlock(k, stride if r == 0 else 1, expand, cin if r == 0 else cout, cout))
        self._blocks = nn.ModuleList(blocks)
        self._conv_head = nn.Conv2d(320, 1280, 1, bias=False)
        self._bn1 = nn.BatchNorm2d(1280, eps=BN_EPS)
        self._fc = nn.Linear(1280, 1000)

    def endpoints(self, x):
        """lss_submodule.py:90-107: x (BN,3,H,W) -> {'reduction_i': map}; an endpoint is the input of every block that reduces the
        height, and the last block's output."""
        p = same_pads(3, 2)
        x = swish(self._bn0(self._conv_stem(F.pad(x, (p[0], p[1], p[0], p[1])))))
        out, prev = {}, x
        for blk in self._blocks:
            x = blk(x)
            if prev.size(2) > x.size(2):
                out[f"reduction_{len(out) + 1}"] = prev
            prev = x
        out[f"reduction_{len(out) + 1}"] = x
        return out

    def endpoints_nhwc(self, x):
        """x (BN, 3|4, H, W) fp32 CUDA, contiguous -> (reduction_3, reduction_4, reduction_5) as Act f32."""
        w, b = _cached(self, "_pk_stem", (self._conv_stem, self._bn0), lambda: ops.pack_stem_conv(self._conv_stem, self._bn0))
        y = ops.stem_conv_swish(x, w, b)
        out = []
        for i, blk in enumerate(self._blocks):
            y = blk.forward_nhwc(y)
            if i in ENDPOINT_BLOCKS:
                out.append(y)
        return out
