"""AlignNet mirror (opencood/models/sub_modules/feature_alignnet.py:12-39) with the two `core_method`s HEAL's yamls use:
`identity` (base modality) and `convnext` (stage-2 modalities, m1m2m3m4.yaml:204-209: 3 ConvNeXt blocks, dim 64).

ConvNeXtBlock (feature_alignnet_modules.py:299-345): dwconv 7x7 -> LayerNorm(channels_last, eps 1e-6) -> Linear(dim, 4 dim) ->
GELU -> Linear(4 dim, dim) -> gamma -> + input.  The nn modules below only hold the parameters under the reference's state-dict
names; per block the compute is three kernels on channels-last `Act`s:
  heal_dwconv_layernorm                         depthwise conv + bias + LayerNorm, one HBM pass
  heal_conv2d_tc 1x1 dim -> 4 dim, GELU         (pwconv1 as a 1x1 convolution on wgmma, erf GELU in the epilogue)
  heal_conv2d_tc 1x1 4 dim -> dim + residual    (pwconv2 with gamma folded into weight and bias, block input as the residual)
The other aligners of the reference (scaligner, resnet1x1/3x3, sdta, cbam, fanet) are not used by any HEAL yaml and raise."""
import torch
import torch.nn as nn

from ... import ops
from ...engine import conv_bn_act, require_eval, act_fmt, _sig


class LayerNorm(nn.Module):
    """feature_alignnet_modules.py:12-31 (parameter container; channels_last only on this path)."""

    def __init__(self, normalized_shape, eps=1e-6, data_format="channels_last"):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(normalized_shape))
        self.bias = nn.Parameter(torch.zeros(normalized_shape))
        self.eps = eps
        if data_format != "channels_last":
            raise NotImplementedError(data_format)


class ConvNeXtBlock(nn.Module):
    def __init__(self, dim, drop_path=0., layer_scale_init_value=1e-6, kernel_size=7, deform=False):
        super().__init__()
        if deform:
            raise NotImplementedError("deformable ConvNeXt blocks need mmcv and are not used by the HEAL yamls")
        self.dim, self.kernel_size = dim, kernel_size
        self.dwconv = nn.Conv2d(dim, dim, kernel_size=kernel_size, padding=kernel_size // 2, groups=dim)
        self.norm = LayerNorm(dim, eps=1e-6)
        self.pwconv1 = nn.Linear(dim, 4 * dim)
        self.act = nn.GELU()
        self.pwconv2 = nn.Linear(4 * dim, dim)
        self.gamma = nn.Parameter(layer_scale_init_value * torch.ones((dim)), requires_grad=True) if layer_scale_init_value > 0 else None
        self._derived = None

    def _prepare(self):
        """dw weights tap-major, the two Linear layers as 1x1 Conv2d containers (gamma folded into the second)."""
        sig = (_sig(self.dwconv, self.norm, self.pwconv1, self.pwconv2),
               None if self.gamma is None else (self.gamma.data_ptr(), self.gamma._version, str(self.gamma.device)))
        if self._derived is not None and self._derived[0] == sig:
            return self._derived[1]
        dev, d, k = self.dwconv.weight.device, self.dim, self.kernel_size
        with torch.no_grad():
            dw = self.dwconv.weight.detach().float().reshape(d, k * k).t().contiguous()            # (k*k, C)
            c1 = nn.Conv2d(d, 4 * d, 1).to(dev)
            c1.weight.copy_(self.pwconv1.weight.detach().reshape(4 * d, d, 1, 1))
            c1.bias.copy_(self.pwconv1.bias.detach())
            c2 = nn.Conv2d(4 * d, d, 1).to(dev)
            g = self.gamma.detach().double() if self.gamma is not None else torch.ones(d, dtype=torch.float64, device=dev)
            c2.weight.copy_((self.pwconv2.weight.detach().double() * g[:, None]).float().reshape(d, 4 * d, 1, 1))
            c2.bias.copy_((self.pwconv2.bias.detach().double() * g).float())
        out = (dw, self.dwconv.bias.detach().float().contiguous(), c1, c2)
        self._derived = (sig, out)
        return out

    def forward_nhwc(self, x: "ops.Act") -> "ops.Act":
        dw, db, c1, c2 = self._prepare()
        y = ops.dwconv_layernorm(x, dw, db, self.kernel_size, self.norm.weight.detach(), self.norm.bias.detach(), self.norm.eps,
                                 out_fmt=act_fmt())
        y = conv_bn_act(y, c1, None, relu=2)                              # Linear + GELU
        return conv_bn_act(y, c2, None, relu=False, residual=x)           # Linear * gamma + input


class ConvNeXt(nn.Module):
    def __init__(self, args):
        super().__init__()
        dim, ks, nb = args['dim'], args.get("kernel_size", 7), args['num_of_blocks']
        self.model = nn.Sequential(*[ConvNeXtBlock(dim, kernel_size=ks, deform=args.get('deform', False)) for _ in range(nb)])

    def forward_nhwc(self, x):
        for blk in self.model:
            x = blk.forward_nhwc(x)
        return x


class AlignNet(nn.Module):
    def __init__(self, args):
        super().__init__()
        model_name = (args or {}).get('core_method', 'identity')
        if model_name == 'identity':
            self.channel_align = nn.Identity()
        elif model_name == 'convnext':
            self.channel_align = ConvNeXt(args['args'])
        else:
            raise NotImplementedError(f"aligner '{model_name}' is not used by any HEAL yaml and is outside the heal_b200 scope "
                                      "(identity, convnext)")
        if (args or {}).get("spatial_align", False):
            raise NotImplementedError("spatial_align")       # the reference raises too (feature_alignnet.py:35-36)

    @property
    def is_identity(self):
        return isinstance(self.channel_align, nn.Identity)

    def forward_nhwc(self, x):
        if self.is_identity:
            return x
        require_eval(self)
        if isinstance(x, ops.SparseCanvas):
            x = x.dense(act_fmt())
        return self.channel_align.forward_nhwc(x)

    def forward(self, x):
        """reference signature: (N,C,H,W) tensor in, tensor out."""
        if self.is_identity:
            return x
        return ops.act_to_nchw(self.forward_nhwc(ops.to_act(x)))
