"""Channel compressor `NaiveCompressor` (reference: opencood/models/sub_modules/naive_compress.py:5-31).

The reference's constructor, `nn.Sequential` layout and state-dict keys (`encoder.{0,1}`, `decoder.{0,1,3,4}`); the ReLUs and the
eval-mode BatchNorms (eps 1e-3) are folded into the three 3x3 convolutions, which run as three launches:
  encoder     Conv3x3(C -> c) + BN + ReLU     `engine.conv_bn_act` (Cin = C, a multiple of 64: the wgmma engine)
  decoder[0]  Conv3x3(c -> C) + BN + ReLU     c <= NARROW_MAX_C: heal_conv3x3_narrow_tc, whose K is the whole 3x3 neighbourhood
                                              of the narrow map; NARROW_MAX_C < c < 64: heal_conv2d_tc on the compressed map
                                              zero-padded to 64 channels (the encoder writes into a zeroed 64-channel buffer);
                                              c >= 64 (ratio 1): `engine.conv_bn_act`
  decoder[3]  Conv3x3(C -> C) + BN + ReLU     `engine.conv_bn_act`
with c = C // ratio.  In 'fp32' every conv runs on heal_conv2d_simt; that kernel reads channels in fours, so a compressed map
whose c is not a multiple of 4 gets a zero-filled channel pad there (and zero weights for the pad channels)."""
import torch.nn as nn

from ... import engine, ops
from ...engine import conv_bn_act, require_eval

# Widest compressed map that takes heal_conv3x3_narrow_tc.  Measured with profiles/compressor_experiment.py on an H100 80GB HBM3 at
# 700 W (DESIGN.md section 9): the narrow kernel beats the zero-padded engine path at c <= 16 in tc32 (c = 16: 129 vs 188 us at
# 5 x 64 x 256^2, 443 vs 503 us at 5 x 256 x 256^2) and loses at c = 32 (623 vs 501 us at 5 x 256 x 256^2, 174 vs 139 us at 128^2).
NARROW_MAX_C = 16


class NaiveCompressor(nn.Module):
    """A very naive compression that only compress on the channel (the reference's docstring)."""

    def __init__(self, input_dim, compress_raito):
        super().__init__()
        self.encoder = nn.Sequential(
            nn.Conv2d(input_dim, input_dim // compress_raito, kernel_size=3, stride=1, padding=1),
            nn.BatchNorm2d(input_dim // compress_raito, eps=1e-3, momentum=0.01),
            nn.ReLU())
        self.decoder = nn.Sequential(
            nn.Conv2d(input_dim // compress_raito, input_dim, kernel_size=3, stride=1, padding=1),
            nn.BatchNorm2d(input_dim, eps=1e-3, momentum=0.01),
            nn.ReLU(),
            nn.Conv2d(input_dim, input_dim, kernel_size=3, stride=1, padding=1),
            nn.BatchNorm2d(input_dim, eps=1e-3, momentum=0.01),
            nn.ReLU())

    def forward_nhwc(self, x: ops.Act) -> ops.Act:
        require_eval(self)
        enc, dec0 = self.encoder[0], self.decoder[0]
        c = enc.out_channels
        if engine.PRECISION == "fp32" and c % 4:
            z = ops.act_zeros(x.N, x.H, x.W, (c + 3) // 4 * 4, "f32", x.device)
            conv_bn_act(x, enc, self.encoder[1], relu=True, out=ops.Act(z.t[..., :c], "f32"))
            y = ops.conv2d_simt(z, engine.packed(dec0, self.decoder[1], True, kind="simt_cin4"), out_fmt="f32")
        elif engine.PRECISION != "fp32" and c <= NARROW_MAX_C and ops.narrow_eligible(dec0):
            z = conv_bn_act(x, enc, self.encoder[1], relu=True)
            y = ops.conv3x3_narrow_tc(z, engine.packed(dec0, self.decoder[1], True, kind="narrow"),
                                      planes=2 if engine.PRECISION == "tc32" else 1, out_fmt=engine.act_fmt())
        elif engine.PRECISION != "fp32" and c < 64:
            fmt = engine.act_fmt()
            z = ops.act_zeros(x.N, x.H, x.W, 64, fmt, x.device)
            conv_bn_act(x, enc, self.encoder[1], relu=True, out=ops.Act(z.t[..., :c], fmt))
            y, _ = ops.conv2d_tc(z, engine.packed(dec0, self.decoder[1], True, kind="tc2_cin64"))
        else:
            z = conv_bn_act(x, enc, self.encoder[1], relu=True)
            y = conv_bn_act(z, dec0, self.decoder[1], relu=True)
        return conv_bn_act(y, self.decoder[3], self.decoder[4], relu=True)

    def forward(self, x):
        return ops.act_to_nchw(self.forward_nhwc(ops.to_act(x)))
