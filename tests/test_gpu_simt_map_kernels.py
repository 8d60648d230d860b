"""The conversion, fp32 conv and map kernels against exact or float64 references, one or more cases per kernel instantiation.

heal_act_convert (k_act_convert, k_act_convert_scalar), heal_conv2d_simt (k_conv2d_dense, k_conv2d_grouped<4,4,4>, <8,8,4>,
<16,4,4>), heal_dwconv_layernorm (k_dwconv_ln), heal_mean_layernorm (k_mean_layernorm) and heal_maxpool3x3s2 (k_maxpool3s2).
Every reference is computed on the exact values the kernel read: hi + lo for split input, the bf16 value for bf16 input.  Every
other test of the library finds "what a kernel read" with ops.convert(a, "f32"), so heal_act_convert is checked against
host-side roundings that do not go through it.

Exact operations are checked bit for bit:
  convert   f32 -> bf16 is torch's round-to-nearest-even .to(torch.bfloat16); f32 -> split is ops.split_bf16 (hi = bf16(x),
            lo = bf16(x - hi)); split -> f32 is hi + lo; bf16 -> f32 and bf16 -> split are exact; split -> bf16 / split round
            hi + lo (an fp32 sum, exact: hi and lo span 16 bits) the same way.  All nine (src, dst) pairs, with +-0, fp32
            subnormals, bf16 halfway ties on even and odd mantissas and the largest values that still round to a finite bf16.
            The vector and scalar kernels give identical bits.
  maxpool   F.max_pool2d(x, 3, 2, 1) (-inf padding) of the read input, in both storage modes.

Rounded operations are checked against a first-order bound in the reference's own quantities; U = 2^-24 and REL = 2^-22 covers
the final fp32 roundings.
  conv      |err| <= ALPHA(K) (sum |w x| + |b| + |r|) + REL |y|, K = Cin/groups kh kw the products per output, w and b the packed
            fp32 weights and bias the kernel read (pc.weight, pc.bias: the bound measures the kernel, not the host BN fold), r the
            residual.  The kernel accumulates the K products with fp32 FMAs in one chain, adds the bias, the residual and
            applies the activation.  The rigorous bound of such a chain is K U (sum |w x| + |b| + |r|); the rounding errors of a
            chain over products of both signs do not add up like that, so ALPHA(K) = min(K, A0 sqrt(K)) U, never looser than
            K U.  ReLU is 1-Lipschitz; GELU multiplies the first term by max |GELU'| = 1.13 and adds 2^-22 |v| for erff and the
            products 0.5 v (1 + erf) (the pre-activation v; 1 + erf cancels for v < 0).
  dwconv+LN z_c the dwconv output with error E_c = ALPHA(k^2) (sum |w x| + |b|).  LayerNorm over the C channels of a pixel with
            fp32 sums (<= 8 serial adds per lane, then 5 shuffle levels: ASUM = 16 U of the sum of magnitudes):
              d_c = z_c - mean, error D_c = E_c + mean(E) + ASUM mean|z|
              var = mean d^2, error V = 2 mean(|d| D) + ASUM var
              y_c = d_c rstd g_c + b_c, rstd = (var + eps)^-1/2 (rsqrtf: 2 ulp)
              |err_c| <= |g_c| rstd (D_c + |d_c| (V / (2 (var + eps)) + 2^-20)) + REL |y_c|
            (2^-20 = 16 U: the subtraction, three products, rsqrtf's 2 ulp, the division by C and the + eps)
  mean+LN   the same with z the fp32 mean over n_avg images: E_c = (n_avg + 1) U mean_k |x_k| for n_avg > 1, 0 for n_avg = 1.

Every rounded case runs its kernel twice: with fp32 output (run A) and with the product's output format (run B).  B must be
bit for bit the rounding of A: bf16(A); for split, hi = bf16(A) and lo = bf16(A - hi).  The channels around input and output
slices (an `out=` view into a wider buffer, an odd out_coffset, deconv planes written into a concat slice) keep their sentinel.
test_bound_rejects_plausible_kernel_bugs (no GPU) restates each plausible kernel bug on the float64 reference of a shrunken case
and shows that the bound, or the exact comparison, rejects it.

Calibration, on an H100 80GB HBM3 at a 700 W power limit.  With ALPHA(K) = K U (the rigorous form) the largest conv
err / bound times sqrt(K) was 0.63 (g128_s1, K = 36), so A0 = 2.5 leaves 4x of headroom.  Largest err / bound per case at
A0 = 2.5:
  conv      bb_3x3_s1_res_split 0.066, bb_3x3_s2_64_128 0.063, bb_3x3_s1_res_f32_in_slice 0.039, bb_3x3_s1_res_bf16 0.046,
            ds_1x1_s2_odd_out 0.185, deconv_up1 0.132, deconv_up2 0.149, deconv_up4 0.103, head_cls2 0.057, head_reg14 0.071,
            head_dir4 0.048, g128_s1 0.228, g128_s2 0.222, g256_s1 0.130, g256_s2 0.140, g512_s1 0.105, g512_s2 0.117,
            compress_dec_cin4 0.179, convnext_pw1_gelu 0.135, convnext_pw2_res 0.113, pw1_gelu_split_res 0.143,
            misaligned_out_f32 0.061, misaligned_out_bf16 0.044
  dwconv+LN dw_c64_k7_split 0.046, dw_c128_k3_f32 0.064, dw_c192_k11_bf16 0.034, dw_c256_k1_split 0.089,
            dw_c64_k7_tiny_nobias 0.027, dw_c128_k7_small_var 0.058
  mean+LN   ml_c64_n1 0.083, ml_c128_n2 0.061, ml_c192_n5_out_view 0.052, ml_c256_n5 0.046, ml_empty 0 (no output)
The convert and maxpool cases are exact."""
import json
import math
import os
import re
import subprocess
import sys
import zlib
from dataclasses import dataclass
from typing import Optional, Tuple

import numpy as np
import pytest
import torch
import torch.nn.functional as F

U = 2.0 ** -24
# ALPHA(K) = min(K, A0 sqrt(K)) U.  Calibrated on an H100 80GB HBM3 at 700 W: with ALPHA(K) = K U the largest conv err / bound,
# times sqrt(K), was 0.63 (g128_s1, K = 36), so the kernel needs A0 >= 0.63; 2.5 leaves 4x of headroom.  test_kernel prints
# err / bound for every case.
A0 = 2.5
REL = 2.0 ** -22
ASUM = 16 * U
GELU_SLOPE = 1.13          # max |GELU'(v)| = 1.1289, at v = sqrt(2)
SENTINEL = -1000.0         # finite and exact in bf16: fills the channels around a slice


def alpha(K):
    return min(K, A0 * math.sqrt(K)) * U


# ------------------------------------------------------------------------------------------------ cases
@dataclass(frozen=True)
class Cvt:
    """heal_act_convert of an (N,H,W,C) map from format src to dst; slices are (buffer width, channel offset)."""
    name: str
    src: str
    dst: str
    shape: Tuple[int, int, int, int]
    reaches: Tuple[str, ...]
    src_slice: Optional[Tuple[int, int]] = None
    dst_slice: Optional[Tuple[int, int]] = None
    kernel = "convert"


@dataclass(frozen=True)
class Conv:
    """heal_conv2d_simt of one Conv2d (+BN) (+act) (+residual), or a ConvTranspose2d with kernel = stride = up (up > 0)."""
    name: str
    shape: Tuple[int, int, int]                   # N, H, W of the input
    cin: int
    cout: int
    k: int
    fin: str                                      # input storage format
    fout: str                                     # the product's output format (run B)
    reaches: Tuple[str, ...]
    stride: int = 1
    groups: int = 1
    up: int = 0                                   # ConvTranspose2d kernel = stride = up
    act: int = 1                                  # 0 none, 1 ReLU, 2 GELU (erf)
    bn: bool = True
    res: Optional[str] = None                     # residual storage format
    in_slice: Optional[Tuple[int, int]] = None    # (buffer width, channel offset), read through in_coffset
    out_slice: Optional[Tuple[int, int, bool]] = None   # (buffer width, channel offset, an `out=` view (True) or out_coffset)
    cin_to: Optional[int] = None                  # simt_cin4 packing: input channels zero-padded to cin_to
    kernel = "conv"

    @property
    def K(self):
        return self.cin_read // self.groups * (1 if self.up else self.k * self.k)

    @property
    def cin_read(self):
        return self.cin_to or self.cin


@dataclass(frozen=True)
class DwLn:
    name: str
    shape: Tuple[int, int, int]
    C: int
    k: int
    fin: str
    fout: str
    bias: bool = True
    small_var: bool = False                       # channels of the dwconv output nearly equal: var ~ 2e-8 << eps
    in_slice: Optional[Tuple[int, int]] = None
    reaches: Tuple[str, ...] = ("k_dwconv_ln",)
    kernel = "dwln"


@dataclass(frozen=True)
class MeanLn:
    name: str
    n_out: int
    n_avg: int
    HW: Tuple[int, int]
    C: int
    fin: str
    fout: str
    out_slice: Optional[Tuple[int, int]] = None   # an `out=` view into a wider buffer
    reaches: Tuple[str, ...] = ("k_mean_layernorm",)
    kernel = "meanln"


@dataclass(frozen=True)
class Pool:
    """heal_maxpool3x3s2 of a logical (N,H,W,C) map; d2s: stored depth-to-space folded as (N,H/2,W/2,4C)."""
    name: str
    shape: Tuple[int, int, int, int]
    fin: str
    fout: str
    d2s: bool = False
    negative: bool = False                        # every input value < 0: zero padding would show at every border output
    in_slice: Optional[Tuple[int, int]] = None
    reaches: Tuple[str, ...] = ("k_maxpool3s2",)
    kernel = "pool"


VEC, SCAL, DENSE = ("k_act_convert",), ("k_act_convert_scalar",), ("k_conv2d_dense",)
G4, G8, G16 = ("k_conv2d_grouped<4,4,4>",), ("k_conv2d_grouped<8,8,4>",), ("k_conv2d_grouped<16,4,4>",)
FMTS = ("f32", "bf16", "split")

CASES = [
    # ---- heal_act_convert: the nine format pairs on 4-aligned views, with the special values in the first pixels
    *[Cvt(f"cvt_{s}_{d}", s, d, (2, 7, 9, 64), VEC) for s in FMTS for d in FMTS],
    Cvt("cvt_c1", "f32", "split", (2, 5, 7, 1), SCAL),
    Cvt("cvt_c3", "split", "bf16", (1, 9, 11, 3), SCAL),
    Cvt("cvt_c4", "bf16", "f32", (3, 5, 7, 4), VEC),
    Cvt("cvt_odd_src", "f32", "split", (2, 5, 9, 64), SCAL, src_slice=(70, 3)),
    Cvt("cvt_odd_dst", "split", "f32", (1, 6, 7, 64), SCAL, dst_slice=(69, 5)),
    Cvt("cvt_slices4", "bf16", "split", (2, 5, 6, 32), VEC, src_slice=(40, 4), dst_slice=(48, 8)),
    # 655360 quads and 607500 elements: past the 132 x 16 blocks of 256 threads, so the grid-stride loops turn
    Cvt("cvt_grid_stride_vec", "f32", "split", (1, 160, 256, 64), VEC),
    Cvt("cvt_grid_stride_scalar", "split", "f32", (1, 450, 450, 3), SCAL),
    Cvt("cvt_empty", "f32", "split", (0, 5, 7, 64), ()),
    # views at channel 2 of a wider buffer (an 8-byte aligned fp32 / 4-byte aligned bf16 data pointer): not refused, the
    # scalar kernel
    Cvt("cvt_misaligned_f32_src", "f32", "split", (2, 5, 7, 64), SCAL, src_slice=(68, 2)),
    Cvt("cvt_misaligned_bf16_src", "bf16", "f32", (2, 5, 7, 64), SCAL, src_slice=(68, 2)),
    Cvt("cvt_misaligned_f32_dst", "split", "f32", (2, 5, 7, 64), SCAL, dst_slice=(68, 2)),
    Cvt("cvt_misaligned_bf16_dst", "f32", "bf16", (2, 5, 7, 64), SCAL, dst_slice=(68, 2)),
    # ---- heal_conv2d_simt: the convs the fp32 mode runs on this kernel.  PointPillars backbone 3x3 (BasicBlock with its
    # residual; 2 x 25 x 37 = 1850 output pixels, not a multiple of 128)
    Conv("bb_3x3_s1_res_split", (2, 25, 37), 64, 64, 3, "split", "split", DENSE, res="split"),
    Conv("bb_3x3_s2_64_128", (3, 25, 37), 64, 128, 3, "bf16", "bf16", DENSE, stride=2),
    Conv("bb_3x3_s1_res_f32_in_slice", (1, 13, 19), 128, 128, 3, "f32", "f32", DENSE, res="f32", in_slice=(192, 64),
         out_slice=(160, 32, True)),
    Conv("bb_3x3_s1_res_bf16", (1, 9, 13), 64, 64, 3, "bf16", "split", DENSE, res="bf16"),
    # 1x1 stride-2 downsample, N = 5, into an odd channel offset (the one-channel store branch)
    Conv("ds_1x1_s2_odd_out", (5, 17, 23), 64, 128, 1, "f32", "split", DENSE, stride=2, act=0, out_slice=(133, 3, False)),
    # deconvs (ConvTranspose2d kernel = stride) into channels [128, 256) of the 384-channel concat
    Conv("deconv_up1", (2, 16, 24), 128, 128, 1, "split", "split", DENSE, up=1, out_slice=(384, 128, False)),
    Conv("deconv_up2", (2, 8, 12), 128, 128, 2, "bf16", "bf16", DENSE, up=2, out_slice=(384, 128, False)),
    Conv("deconv_up4", (1, 4, 6), 256, 128, 4, "f32", "f32", DENSE, up=4, out_slice=(384, 128, False)),
    # heads: 1x1 with Cout 2 and 14 (tails of 2 channels) and 4, fp32 out
    Conv("head_cls2", (2, 13, 19), 384, 2, 1, "split", "f32", DENSE, act=0, bn=False),
    Conv("head_reg14", (2, 13, 19), 384, 14, 1, "bf16", "f32", DENSE, act=0, bn=False),
    Conv("head_dir4", (1, 13, 19), 384, 4, 1, "f32", "f32", DENSE, act=0, bn=False),
    # ResNeXt grouped 3x3, 32 groups, stride 1 and 2, every Wo with a partial last 4-pixel tile
    Conv("g128_s1", (2, 11, 21), 128, 128, 3, "split", "split", G4, groups=32),
    Conv("g128_s2", (1, 21, 29), 128, 128, 3, "f32", "f32", G4, stride=2, groups=32),
    Conv("g256_s1", (1, 9, 14), 256, 256, 3, "bf16", "bf16", G8, groups=32),
    Conv("g256_s2", (2, 13, 19), 256, 256, 3, "split", "split", G8, stride=2, groups=32),
    Conv("g512_s1", (1, 7, 10), 512, 512, 3, "split", "split", G16, groups=32),
    Conv("g512_s2", (1, 11, 13), 512, 512, 3, "f32", "bf16", G16, stride=2, groups=32),
    # the compressor decoder in fp32 mode: 2 channels zero-padded to 4 (simt_cin4)
    Conv("compress_dec_cin4", (2, 16, 24), 2, 64, 3, "f32", "f32", DENSE, cin_to=4),
    # the ConvNeXt aligner's Linear layers in fp32 mode: 64 -> 256 + GELU, 256 -> 64 + the block's residual
    Conv("convnext_pw1_gelu", (2, 19, 23), 64, 256, 1, "f32", "f32", DENSE, act=2, bn=False),
    Conv("convnext_pw2_res", (2, 19, 23), 256, 64, 1, "f32", "f32", DENSE, act=0, bn=False, res="f32"),
    Conv("pw1_gelu_split_res", (1, 11, 13), 64, 128, 1, "split", "bf16", DENSE, act=2, bn=False, res="split"),
    # an `out=` view at channel 2 of a wider buffer: not refused, the dense conv stores it one channel at a time
    Conv("misaligned_out_f32", (1, 9, 13), 64, 64, 3, "f32", "f32", DENSE, out_slice=(68, 2, True)),
    Conv("misaligned_out_bf16", (1, 9, 13), 64, 64, 3, "split", "bf16", DENSE, out_slice=(68, 2, True)),
    # ---- heal_dwconv_layernorm
    DwLn("dw_c64_k7_split", (2, 19, 23), 64, 7, "split", "split", in_slice=(128, 64)),
    DwLn("dw_c128_k3_f32", (1, 13, 21), 128, 3, "f32", "bf16"),
    DwLn("dw_c192_k11_bf16", (1, 15, 17), 192, 11, "bf16", "f32"),
    DwLn("dw_c256_k1_split", (2, 9, 11), 256, 1, "split", "bf16"),
    DwLn("dw_c64_k7_tiny_nobias", (2, 2, 3), 64, 7, "f32", "split", bias=False),
    DwLn("dw_c128_k7_small_var", (1, 10, 13), 128, 7, "split", "split", small_var=True),
    # ---- heal_mean_layernorm
    MeanLn("ml_c64_n1", 3, 1, (5, 7), 64, "f32", "bf16"),
    MeanLn("ml_c128_n2", 2, 2, (6, 9), 128, "split", "split"),
    MeanLn("ml_c192_n5_out_view", 1, 5, (7, 5), 192, "bf16", "f32", out_slice=(320, 64)),
    MeanLn("ml_c256_n5", 2, 5, (3, 4), 256, "split", "split", out_slice=(264, 4)),
    MeanLn("ml_empty", 0, 2, (3, 4), 64, "f32", "f32", reaches=()),
    # ---- heal_maxpool3x3s2
    Pool("mp_f32_odd", (2, 37, 51, 64), "f32", "f32"),
    Pool("mp_bf16_odd_negative", (1, 21, 17, 32), "bf16", "bf16", negative=True),
    Pool("mp_split_slice", (2, 16, 22, 64), "split", "split", in_slice=(96, 32)),
    Pool("mp_d2s_c64_2x2", (3, 2, 2, 64), "f32", "f32", d2s=True),
    Pool("mp_d2s_c64_bf16_negative", (2, 40, 56, 64), "bf16", "bf16", d2s=True, negative=True),
    Pool("mp_d2s_c64_split", (1, 14, 18, 64), "split", "split", d2s=True),
    Pool("mp_d2s_c4_2x2", (2, 2, 2, 4), "split", "split", d2s=True),
    Pool("mp_d2s_c4_f32", (1, 6, 10, 4), "f32", "bf16", d2s=True),
]
CASE = {c.name: c for c in CASES}
assert len(CASE) == len(CASES)

REACHABLE = {"k_act_convert", "k_act_convert_scalar", "k_conv2d_dense", "k_conv2d_grouped<4,4,4>", "k_conv2d_grouped<8,8,4>",
             "k_conv2d_grouped<16,4,4>", "k_dwconv_ln", "k_mean_layernorm", "k_maxpool3s2"}


def _launches(case):
    """Library launches of one case (a convert case is one call, the others runs A and B)."""
    if not case.reaches:
        return 0
    if case.kernel == "convert":
        return 1
    if case.kernel == "conv" and case.up:
        return 2 * case.up * case.up
    return 2


def test_case_table():
    """Every case names instantiations the launchers can dispatch to, the cases together name all of them, and the shapes
    the issue of each kernel calls for are present."""
    named = set()
    for c in CASES:
        assert set(c.reaches) <= REACHABLE, c.name
        named |= set(c.reaches)
    assert named == REACHABLE
    cvt = [c for c in CASES if c.kernel == "convert"]
    assert {(c.src, c.dst) for c in cvt} == {(s, d) for s in FMTS for d in FMTS}
    assert {1, 3, 4, 64} <= {c.shape[3] for c in cvt}
    assert any(c.shape[0] == 0 for c in cvt)
    cap = 132 * 16 * 256
    assert any(c.reaches == VEC and math.prod(c.shape) // 4 > cap for c in cvt)
    assert any(c.reaches == SCAL and math.prod(c.shape) > cap for c in cvt)
    conv = [c for c in CASES if c.kernel == "conv"]
    assert {c.fin for c in conv} == set(FMTS) and {c.res for c in conv} >= set(FMTS) and {c.fout for c in conv} == set(FMTS)
    assert {c.up for c in conv} >= {1, 2, 4} and any(c.cout % 4 for c in conv) and any(c.act == 2 for c in conv)
    assert {(c.cin, c.stride) for c in conv if c.groups > 1} == {(w, s) for w in (128, 256, 512) for s in (1, 2)}
    for c in conv:
        if c.groups > 1:
            Wo = (c.shape[2] - 1) // c.stride + 1
            assert Wo % 4, f"{c.name}: no partial 4-pixel tile"
    assert any(c.shape[0] * ((c.shape[1] - 1) // c.stride + 1) * ((c.shape[2] - 1) // c.stride + 1) % 128 for c in conv)
    dw = [c for c in CASES if c.kernel == "dwln"]
    assert {c.C for c in dw} == {64, 128, 192, 256} and {c.k for c in dw} == {1, 3, 7, 11}
    assert {c.fin for c in dw} == set(FMTS) and {c.fout for c in dw} == set(FMTS)
    assert any(c.fin == c.fout == "split" and (c.C, c.k) == (64, 7) for c in dw)
    ml = [c for c in CASES if c.kernel == "meanln"]
    assert {c.C for c in ml} == {64, 128, 192, 256} and {c.n_avg for c in ml} >= {1, 2, 5} and any(c.n_out == 0 for c in ml)
    pool = [c for c in CASES if c.kernel == "pool"]
    for d2s in (False, True):
        assert {c.fin for c in pool if c.d2s == d2s} == set(FMTS)
    assert {c.shape[3] for c in pool if c.d2s and c.shape[1:3] == (2, 2)} == {4, 64}


# ------------------------------------------------------------------------------------------------ inputs
def _gen(name, what=""):
    return torch.Generator().manual_seed(zlib.crc32(f"{name}/{what}".encode()))


# fp32 bit patterns: +-0, subnormals (a bf16 tie below the smallest normal, on an even and an odd bf16 mantissa), the largest
# subnormal (rounds up to the smallest normal), bf16 ties around 1 (even: down, odd: up) and either side of them, bf16 max,
# and the largest fp32 values that still round to a finite bf16
SPECIAL_BITS = [0x00000000, 0x80000000, 0x00000001, 0x80000001, 0x00008000, 0x00018000, 0x807FFFFF, 0x007FFFFF, 0x00800000,
                0x3F808000, 0x3F818000, 0xBF808000, 0xBF818000, 0x3F807FFF, 0x3F808001, 0x7F7F0000, 0xFF7F0000,
                0x7F7F7FFF, 0xFF7F7FFF, 0x7F7E8000, 0x00400000, 0x80408000]


def _specials():
    return torch.tensor(np.array(SPECIAL_BITS, dtype=np.uint32).view(np.int32)).view(torch.float32)


def _cvt_input(case):
    N, H, W, C = case.shape
    x = torch.randn(N, H, W, C, generator=_gen(case.name)) * 3
    flat = x.reshape(-1)
    sp = _specials()
    n = min(len(sp), flat.numel())
    flat[:n] = sp[:n]
    return x


def _store(x32, fmt):
    """fp32 (N,H,W,C) -> the storage tensor: fp32 as is, bf16 (1,N,H,W,C), split (2,N,H,W,C) = hi, lo."""
    if fmt == "f32":
        return x32.clone()
    hi = x32.to(torch.bfloat16)
    if fmt == "bf16":
        return hi[None].clone()
    return torch.stack([hi, (x32 - hi.float()).to(torch.bfloat16)])


def _value(st, fmt, drop_lo=False):
    """The value a kernel reads from a storage tensor, in float64 (N,H,W,C); drop_lo: the hi plane alone."""
    if fmt == "f32":
        return st.double()
    return st[0].double() if drop_lo else st.double().sum(0)


def _f32_value(st, fmt):
    """The fp32 value heal_act_convert reads: hi + lo as one fp32 sum for split."""
    if fmt == "f32":
        return st.clone()
    return st[0].float() if fmt == "bf16" else st[0].float() + st[1].float()


def _bits(t):
    t = t.contiguous()
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


def _rne(v32, fmt, truncate=False):
    """fp32 -> storage tensor in fmt, with RNE rounding (torch) or, for the sharpness test, truncation."""
    if truncate:
        hi = (v32.view(torch.int32) & -65536).view(torch.float32).to(torch.bfloat16)
        return hi[None] if fmt == "bf16" else torch.stack([hi, (v32 - hi.float()).to(torch.bfloat16)])
    if fmt == "f32":
        return v32.clone()
    from heal_b200 import ops
    return ops.split_bf16(v32, 1 if fmt == "bf16" else 2)


# ------------------------------------------------------------------------------------------------ conv: modules and reference
def _conv_modules(case):
    g = _gen(case.name, "modules")
    if case.up:
        conv = torch.nn.ConvTranspose2d(case.cin, case.cout, case.up, stride=case.up)
    else:
        conv = torch.nn.Conv2d(case.cin, case.cout, case.k, stride=case.stride, padding=case.k // 2, groups=case.groups)
    bn = torch.nn.BatchNorm2d(case.cout, eps=1e-3).eval() if case.bn else None
    with torch.no_grad():
        conv.weight.copy_(torch.randn(conv.weight.shape, generator=g) * (1.0 / case.K) ** 0.5)
        # GELU: biases spread widely, so that pre-activations reach the region where erf and tanh forms differ most
        conv.bias.copy_(torch.randn(case.cout, generator=g) * (1.5 if case.act == 2 else 0.1))
        if bn is not None:
            bn.weight.copy_(torch.rand(case.cout, generator=g) + 0.5)
            bn.bias.copy_(torch.randn(case.cout, generator=g) * 0.1)
            bn.running_mean.copy_(torch.randn(case.cout, generator=g) * 0.1)
            bn.running_var.copy_(torch.rand(case.cout, generator=g) + 0.5)
    return conv, bn


def _packed(case):
    from heal_b200 import ops
    conv, bn = _conv_modules(case)
    if case.up:
        return ops.pack_deconv(conv, bn, case.act == 1)
    pc = ops.pack_conv(conv, bn, case.act == 1, cin_to=case.cin_to)
    pc.relu = case.act
    return pc


def _conv_out_hw(case, H, W):
    if case.up:
        return H * case.up, W * case.up
    return (H + 2 * (case.k // 2) - case.k) // case.stride + 1, (W + 2 * (case.k // 2) - case.k) // case.stride + 1


def _conv_inputs(case, H=None, W=None):
    N = case.shape[0]
    H, W = H or case.shape[1], W or case.shape[2]
    g = _gen(case.name, "inputs")
    x = torch.randn(N, H, W, case.cin_read, generator=g)
    if case.cin_to:
        x[..., case.cin:] = 0          # the product's zero-filled channel pad
    Ho, Wo = _conv_out_hw(case, H, W)
    r = torch.randn(N, Ho, Wo, case.cout, generator=g) if case.res else None
    return x, r


def _conv_weight(case, pc):
    """The packed fp32 weights the kernel reads as a float64 torch weight: (Cout, Cin/g, k, k), (Cin, Cout, up, up) deconv."""
    wp = pc.weight.double().cpu()
    if case.up:
        return wp[..., :case.cout].permute(2, 3, 0, 1)
    if case.groups > 1:
        cg = case.cin // case.groups
        return wp.reshape(3, 3, cg, cg, case.groups).permute(4, 3, 2, 0, 1).reshape(case.cout, cg, 3, 3)
    return wp[..., :case.cout].permute(3, 2, 0, 1)


def _conv_reference(case, pc, x, r, fault=None):
    """float64 (N,Ho',Wo',Cout) output and bound.  x, r: float64 NHWC values the kernel read.  `fault` restates a plausible
    kernel bug (test_bound_rejects_plausible_kernel_bugs)."""
    w = _conv_weight(case, pc)
    b = pc.bias.double().cpu()
    if fault == "tail_bias":
        b = b.clone()
        b[case.cout // 4 * 4:] = 0
    xn = x.permute(0, 3, 1, 2)
    if fault == "border_tap":           # every tap that reads the last input column dropped (an off-by-one bounds check)
        xn = xn.clone()
        xn[..., -1] = 0
    if case.up:
        conv = lambda t, ww: F.conv_transpose2d(t, ww, stride=case.up)
    elif fault == "pad_side":           # the two pad columns / rows all on the bottom-right
        p = case.k // 2
        conv = lambda t, ww: F.conv2d(F.pad(t, (0, 2 * p, 0, 2 * p)), ww, stride=case.stride, groups=case.groups)
    else:
        conv = lambda t, ww: F.conv2d(t, ww, stride=case.stride, padding=case.k // 2, groups=case.groups)
    v = conv(xn, w).permute(0, 2, 3, 1) + b
    S = conv(xn.abs(), w.abs()).permute(0, 2, 3, 1) + b.abs()
    if fault == "up_swap" and case.up:
        N, Hs, Ws, C = v.shape
        k = case.up
        v = v.reshape(N, Hs // k, k, Ws // k, k, C).permute(0, 1, 4, 3, 2, 5).reshape(N, Hs, Ws, C)
    if r is not None:
        if fault == "relu_before_res":
            v = torch.relu(v) + r
        else:
            v = v + r
        S = S + r.abs()
    first = alpha(case.K) * S
    if case.act == 1 and fault != "relu_before_res":
        y = torch.relu(v)
    elif case.act == 2:
        y = F.gelu(v, approximate="tanh" if fault == "gelu_tanh" else "none")
        first = GELU_SLOPE * first + 2.0 ** -22 * v.abs()
    else:
        y = v
    return y, first + REL * y.abs()


# ------------------------------------------------------------------------------------------------ LayerNorm references
def _ln(z, E, lw, lb, eps, fault=None):
    """LayerNorm over the last dim of float64 z (fp32-computed with per-element error bound E) and the docstring's bound."""
    C = z.shape[-1]
    mu = z.mean(-1, keepdim=True)
    d = z - mu
    var = (d * d).mean(-1, keepdim=True)
    var_k = var * C / (C - 1) if fault == "unbiased" else var
    rstd = 1 / torch.sqrt(var_k + (0.0 if fault == "eps" else eps))
    y = d * rstd * lw + lb
    D = E + E.mean(-1, keepdim=True) + ASUM * z.abs().mean(-1, keepdim=True)
    V = 2 * (d.abs() * D).mean(-1, keepdim=True) + ASUM * var
    r0 = 1 / torch.sqrt(var + eps)
    bound = lw.abs() * r0 * (D + d.abs() * (V / (2 * (var + eps)) + 2.0 ** -20)) + REL * y.abs()
    return y, bound


def _dw_params(case):
    g = _gen(case.name, "params")
    C, k = case.C, case.k
    if case.small_var:
        w = torch.full((k * k, C), 1.0 / (k * k)) + torch.randn(k * k, C, generator=g) * 1e-5
    else:
        w = torch.randn(k * k, C, generator=g) * (0.6 / k)
    b = torch.randn(C, generator=g) * 0.1 if case.bias and not case.small_var else (torch.zeros(C) if case.bias else None)
    lw, lb = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g) * 0.1
    return w, b, lw, lb


def _dw_input(case, H=None, W=None):
    N = case.shape[0]
    H, W = H or case.shape[1], W or case.shape[2]
    g = _gen(case.name, "inputs")
    if case.small_var:
        # one value per pixel for every channel plus 1e-3 noise, and near-uniform weights: the channel variance of the dwconv
        # output is ~2e-8, well below eps = 1e-6
        return torch.randn(N, H, W, 1, generator=g) + torch.randn(N, H, W, case.C, generator=g) * 1e-3
    return torch.randn(N, H, W, case.C, generator=g) * 2 + 0.5


EPS = 1e-6


def _dw_reference(case, x, w, b, lw, lb, fault=None):
    C, k = case.C, case.k
    wc = w.double().t().reshape(C, 1, k, k)
    xn = x.permute(0, 3, 1, 2)
    if fault == "border_tap":
        xn = xn.clone()
        xn[..., -1] = 0
    bd = b.double() if b is not None else torch.zeros(C, dtype=torch.float64)
    z = F.conv2d(xn, wc, padding=k // 2, groups=C).permute(0, 2, 3, 1) + bd
    S = F.conv2d(xn.abs(), wc.abs(), padding=k // 2, groups=C).permute(0, 2, 3, 1) + bd.abs()
    return _ln(z, alpha(k * k) * S, lw.double(), lb.double(), EPS, fault)


def _ml_params(case):
    g = _gen(case.name, "params")
    return torch.rand(case.C, generator=g) + 0.5, torch.randn(case.C, generator=g) * 0.1


def _ml_input(case, HW=None):
    H, W = HW or case.HW
    return torch.randn(case.n_out * case.n_avg, H, W, case.C, generator=_gen(case.name, "inputs")) * 3 + 1


def _ml_reference(case, x, lw, lb, fault=None):
    n, H, W, C = x.shape
    xs = x.reshape(case.n_out, case.n_avg, H, W, C)
    z = xs[:, :-1].mean(1) if fault == "n_minus_1" else xs.sum(1) / case.n_avg
    E = (case.n_avg + 1) * U * xs.abs().mean(1) if case.n_avg > 1 else torch.zeros_like(z)
    return _ln(z, E, lw.double(), lb.double(), 1e-5, fault)


# ------------------------------------------------------------------------------------------------ max pooling reference
def _pool_input(case, H=None, W=None):
    N, H0, W0, C = case.shape
    H, W = H or H0, W or W0
    x = torch.randn(N, H, W, C, generator=_gen(case.name, "inputs"))
    if case.negative:
        x = -(x.abs() + 0.25)
    if case.d2s:      # the stored (N,H/2,W/2,4C) tensor, channel block (y & 1) * 2 + (x & 1)
        x = x.reshape(N, H // 2, 2, W // 2, 2, C).permute(0, 1, 3, 2, 4, 5).reshape(N, H // 2, W // 2, 4 * C)
    return x


def _pool_reference(case, v, fault=None):
    """F.max_pool2d(x, 3, 2, 1) of the logical map of the read values v (float64 stored NHWC)."""
    if case.d2s:
        N, h, w, C4 = v.shape
        C = C4 // 4
        t = v.reshape(N, h, w, 2, 2, C)          # (.., y & 1, x & 1, c)
        if fault == "d2s_phase":
            t = t.transpose(3, 4)
        v = t.permute(0, 1, 3, 2, 4, 5).reshape(N, 2 * h, 2 * w, C)
    xn = v.permute(0, 3, 1, 2)
    if fault == "pad_zero":
        y = F.max_pool2d(F.pad(xn, (1, 1, 1, 1)), 3, 2, 0)
    else:
        y = F.max_pool2d(xn, 3, 2, 1)
    return y.permute(0, 2, 3, 1)


# ------------------------------------------------------------------------------------------------ the bound is sharp (CPU)
def _faults(case):
    k = case.kernel
    f = []
    if not case.reaches:           # an empty map
        return f
    if k == "convert":
        if case.src == "f32" and case.dst != "f32":
            f.append("truncate")
        return f
    if case.fin == "split":
        f.append("lo")
    if k == "conv":
        if case.k > 1 and not case.up:
            f.append("border_tap")
        if case.stride == 2 and case.k > 1:
            f.append("pad_side")
        if case.up > 1:
            f.append("up_swap")
        if case.res and case.act == 1:
            f.append("relu_before_res")
        if case.act == 2:
            f.append("gelu_tanh")
        if case.cout % 4:
            f.append("tail_bias")
    elif k == "dwln":
        # (with var << eps the variance's C / (C - 1) moves nothing the bound can see)
        f += (["eps"] if case.small_var else ["unbiased"]) + (["border_tap"] if case.k > 1 else [])
    elif k == "meanln":
        f += ["unbiased"] + (["n_minus_1"] if case.n_avg > 1 else [])
    elif k == "pool":
        if case.negative:
            f.append("pad_zero")
        if case.d2s and case.shape[1] > 2:      # a 2x2 map pools all four phases into its one output
            f.append("d2s_phase")
    return f


def _shrunk(case):
    if case.kernel == "conv":
        N, H, W = case.shape
        return min(H, 9), min(W, 11)
    if case.kernel == "dwln":
        return min(case.shape[1], 9), min(case.shape[2], 11)
    if case.kernel == "pool":
        return min(case.shape[1], 10), min(case.shape[2], 12)
    return None


def _cpu_reference(case, fault=None, drop_lo=False):
    """(y, bound) of a shrunken case on the CPU, the input read as stored (or its hi plane alone)."""
    H, W = _shrunk(case) or (None, None)
    if case.kernel == "conv":
        pc = _packed(case)
        x, r = _conv_inputs(case, H, W)
        xv = _value(_store(x, case.fin), case.fin, drop_lo)
        rv = _value(_store(r, case.res), case.res) if r is not None else None
        return _conv_reference(case, pc, xv, rv, fault)
    if case.kernel == "dwln":
        w, b, lw, lb = _dw_params(case)
        xv = _value(_store(_dw_input(case, H, W), case.fin), case.fin, drop_lo)
        return _dw_reference(case, xv, w, b, lw, lb, fault)
    if case.kernel == "meanln":
        lw, lb = _ml_params(case)
        xv = _value(_store(_ml_input(case), case.fin), case.fin, drop_lo)
        return _ml_reference(case, xv, lw, lb, fault)
    xv = _value(_store(_pool_input(case, H, W), case.fin), case.fin, drop_lo)
    y = _pool_reference(case, xv, fault)
    return y, torch.zeros_like(y)


@pytest.mark.parametrize("name", [c.name for c in CASES if _faults(c)])
def test_bound_rejects_plausible_kernel_bugs(name):
    """Each plausible kernel bug, restated on the float64 reference of a shrunken case, leaves the bound (or, for the exact
    kernels, differs) on some element: the lo plane of split input dropped, truncation instead of RNE bf16 rounding, the taps
    that read the last input column dropped, both pad rows / columns of a stride-2 conv on the bottom-right, the deconv's
    up_i / up_j swapped, ReLU applied before the residual, the tanh-approximate GELU, the bias missing on the Cout tail quad,
    the unbiased variance, eps dropped, the mean over the first n_avg - 1 images only, max-pool padding treated as 0, and the depth-to-space
    phase read as (x & 1) * 2 + (y & 1)."""
    case = CASE[name]
    for fault in _faults(case):
        if case.kernel == "convert":
            x = _cvt_input(case)
            st = _store(x, case.src)
            v32 = _f32_value(st, case.src)
            good, bad = _rne(v32, case.dst), _rne(v32, case.dst, truncate=True)
            assert not torch.equal(_bits(good), _bits(bad)), f"{name}: truncation gives the same bits"
            continue
        y, bound = _cpu_reference(case)
        assert bool(torch.isfinite(y).all())
        if fault == "lo":
            yf = _cpu_reference(case, drop_lo=True)[0]
        else:
            yf = _cpu_reference(case, fault)[0]
        assert yf.shape == y.shape, f"{name}: '{fault}' changes the output shape"
        d = (yf - y).abs()
        ratio = torch.where(d == 0, 0.0, d / bound).max().item()
        assert ratio > 1, f"{name}: the bound does not reject '{fault}' (max err / bound {ratio:.3f})"


def test_alpha_never_looser_than_rigorous():
    for K in (1, 4, 9, 36, 49, 121, 384, 576, 1152, 2304, 4608):
        assert alpha(K) <= K * U


# ------------------------------------------------------------------------------------------------ the kernels (GPU)
def _put(st, fmt, sl):
    """A CUDA buffer holding storage tensor `st` in channels [coff, coff + C) and SENTINEL elsewhere (lo plane 0), and the
    Act over the slice."""
    from heal_b200 import ops
    width, coff = sl or (st.shape[-1], 0)
    buf = torch.full(st.shape[:-1] + (width,), SENTINEL, dtype=st.dtype)
    if fmt == "split":
        buf[1] = 0
    buf[..., coff:coff + st.shape[-1]] = st
    buf = buf.cuda()
    return buf, ops.Act(buf[..., coff:coff + st.shape[-1]], fmt)


def _out_buffer(N, H, W, width, fmt, sliced):
    fill = SENTINEL if sliced else float("nan")
    if fmt == "f32":
        return torch.full((N, H, W, width), fill, dtype=torch.float32, device="cuda")
    buf = torch.full((2 if fmt == "split" else 1, N, H, W, width), fill, dtype=torch.bfloat16, device="cuda")
    if fmt == "split" and sliced:
        buf[1] = 0
    return buf


def _read_back(buf, fmt, sl, C, name, what):
    """float64 values of channels [coff, coff + C) of a CUDA buffer; asserts the channels around them kept their sentinel."""
    b = buf.cpu()
    width, coff = sl or (b.shape[-1], 0)
    if width != C:
        whole = b.double() if fmt == "f32" else b[0].double()
        around = torch.cat([whole[..., :coff].flatten(), whole[..., coff + C:].flatten()])
        assert bool((around == SENTINEL).all()), f"{name}: the {what} buffer around the slice changed"
        if fmt == "split":
            lo = torch.cat([b[1][..., :coff].flatten(), b[1][..., coff + C:].flatten()])
            assert bool((lo == 0).all()), f"{name}: a lo-plane write spilled out of the {what} slice"
    return b[..., coff:coff + C]


def _launch(case):
    """Runs the case's launches.  Returns what the checks need (inputs as stored, CUDA buffers, outputs)."""
    from heal_b200 import ops
    k = case.kernel
    if k == "convert":
        x = _cvt_input(case)
        st = _store(x, case.src)
        sbuf, sact = _put(st, case.src, case.src_slice)
        N, H, W, C = case.shape
        dbuf = _out_buffer(N, H, W, (case.dst_slice or (C, 0))[0], case.dst, case.dst_slice is not None)
        coff = (case.dst_slice or (C, 0))[1]
        ops.convert(sact, case.dst, out=ops.Act(dbuf[..., coff:coff + C], case.dst))
        return dict(st=st, sbuf=sbuf, dbuf=dbuf)
    if k == "conv":
        pc = _packed(case).to("cuda")
        x, r = _conv_inputs(case)
        N, H, W = case.shape
        xst = _store(x, case.fin)
        xbuf, _ = _put(xst, case.fin, case.in_slice)
        xact = ops.Act(xbuf, case.fin)
        icoff = case.in_slice[1] if case.in_slice else 0
        rst = _store(r, case.res) if r is not None else None
        ract = ops.Act(rst.cuda(), case.res) if r is not None else None
        Ho, Wo = _conv_out_hw(case, H, W)
        width, oco, as_view = case.out_slice or (case.cout, 0, False)
        outs = {}
        for run, fmt in (("A", "f32"), ("B", case.fout)):
            buf = _out_buffer(N, Ho, Wo, width, fmt, case.out_slice is not None)
            if as_view:
                ops.conv2d_simt(xact, pc, residual=ract, out=ops.Act(buf[..., oco:oco + case.cout], fmt), in_coffset=icoff,
                                cin=case.cin_read)
            else:
                ops.conv2d_simt(xact, pc, residual=ract, out=ops.Act(buf, fmt), out_coffset=oco, in_coffset=icoff,
                                cin=case.cin_read)
            outs[run] = buf
        return dict(pc=pc, xst=xst, xbuf=xbuf, rst=rst, outs=outs)
    if k == "dwln":
        w, b, lw, lb = _dw_params(case)
        xst = _store(_dw_input(case), case.fin)
        xbuf, xact = _put(xst, case.fin, case.in_slice)
        outs = {}
        for run, fmt in (("A", "f32"), ("B", case.fout)):
            outs[run] = ops.dwconv_layernorm(xact, w.cuda(), b.cuda() if b is not None else None, case.k, lw.cuda(), lb.cuda(),
                                             EPS, out_fmt=fmt).t
        return dict(xst=xst, xbuf=xbuf, outs=outs, params=(w, b, lw, lb))
    if k == "meanln":
        lw, lb = _ml_params(case)
        xst = _store(_ml_input(case), case.fin)
        xbuf, xact = _put(xst, case.fin, None)
        H, W = case.HW
        width, oco = case.out_slice or (case.C, 0)
        outs = {}
        for run, fmt in (("A", "f32"), ("B", case.fout)):
            buf = _out_buffer(case.n_out, H, W, width, fmt, case.out_slice is not None)
            ops.mean_layernorm(xact, case.n_avg, lw.cuda(), lb.cuda(), 1e-5, out=ops.Act(buf[..., oco:oco + case.C], fmt))
            outs[run] = buf
        return dict(xst=xst, xbuf=xbuf, outs=outs, params=(lw, lb))
    xst = _store(_pool_input(case), case.fin)
    xbuf, xact = _put(xst, case.fin, case.in_slice)
    outs = {}
    for run, fmt in (("A", "f32"), ("B", case.fout)):
        outs[run] = ops.maxpool3x3s2(xact, out_fmt=fmt, depth_to_space_in=case.d2s).t
    return dict(xst=xst, xbuf=xbuf, outs=outs)


def _check_rounding(name, a, b, fmt):
    """Run B (storage tensor in fmt) is bit for bit the rounding of run A (fp32)."""
    if fmt == "f32":
        assert torch.equal(_bits(b), _bits(a)), f"{name}: the two fp32 runs differ"
        return
    hi = a.to(torch.bfloat16)
    assert torch.equal(_bits(b[0]), _bits(hi)), f"{name}: hi plane != bf16(fp32 output)"
    if fmt == "split":
        assert torch.equal(_bits(b[1]), _bits((a - hi.float()).to(torch.bfloat16))), f"{name}: lo plane != bf16(fp32 - hi)"


def _check_bound(name, got, y, bound):
    err = (got.double() - y).abs()
    ok = err <= bound
    ratio = torch.where(err == 0, 0.0, err / bound).max().item() if err.numel() else 0.0
    print(f"{name}: max err / bound {ratio:.4f}  (max err {err.max().item() if err.numel() else 0:.3e})")
    assert bool(ok.all()), f"{name}: {int((~ok).sum())} elements outside the bound, max err / bound {ratio:.3f}"
    return ratio


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASE))
def test_kernel(name):
    from heal_b200._lib import lib
    case = CASE[name]
    torch.cuda.synchronize()
    before = lib.heal_launch_count()
    r = _launch(case)
    torch.cuda.synchronize()
    assert lib.heal_launch_count() - before == _launches(case), f"{name}: launch count"
    k = case.kernel
    if k == "convert":
        N, H, W, C = case.shape
        _read_back(r["sbuf"], case.src, case.src_slice, C, name, "input")
        got = _read_back(r["dbuf"], case.dst, case.dst_slice, C, name, "output")
        want = _rne(_f32_value(r["st"], case.src), case.dst)
        assert torch.equal(_bits(got), _bits(want)), f"{name}: not bit-exact"
        return
    outs = r["outs"]
    if k == "conv":
        N, H, W = case.shape
        xv = _value(_read_back(r["xbuf"], case.fin, case.in_slice, case.cin_read, name, "input"), case.fin)
        rv = _value(r["rst"], case.res) if r["rst"] is not None else None
        y, bound = _conv_reference(case, r["pc"], xv, rv)
        width, oco, _ = case.out_slice or (case.cout, 0, False)
        sl, C = (width, oco), case.cout
    elif k == "dwln":
        xv = _value(_read_back(r["xbuf"], case.fin, case.in_slice, case.C, name, "input"), case.fin)
        y, bound = _dw_reference(case, xv, *r["params"])
        sl, C = None, case.C
    elif k == "meanln":
        xv = _value(r["xst"], case.fin)
        y, bound = _ml_reference(case, xv, *r["params"])
        sl, C = case.out_slice, case.C
    else:
        xv = _value(_read_back(r["xbuf"], case.fin, case.in_slice, r["xst"].shape[-1], name, "input"), case.fin)
        y = _pool_reference(case, xv)
        bound = torch.zeros_like(y)
        sl, C = None, case.shape[3]
    a = _read_back(outs["A"], "f32", sl, C, name, "run A output")
    b = _read_back(outs["B"], case.fout, sl, C, name, "run B output")
    assert a.shape == y.shape, f"{name}: shape {tuple(a.shape)} != {tuple(y.shape)}"
    if k == "pool":
        assert torch.equal(a.double(), y), f"{name}: max pooling is not exact"
    else:
        _check_bound(name, a, y, bound)
    _check_rounding(name, a, b, case.fout)


@pytest.mark.gpu
@pytest.mark.parametrize("src", FMTS)
@pytest.mark.parametrize("dst", FMTS)
def test_convert_vector_equals_scalar(src, dst):
    """The same conversion through k_act_convert (4-aligned views) and k_act_convert_scalar (a view at channel 3) gives
    identical bits, on random values and the special values."""
    from heal_b200 import ops
    case = Cvt("vs", src, dst, (2, 5, 9, 64), VEC)
    st = _store(_cvt_input(case), src)
    outs = []
    for sl in (None, (67, 3)):
        _, sact = _put(st, src, sl)
        dbuf = _out_buffer(2, 5, 9, 64, dst, False)
        ops.convert(sact, dst, out=ops.Act(dbuf, dst))
        outs.append(dbuf.cpu())
    assert torch.equal(_bits(outs[0]), _bits(outs[1]))


# ------------------------------------------------------------------------------------------------ instantiations (profiler)
_KERNEL = re.compile(r"\b(k_act_convert_scalar|k_act_convert|k_conv2d_dense|k_conv2d_grouped|k_dwconv_ln|k_mean_layernorm|"
                     r"k_maxpool3s2)\b(?:<\s*(\d+)\s*,\s*(\d+)\s*,\s*(\d+)\s*>)?")


def _launched_name(key):
    """`k_name` / `k_conv2d_grouped<a,b,c>` for one of these kernels' profiler names, None for any other kernel."""
    m = _KERNEL.search(key)
    if not m:
        return None
    return m.group(1) + (f"<{m.group(2)},{m.group(3)},{m.group(4)}>" if m.group(2) else "")


def _launched(prof):
    return {n for n in (_launched_name(e.key) for e in prof.key_averages()) if n}


def _profiled_kernels():
    """Runs every case under one torch.profiler session; returns the kernels it recorded, in launch order.  A session that
    recorded none of the launches the library counted is repeated once (a wrong kernel never is)."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    from heal_b200._lib import lib
    for _ in range(2):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for case in CASES:
                before = lib.heal_launch_count()
                _launch(case)
                torch.cuda.synchronize()
                assert lib.heal_launch_count() - before == _launches(case), f"{case.name}: launch count"
        ours = sorted((e.time_range.start, _launched_name(e.name)) for e in prof.events()
                      if e.device_type == DeviceType.CUDA and _launched_name(e.name))
        if ours:
            break
    return [n for _, n in ours]


@pytest.mark.gpu
def test_each_case_launches_its_instantiations():
    """Each case runs the instantiations its row names (kernel names from torch.profiler), and together the cases run all
    nine.  The session runs in a child process, for the reason test_gpu_fuse_kernels.py gives: torch.profiler's CUDA records
    can come back empty from a short session late in a long process."""
    tests_dir = os.path.dirname(os.path.abspath(__file__))
    code = ("import json, sys; sys.path[:0] = [%r, %r]; import test_gpu_simt_map_kernels as t; "
            "print('KERNELS ' + json.dumps(t._profiled_kernels()))" % (tests_dir, os.path.dirname(tests_dir)))
    r = subprocess.run([sys.executable, "-s", "-c", code], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                       timeout=900)
    assert r.returncode == 0, r.stdout[-4000:]
    names = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("KERNELS ")][-1][len("KERNELS "):])
    total = sum(_launches(c) for c in CASES)
    assert len(names) == total, f"the session recorded {len(names)} kernels for {total} launches"
    i = 0
    for case in CASES:
        n = _launches(case)
        assert set(names[i:i + n]) == set(case.reaches), f"{case.name}: ran {names[i:i + n]}, expected {sorted(case.reaches)}"
        i += n
    print(f"instantiations reached: {len(set(names) & REACHABLE)} of {len(REACHABLE)}")
    assert set(names) == REACHABLE


# ------------------------------------------------------------------------------------------------ misaligned views
def _act(N, H, W, c, fmt, bad):
    """An Act of c channels at channel 2 (bad: an 8-byte aligned fp32 / 4-byte aligned bf16 data pointer) or 0 of a buffer
    of c + 4 channels, filled with small random values."""
    from heal_b200 import ops
    g = torch.Generator().manual_seed(N * 1000 + H * 10 + c)
    t = torch.randn((N, H, W, c + 4), generator=g)
    t = t if fmt == "f32" else t.to(torch.bfloat16)[None]
    t = t.cuda()
    return ops.Act(t[..., 2:2 + c] if bad else t[..., :c], fmt)


def _refused_call(what, fmt):
    from heal_b200 import ops
    if what in ("conv_dense_in", "conv_grouped_in", "conv_grouped_out"):
        grouped = what != "conv_dense_in"
        case = Conv("mis", (1, 6, 7), 128, 128, 3, fmt, fmt, G4 if grouped else DENSE, groups=32 if grouped else 1)
        pc = _packed(case).to("cuda")
        x = _act(1, 6, 7, 128, fmt, what.endswith("_in"))
        o = _act(1, 6, 7, 128, fmt, what == "conv_grouped_out")
        return lambda: ops.conv2d_simt(x, pc, out=o)
    if what == "pool_in":
        x = _act(1, 9, 11, 64, fmt, True)
        return lambda: ops.maxpool3x3s2(x, out_fmt=fmt)
    if what == "pool_out":
        # ops.maxpool3x3s2 allocates its output: the misaligned out view goes to the launcher directly
        x, o = _act(1, 9, 11, 64, fmt, False), _act(1, 5, 6, 64, fmt, True)
        return lambda: ops._call("heal_maxpool3x3s2", x.view(), 1, 9, 11, 64, 0, o.view())
    # dw_weight at a 4-byte offset
    x = _act(1, 6, 7, 64, fmt, False)
    wbuf = torch.randn(49 * 64 + 1).cuda()
    lw, lb = torch.ones(64, device="cuda"), torch.zeros(64, device="cuda")
    return lambda: ops.dwconv_layernorm(x, wbuf[1:].view(49, 64), None, 7, lw, lb, EPS)


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["f32", "bf16"])
@pytest.mark.parametrize("what", ["conv_dense_in", "conv_grouped_in", "conv_grouped_out", "pool_in", "pool_out", "dw_weight"])
def test_misaligned_view_is_refused(what, fmt):
    """A view whose data pointer the 4-channel loads or stores cannot use (channel 2 of a wider buffer), or a dw_weight the
    float2 loads cannot use, is refused (HEAL_ERR_UNSUPPORTED -> RuntimeError) and nothing is launched."""
    from torch.profiler import ProfilerActivity, profile
    from heal_b200._lib import lib
    call = _refused_call(what, fmt)
    torch.cuda.synchronize()
    before = lib.heal_launch_count()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        with pytest.raises(RuntimeError, match="HEAL_ERR_UNSUPPORTED"):
            call()
        torch.cuda.synchronize()
    assert lib.heal_launch_count() == before
    assert not _launched(prof), f"{what}: launched {sorted(_launched(prof))}"


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["f32", "bf16"])
def test_misaligned_dense_output_takes_scalar_stores(fmt):
    """The dense conv writes a misaligned output view (channel 2 of a wider buffer) one channel at a time: the same bits as
    into an aligned view, and the channels around it keep their sentinel."""
    from heal_b200 import ops
    case = Conv("mis_out", (2, 9, 13), 64, 64, 3, "f32", fmt, DENSE)
    pc = _packed(case).to("cuda")
    x = _act(2, 9, 13, 64, "f32", False)
    outs = []
    for off in (0, 2):
        buf = _out_buffer(2, 9, 13, 68, fmt, True)
        ops.conv2d_simt(x, pc, out=ops.Act(buf[..., off:off + 64], fmt))
        outs.append(_read_back(buf, fmt, (68, off), 64, case.name, "output"))
    assert torch.equal(_bits(outs[0]), _bits(outs[1]))
