"""The attention kernels of csrc/v2xvit.cu and csrc/swap_attn.cu against a float64 reference, one case per kernel instantiation
the dispatch can reach.

heal_window_attention (k_window_attention<WS, DH, SPLIT>: WS in {4, 8, 16}, DH in {16, 32, 64}, SPLIT for fp32 and split
input, not for bf16 input), heal_cav_attention (k_cav_attention), heal_split_attn (k_split_pool -> k_split_gate ->
k_split_combine), heal_sttf_resample (k_sttf_resample) and heal_swap_attention (k_swap_attention, window and grid mode).  Every
case runs its kernels twice: with fp32 output (run A) and with the product's output format, the format of the input (run B).
The checks:
  - A is within a per-element bound of a float64 reference computed on the exact input the kernel read (hi + lo for split
    input, the bf16 value for bf16 input);
  - B is bit for bit the rounding of A: bf16(A); for split, hi = bf16(A) and lo = bf16(A - hi); for fp32, A itself;
  - the channels around an input or output slice keep their sentinel, and output the kernel does not write (pre-filled with
    NaN) would fail the bound.

The bound is first order in the reference's own quantities.  For a query with float64 softmax weights p_j over its keys, the
output o = sum_j p_j v_j and T_j = sum_c |q_c| |k_jc| + |s_j| (s_j the score, bias included):
  attention  |err| <= A_S sum_j p_j T_j |v_j - o| + A_P sum_j p_j |v_j| + REL |o|   (per channel).
  The first term carries the score errors: a score error ds_j <= A_S T_j moves the output by sum_j dp_j v_j with
  dp_j = p_j (ds_j - sum_k p_k ds_k), i.e. by sum_j p_j ds_j (v_j - o).  The second carries the rounding of P and V and of
  the sums of P V.  (A_S, A_P) per kernel and mode:
    cav, swap (fp32 on the CUDA cores, every input format)            (ALPHA, ALPHA)
    window, split or fp32 input (hi / lo products; lo * lo dropped)   (WIN_SPLIT, WIN_SPLIT)
    window, bf16 input (bf16 products are exact in fp32; P is rounded
    to bf16 before P V, 2^-9 relative)                                (WIN_BF16_S, WIN_BF16_P)
  split      the gate's error propagated through every stage to first order: with G = mean over the pixels of
             |o_0| + |o_1| + |o_2|, Y = |fc1| G, the LayerNorm's normalised yh and sigma,
             dyh = (Y + mean(Y) + |yh| mean(|yh| Y)) / sigma + |yh|,  dr = |ln_w| dyh + |r|,  dz = |fc2| (dr + relu(r)),
             dg_b = g_b (dz_b + sum_b' g_b' dz_b') + g_b  (the softmax over the three branches), and then
             |err| <= ALPHA (sum_b |o_b| (dg_b + g_b) + |x|) + REL |out|.
  sttf       taps and bilinear weights taken from PyTorch's fp32 F.affine_grid (align_corners=True) and the kernel's fp32
             unnormalisation (gx + 1) * ((W - 1) / 2), floor and weight products; the weighted sum in float64:
             |err| <= ALPHA sum_t w_t |v_t| + REL |y|.  On an axis of one pixel F.affine_grid's base coordinate is 0, not
             linspace's -1 (the H = 1 and W = 1 cases; k_sttf_resample used -1 until these cases found it).
REL = 2^-22 covers the final fp32 rounding.  test_bound_rejects_plausible_kernel_bugs (no GPU) shows that the bound rejects
each plausible kernel bug on these cases, and test_reference_matches_the_modules (no GPU) pins each float64 restatement to the
functional restatement of the reference's module in oracle/.

The window cases include built inputs for the online softmax (KC = 32 keys per chunk when a window holds more than 32
tokens): a key whose bias leads every other score by >= 30 in the first chunk, or in the last; scores whose largest exceeds
88, where expf without the running maximum overflows; an all-zero q with a zero bias, whose output is the exact mean of v; a
bias with entries of -1e4.

Calibration, on an H100 80GB HBM3 at a 700 W power limit: largest err / bound per case with the constants below (a ratio of
0 means the output was exact)
  window   <16,16,false>-bf16_h3 0.151, <16,16,true>-split_h2_big 0.144, <16,32,false>-bf16_h2_zero_q 0,
           <16,32,true>-f32_h2_first 0.462, <16,32,true>-split_h2_last 0, <16,64,false>-bf16_h1_big 0.378,
           <16,64,false>-bf16_h2_first 0, <16,64,true>-split_h4_shipped 0.050, <4,16,false>-bf16_h3 0.286,
           <4,32,false>-bf16_h3 0.314, <4,32,true>-split_h2_zero_q 0.005, <4,64,false>-bf16_h1 0.275, <4,64,true>-f32_h2
           0.180, <8,16,false>-bf16_h2 0.239, <8,16,true>-f32_h3_neg_bias 0.138, <8,32,false>-bf16_h2_last 0,
           <8,32,true>-split_h2_first 0, <8,32,true>-split_h8_shipped 0.077, <8,64,false>-bf16_h1 0.276,
           <8,64,false>-bf16_h1_neg_bias 0.222, <8,64,true>-split_h2_big 0.080
  cav      bf16_c64_130scenes_ego 0.245, bf16_c64_n8315_ego 0.158, f32_c128_n284 0.210, f32_c256_onehot 0.380,
           f32_c64_65scenes 0.223, split_c256_n1to8 0.243, split_c512_n82_ego 0.206, split_c64_130scenes 0.235
  split    bf16_xbf16_hw117_small 0.074, bf16_xf32_hw31_small 0.070, bf16_xsplit_hw4087_big_logits 0.041,
           f32_xbf16_hw1_small 0.063, f32_xf32_hw117_big_logits 0.013, f32_xsplit_hw33_small 0.075, split_xbf16_hw7_small
           0.071, split_xf32_hw1000 0.004, split_xsplit_hw32 0.001
  sttf     bf16_16x24_c64 0.237, bf16_7x1_c8 0.084, f32_10x14_c64 0.175, f32_1x9_c16 0.100, split_12x20_c32 0.222,
           split_33x47_c32 0.233
  swap     grid_bf16_w4_L4_c64 0.218, grid_f32_w2_L5_c32 0.253, grid_split_w1_L1_c256 0, grid_split_w2_L2_c32_65scenes
           0.312, grid_split_w4_L8_c96 0.218, grid_split_w8_L2_c512 0.339, window_bf16_w1_L3_c64 0.201,
           window_bf16_w8_L2_c128 0.229, window_f32_w2_L3_c64_65scenes 0.339, window_f32_w4_L1_c512 0.300,
           window_f32_w4_L8_c64 0.263
so ALPHA = 2^-21 leaves 2.6x of headroom over the largest fp32 CUDA-core ratio (cav onehot), WIN_SPLIT = 2^-16 2.2x over
f32_h2_first (the fp32 input's own hi / lo split costs up to 2^-18 of |v|), and (WIN_BF16_S, WIN_BF16_P) = (2^-20, 2^-7)
2.6x over bf16_h1_big.
"""
import ctypes
import math
import zlib
from dataclasses import dataclass, field
from typing import Optional, Tuple

import numpy as np
import pytest
import torch
import torch.nn.functional as F

# Calibrated on an H100 80GB HBM3 at a 700 W power limit; the module docstring lists every case's err / bound, which
# test_attention_kernel prints.
ALPHA = 2.0 ** -21          # fp32 CUDA-core kernels: cav, swap, split, sttf
WIN_SPLIT = 2.0 ** -16      # window attention, SPLIT products (score and P V)
WIN_BF16_S = 2.0 ** -20     # window attention, bf16 input: scores
WIN_BF16_P = 2.0 ** -7      # window attention, bf16 input: P rounded to bf16
REL = 2.0 ** -22
SENTINEL = -1000.0          # finite and exact in bf16: fills the channels around a slice
KC = 32                     # keys per online-softmax chunk of k_window_attention (windows of more than 32 tokens)
CAV_SCENES = SWAP_SCENES = 64


@dataclass
class Case:
    name: str
    kernel: str                                   # window | cav | split | sttf | swap
    fmt: str                                      # input storage format: f32 | bf16 | split
    p: dict = field(default_factory=dict)         # the kernel's shape and options
    in_slice: Optional[Tuple[int, int]] = None    # (buffer width, channel offset) of the (first) input
    out_slice: Optional[Tuple[int, int]] = None   # (buffer width, channel offset) of the output

    @property
    def reaches(self):
        if self.kernel == "window":
            return (f"k_window_attention<{self.p['ws']},{self.p['dh']},{'false' if self.fmt == 'bf16' else 'true'}>",)
        return {"cav": ("k_cav_attention",), "split": ("k_split_pool", "k_split_gate", "k_split_combine"),
                "sttf": ("k_sttf_resample",), "swap": ("k_swap_attention",)}[self.kernel]


def _win(ws, dh, fmt, heads, N, H, W, special=None, in_slice=None, out_slice=None, tag=""):
    name = f"k_window_attention<{ws},{dh},{'false' if fmt == 'bf16' else 'true'}>-{fmt}_h{heads}" + \
        (f"_{special}" if special else "") + tag
    return Case(name, "window", fmt, dict(ws=ws, dh=dh, heads=heads, N=N, H=H, W=W, special=special), in_slice, out_slice)


def _cav(fmt, C, rl, ego_only, H, W, tag, special=None, in_slice=None, out_slice=None):
    return Case(f"k_cav_attention-{fmt}_c{C}_{tag}{'_ego' if ego_only else ''}", "cav", fmt,
                dict(C=C, rl=tuple(rl), ego_only=ego_only, H=H, W=W, special=special), in_slice, out_slice)


def _swap(fmt, C, rl, L, w, grid, H, W, tag="", in_slice=None, out_slice=None):
    return Case(f"k_swap_attention-{'grid' if grid else 'window'}_{fmt}_w{w}_L{L}_c{C}{tag}", "swap", fmt,
                dict(C=C, rl=tuple(rl), L=L, w=w, grid=grid, H=H, W=W), in_slice, out_slice)


def _split(fmt, xfmt, N, H, W, tag="", big=False, small=False, in_slice=None, out_slice=None):
    tag += "_big_logits" if big else ""
    tag += "_small" if small else ""
    return Case(f"k_split_pool+gate+combine-{fmt}_x{xfmt}_hw{H * W}{tag}", "split", fmt,
                dict(xfmt=xfmt, N=N, H=H, W=W, big=big, small=small), in_slice, out_slice)


def _sttf(fmt, thetas, H, W, C, tag="", in_slice=None, out_slice=None):
    return Case(f"k_sttf_resample-{fmt}_{H}x{W}_c{C}{tag}", "sttf", fmt, dict(thetas=tuple(thetas), H=H, W=W, C=C),
                in_slice, out_slice)


SCENES65 = [(5 * i + 3) % 8 + 1 for i in range(65)]
SCENES130 = [(3 * i) % 8 + 1 for i in range(130)]

CASES = [
    # ---- heal_window_attention: every (WS, DH) with SPLIT (split or fp32 input) and without (bf16 input).  The shipped
    # V2X-ViT branches are heads / dim_head / window 16 / 16 / 4, 8 / 32 / 8 and 4 / 64 / 16 (mswin.py, lidar_v2xvit.yaml).
    _win(4, 16, "split", 16, 2, 8, 12, in_slice=(3 * 256 + 8, 4), out_slice=(256 + 8, 4), tag="_shipped"),
    _win(4, 16, "bf16", 3, 3, 12, 8),
    _win(4, 32, "split", 2, 2, 8, 8, "zero_q"),
    _win(4, 32, "bf16", 3, 2, 12, 16, in_slice=(3 * 96 + 6, 2), out_slice=(96 + 4, 2)),
    _win(4, 64, "f32", 2, 2, 8, 12),
    _win(4, 64, "bf16", 1, 3, 4, 8),
    _win(8, 16, "f32", 3, 2, 16, 24, "neg_bias"),
    _win(8, 16, "bf16", 2, 2, 16, 16, out_slice=(32 + 8, 6)),
    _win(8, 32, "split", 8, 2, 16, 24, tag="_shipped"),
    _win(8, 32, "split", 2, 2, 16, 16, "first"),
    _win(8, 32, "bf16", 2, 2, 24, 16, "last"),
    _win(8, 64, "split", 2, 2, 16, 16, "big", in_slice=(3 * 128 + 4, 2)),
    _win(8, 64, "bf16", 1, 2, 16, 24),
    _win(8, 64, "bf16", 1, 1, 16, 16, "neg_bias"),
    _win(16, 16, "split", 2, 2, 32, 48, "big"),
    _win(16, 16, "bf16", 3, 1, 32, 32),
    _win(16, 32, "f32", 2, 2, 32, 32, "first", out_slice=(64 + 8, 4)),
    _win(16, 32, "split", 2, 2, 32, 32, "last"),
    _win(16, 32, "bf16", 2, 1, 32, 48, "zero_q"),
    _win(16, 64, "split", 4, 2, 32, 32, tag="_shipped"),
    _win(16, 64, "bf16", 2, 1, 32, 48, "first"),
    _win(16, 64, "bf16", 1, 1, 16, 32, "big"),
    # ---- heal_cav_attention: scenes of 1 .. 8 agents (CAV_MAX_L), H W C / 4 never a multiple of 256 (a partial last block),
    # 65 and 130 scenes (two and three launches, the later ones continuing the scene table)
    _cav("split", 256, range(1, 9), False, 5, 7, "n1to8", in_slice=(3 * 256 + 8, 4)),
    _cav("bf16", 64, [8, 3, 1, 5], True, 3, 5, "n8315", out_slice=(64 + 8, 4)),
    _cav("f32", 128, [2, 8, 4], False, 6, 3, "n284"),
    _cav("split", 512, [8, 2], True, 3, 3, "n82"),
    _cav("f32", 64, SCENES65, False, 3, 3, "65scenes"),
    _cav("bf16", 64, SCENES130, True, 2, 3, "130scenes"),
    _cav("split", 64, SCENES130, False, 2, 3, "130scenes", out_slice=(64 + 4, 4)),
    _cav("f32", 256, [3, 6], False, 4, 5, "onehot", special="onehot"),
    # ---- heal_split_attn (C = 256): maps of 1 .. 4087 pixels, so some of the 32 pooling slabs are empty or ragged
    _split("f32", "bf16", 3, 1, 1, small=True),
    _split("split", "bf16", 2, 1, 7, small=True),
    _split("bf16", "f32", 2, 31, 1, small=True),
    _split("split", "split", 2, 4, 8, in_slice=(3 * 256 + 8, 4)),
    _split("f32", "split", 3, 3, 11, small=True, out_slice=(256 + 4, 4)),
    _split("bf16", "bf16", 2, 9, 13, small=True),
    _split("f32", "f32", 2, 9, 13, big=True),
    _split("split", "f32", 2, 25, 40),
    _split("bf16", "split", 2, 61, 67, big=True),
    # ---- heal_sttf_resample: a theta per image
    _sttf("split", ["identity", "rot", "outside"], 12, 20, 32, out_slice=(40, 4)),
    _sttf("f32", ["identity", "rot"], 1, 9, 16),
    _sttf("bf16", ["rot", "identity"], 7, 1, 8),
    _sttf("f32", ["clamp+", "identity", "clamp-"], 10, 14, 64, in_slice=(72, 4)),
    _sttf("bf16", ["rot", "rot2", "outside"], 16, 24, 64),
    _sttf("split", ["rot2", "identity"], 33, 47, 32),
    # ---- heal_swap_attention: L w^2 up to 128 (a full CTA), L = 1, nb = L and nb = 1, C up to 512, 65 scenes
    _swap("f32", 64, [8, 3], 8, 4, False, 8, 12),
    _swap("split", 96, [8, 1], 8, 4, True, 8, 8, in_slice=(3 * 96 + 8, 4)),
    _swap("bf16", 64, [4, 4], 4, 4, True, 8, 8),
    _swap("bf16", 128, [2, 1], 2, 8, False, 16, 24, out_slice=(128 + 8, 4)),
    _swap("split", 512, [1], 2, 8, True, 16, 16),
    _swap("f32", 32, [5, 2, 1], 5, 2, True, 6, 10),
    _swap("bf16", 64, [3, 1], 3, 1, False, 3, 5),
    _swap("split", 256, [1, 1, 1], 1, 1, True, 4, 5),
    _swap("f32", 512, [1], 1, 4, False, 8, 8),
    _swap("split", 32, [2 - (i % 2) for i in range(65)], 2, 2, True, 4, 4, tag="_65scenes"),
    _swap("f32", 64, [1 + (i % 3) for i in range(65)], 3, 2, False, 4, 6, tag="_65scenes"),
]
CASE = {c.name: c for c in CASES}
assert len(CASE) == len(CASES), "case names must be unique"

# every instantiation the five launchers can dispatch to
REACHABLE = {f"k_window_attention<{ws},{dh},{s}>" for ws in (4, 8, 16) for dh in (16, 32, 64) for s in ("true", "false")} | \
    {"k_cav_attention", "k_split_pool", "k_split_gate", "k_split_combine", "k_sttf_resample", "k_swap_attention"}


# ------------------------------------------------------------------------------------------------ storage
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


# ------------------------------------------------------------------------------------------------ inputs
def _gen(case):
    return torch.Generator().manual_seed(zlib.crc32(case.name.encode()))


def _window_inputs(case):
    p, g = case.p, _gen(case)
    ws, dh, heads = p["ws"], p["dh"], p["heads"]
    n, inner = ws * ws, heads * dh
    qkv = torch.randn(p["N"], p["H"], p["W"], 3 * inner, generator=g)
    qkv[..., :inner] *= dh ** -0.5                        # q pre-scaled, as the to_qkv conv delivers it
    bias = torch.randn(n, n, generator=g)
    sp = p["special"]
    if sp in ("first", "last"):                           # one key leads every score by >= 30 (asserted by _window_ref)
        bias[:, 3 if sp == "first" else n - 5] += 48.0
    elif sp == "big":                                     # scores beyond 88: expf(s) alone would overflow
        qkv[..., :inner] *= 30.0
    elif sp == "zero_q":                                  # s = 0 everywhere: the exact mean of v
        qkv[..., :inner] = 0
        bias.zero_()
    elif sp == "neg_bias":
        drop = torch.rand(n, n, generator=g) < 0.3
        drop.fill_diagonal_(False)
        bias[drop] = -1e4
    return dict(qkv=qkv, bias=bias)


def _cav_inputs(case):
    p, g = case.p, _gen(case)
    C = p["C"]
    qkv = torch.randn(sum(p["rl"]), p["H"], p["W"], 3 * C, generator=g)
    qkv[..., :C] *= 32 ** -0.5 * (20.0 if p["special"] == "onehot" else 1.0)
    return dict(qkv=qkv)


def _swap_inputs(case):
    p, g = case.p, _gen(case)
    C, n = p["C"], p["L"] * p["w"] ** 2
    qkv = torch.randn(len(p["rl"]) * p["L"], p["H"], p["W"], 3 * C, generator=g)
    qkv[..., :C] *= 32 ** -0.5
    return dict(qkv=qkv, bias=torch.randn(C // 32, n, n, generator=g))      # key-major: bias[h, j, i]


def _split_inputs(case):
    p, g = case.p, _gen(case)
    N, H, W, C = p["N"], p["H"], p["W"], 256
    # features with a mean per image and channel (the pooled mean is not a cancellation of random signs), so that the images'
    # gates differ.  small: features of 1e-3, whose pooled mean has a variance over the channels of the order of the
    # LayerNorm's eps; elsewhere the LayerNorm does not see the scale of the pooled mean.
    o = torch.randn(N, H, W, 3 * C, generator=g) + 2 * torch.randn(N, 1, 1, 3 * C, generator=g)
    o *= 1e-3 if p["small"] else 1.0
    x = torch.randn(N, H, W, C, generator=g)
    fc1 = torch.randn(C, C, generator=g) / 16
    fc2 = torch.randn(3 * C, C, generator=g) / (2 if p["big"] else 16)     # big: gate logits of +-20 and more
    lw, lb = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g) * 0.1
    return dict(o=o, x=x, fc1=fc1, fc2=fc2, lw=lw, lb=lb, eps=1e-5)


def _theta(kind, H, W):
    """(2, 3) normalised affine_grid matrix (align_corners=True)."""
    if kind == "identity":
        return [[1.0, 0.0, 0.0], [0.0, 1.0, 0.0]]
    if kind in ("rot", "rot2"):
        a, tx, ty = (0.3, 0.137, -0.219) if kind == "rot" else (-1.1, -0.31, 0.47)
        c, s = math.cos(a), math.sin(a)
        return [[c, -s, tx], [s, c, ty]]
    if kind == "outside":          # every ix >= W + 0.5: both x taps off the map; ix > W + 2 takes the clamp path
        return [[1.0, 0.0, (2 * W + 1) / (W - 1)], [0.0, 1.0, 0.0]]
    return [[1.0, 0.0, 1e4 if kind == "clamp+" else -1e4], [0.0, 1.0, 0.5]]  # clamp+ / clamp-: the x0 clamp path


def _sttf_inputs(case):
    p, g = case.p, _gen(case)
    th = torch.tensor([_theta(k, p["H"], p["W"]) for k in p["thetas"]], dtype=torch.float32)
    return dict(src=torch.randn(len(p["thetas"]), p["H"], p["W"], p["C"], generator=g), theta=th)


INPUTS = {"window": _window_inputs, "cav": _cav_inputs, "swap": _swap_inputs, "split": _split_inputs, "sttf": _sttf_inputs}


def _storage(case, inp):
    """The storage tensors of a case's activation inputs (the kernel reads exactly these)."""
    if case.kernel == "split":
        return dict(o=_store(inp["o"], case.fmt), x=_store(inp["x"], case.p["xfmt"]))
    key = "src" if case.kernel == "sttf" else "qkv"
    return {key: _store(inp[key], case.fmt)}


def _fmt_of(case, key):
    return case.p["xfmt"] if key == "x" else case.fmt


# ------------------------------------------------------------------------------------------------ float64 reference
def _attend(q, k, v, bias=None, keep=None):
    """float64 softmax(q k^T + bias) v over batches: q (B,nq,d), k, v (B,nk,d), bias broadcastable to (B,nq,nk), keep
    (B,nk) bool (masked keys: -inf).  Returns o, t1 = sum_j p_j T_j |v_j - o| and t2 = sum_j p_j |v_j|, each (B,nq,d)."""
    s = q @ k.transpose(-1, -2)
    if bias is not None:
        s = s + bias
    T = q.abs() @ k.abs().transpose(-1, -2) + s.abs()
    if keep is not None:
        s = s.masked_fill(~keep[:, None, :], -math.inf)
    p = torch.softmax(s, -1)
    o = p @ v
    pT = torch.where(p > 0, p * T, 0.0)
    t1 = torch.empty_like(o)
    B, nq, nk, d = q.shape[0], q.shape[1], k.shape[1], q.shape[2]
    step = max(1, int(2e7) // (nq * nk * d))
    for a in range(0, B, step):
        dv = (v[a:a + step, None, :, :] - o[a:a + step, :, None, :]).abs()
        t1[a:a + step] = (pT[a:a + step, :, :, None] * dv).sum(2)
    return o, t1, p @ v.abs()


def _online(s, v, fault):
    """The kernel's online softmax restated in float64 with one of its plausible bugs: the last chunk's rescale skipped, or
    the last chunk dropped.  s (B,nq,nk), v (B,nk,d)."""
    B, nq, nk = s.shape
    m = torch.full((B, nq, 1), -math.inf, dtype=s.dtype)
    l = torch.zeros(B, nq, 1, dtype=s.dtype)
    o = torch.zeros(B, nq, v.shape[-1], dtype=s.dtype)
    last = (nk - 1) // KC * KC
    for j0 in range(0, nk, KC):
        if fault == "drop_last" and j0 == last:
            break
        sc = s[..., j0:j0 + KC]
        mc = torch.maximum(m, sc.max(-1, keepdim=True).values)
        corr = torch.exp(m - mc)
        if fault == "skip_rescale" and j0 == last:
            corr = torch.ones_like(corr)
        e = torch.exp(sc - mc)
        l = l * corr + e.sum(-1, keepdim=True)
        o = o * corr + e @ v[:, j0:j0 + KC]
        m = mc
    return o / l


def _win_tokens(x, ws):
    """(N,H,W,C) -> (N,X,Y,ws*ws,C): token t = (w1, w2) of window (x, y) is pixel (x*ws + w1, y*ws + w2)."""
    N, H, W, C = x.shape
    return x.reshape(N, H // ws, ws, W // ws, ws, C).permute(0, 1, 3, 2, 4, 5).reshape(N, H // ws, W // ws, ws * ws, C)


def _win_untokens(t, ws):
    N, X, Y, n, C = t.shape
    return t.reshape(N, X, Y, ws, ws, C).permute(0, 1, 3, 2, 4, 5).reshape(N, X * ws, Y * ws, C)


def _window_ref(qkv, heads, dh, ws, bias, fault=None, special=None):
    """qkv (N,H,W,3*inner) float64 (q | k | v, q pre-scaled), bias (n,n) query-major -> o, t1, t2 (N,H,W,inner)."""
    inner, n = heads * dh, ws * ws
    t = _win_tokens(qkv, ws)
    N, X, Y = t.shape[:3]
    t = t.reshape(N, X, Y, n, 3, heads, dh).permute(4, 0, 1, 2, 5, 3, 6).reshape(3, -1, n, dh)
    b = (bias.t() if fault == "bias_t" else bias)[None]
    if special in ("first", "last") and fault is None:
        s = (t[0] @ t[1].transpose(-1, -2) + b).sort(-1, descending=True).values
        lead = (s[..., 0] - s[..., 1]).min().item()
        assert lead >= 30, f"the dominant key leads by only {lead:.1f}"
    if special == "big" and fault is None:
        top = (t[0] @ t[1].transpose(-1, -2) + b).max().item()
        assert top > 88, f"the largest score is {top:.1f}: expf(s) would not overflow"
    if fault in ("skip_rescale", "drop_last"):
        o = _online(t[0] @ t[1].transpose(-1, -2) + b, t[2], fault)
        t1 = t2 = torch.zeros_like(o)
    else:
        o, t1, t2 = _attend(t[0], t[1], t[2], b)

    def back(u):
        return _win_untokens(u.reshape(N, X, Y, heads, n, dh).permute(0, 1, 2, 4, 3, 5).reshape(N, X, Y, n, inner), ws)
    return back(o), back(t1), back(t2)


def _cav_table(rl, fault=None):
    """(ego image, first non-ego image, agents) per scene; images egos first, then each scene's others in scene order."""
    B, other, table = len(rl), len(rl), []
    for b, n in enumerate(rl):
        if fault == "restart" and b % CAV_SCENES == 0:     # each launch restarting the non-ego image counter
            other = B
        table.append(((b + 1) % B if fault == "image_of" else b, other, n))
        other += n - 1
    return table


def _cav_ref(qkv, rl, ego_only, fault=None):
    """qkv (N,H,W,3C) float64 (q pre-scaled) -> o, t1, t2 (N or B,H,W,C): per pixel and head of 32, attention over the
    scene's agents."""
    Nimg, H, W, C3 = qkv.shape
    C, HW = C3 // 3, H * W
    heads = C // 32
    out = [torch.zeros(len(rl) if ego_only else Nimg, H, W, C, dtype=qkv.dtype) for _ in range(3)]
    for b, (ego, other0, n) in enumerate(_cav_table(rl, fault)):
        idx = [ego] + list(range(other0, other0 + n - 1))
        x = qkv[idx].reshape(n, HW, 3, heads, 32).permute(2, 1, 3, 0, 4).reshape(3, HW * heads, n, 32)
        res = [r.reshape(HW, heads, n, 32).permute(2, 0, 1, 3).reshape(n, H, W, C) for r in _attend(x[0], x[1], x[2])]
        for dst, r in zip(out, res):
            if ego_only:
                dst[b] = r[0]
            else:
                dst[idx] = r
    return tuple(out)


def _swap_tokens(x, B, L, w, grid):
    """(B*L,H,W,C) -> (B,X,Y,L*w*w,C), tokens (l, w1, w2).  window: pixel (x*w + w1, y*w + w2); grid: (w1*X + x, w2*Y + y)."""
    BL, H, W, C = x.shape
    X, Y = H // w, W // w
    if grid:
        t = x.reshape(B, L, w, X, w, Y, C).permute(0, 3, 5, 1, 2, 4, 6)
    else:
        t = x.reshape(B, L, X, w, Y, w, C).permute(0, 2, 4, 1, 3, 5, 6)
    return t.reshape(B, X, Y, L * w * w, C)


def _swap_untokens(t, L, w, grid):
    B, X, Y, n, C = t.shape
    t = t.reshape(B, X, Y, L, w, w, C)
    t = t.permute(0, 3, 4, 1, 5, 2, 6) if grid else t.permute(0, 3, 1, 4, 2, 5, 6)
    return t.reshape(B * L, X * w, Y * w, C)


def _swap_ref(qkv, rl, L, w, grid, bias, fault=None):
    """qkv (B*L,H,W,3C) float64 (q pre-scaled), bias (heads,n,n) key-major -> o, t1, t2 (B*L,H,W,C): attention over the
    tokens of each window (grid cell) whose agent is real; padded agents are queries, not keys."""
    B, C = len(rl), qkv.shape[-1] // 3
    heads, n = C // 32, L * w * w
    grid = grid != (fault == "mode")
    t = _swap_tokens(qkv, B, L, w, grid)
    X, Y = t.shape[1:3]
    t = t.reshape(B, X, Y, n, 3, heads, 32).permute(4, 0, 1, 2, 5, 3, 6).reshape(3, -1, n, 32)
    bq = bias if fault == "bias_t" else bias.transpose(-1, -2)             # query-major
    bq = bq[None, None, None].expand(B, X, Y, heads, n, n).reshape(-1, n, n)
    keep = torch.arange(n)[None, :] < torch.tensor([n if fault == "pad_keys" else r * w * w for r in rl])[:, None]
    keep = keep[:, None, None, None].expand(B, X, Y, heads, n).reshape(-1, n)
    res = _attend(t[0], t[1], t[2], bq, keep)
    return tuple(_swap_untokens(r.reshape(B, X, Y, heads, n, 32).permute(0, 1, 2, 4, 3, 5).reshape(B, X, Y, n, C), L, w, grid)
                 for r in res)


def _split_ref(o, x, fc1, lw, lb, eps, fc2, fault=None):
    """SplitAttn + residual in float64 and its bound.  o (N,H,W,3C), x (N,H,W,C); fc1 (C,C), fc2 (3C,C) as nn.Linear
    weights.  Returns out, bound (N,H,W,C)."""
    N, H, W, C = x.shape
    HW = H * W
    br = o.reshape(N, HW, 3, C)
    denom = 32 * math.ceil(HW / 32) if fault == "hw_slab" else HW
    gap = br.sum((1, 2)) / denom
    G = br.abs().sum((1, 2)) / HW
    y, Y = gap @ fc1.t(), G @ fc1.abs().t()
    mu = y.mean(-1, keepdim=True)
    sig = torch.sqrt(((y - mu) ** 2).mean(-1, keepdim=True) + eps)
    yh = (y - mu) / sig
    r = yh * lw + lb
    rho = torch.relu(r)
    z = (rho @ fc2.t()).reshape(N, 3, C)
    g = torch.softmax(z, -1 if fault == "gate_channels" else 1)
    out = (br * g[:, None]).sum(2) + x.reshape(N, HW, C)
    dyh = (Y + Y.mean(-1, keepdim=True) + yh.abs() * (yh.abs() * Y).mean(-1, keepdim=True)) / sig + yh.abs()
    dz = ((lw.abs() * dyh + r.abs() + rho) @ fc2.abs().t()).reshape(N, 3, C)
    dg = g * (dz + (g * dz).sum(1, keepdim=True)) + g
    bound = ALPHA * ((br.abs() * (dg + g)[:, None]).sum(2) + x.abs().reshape(N, HW, C)) + REL * out.abs()
    return out.reshape(N, H, W, C), bound.reshape(N, H, W, C)


def _sttf_taps(theta, H, W, align=True):
    """Taps and fp32 bilinear weights of k_sttf_resample: PyTorch's fp32 F.affine_grid, ix = (gx + 1) * ((W - 1) / 2) in fp32
    (align_corners=True; ((gx + 1) W - 1) / 2 without), floor, weights (fx + 1 - ix, ix - fx) and their products in fp32.
    Returns idx (n,4,HW) (-1 off the map) and w (n,4,HW) float64 (0 off the map)."""
    n = theta.shape[0]
    grid = F.affine_grid(theta.float(), [n, 1, H, W], align_corners=align).reshape(n, H * W, 2)
    gx, gy = grid[..., 0], grid[..., 1]
    if align:
        ix, iy = (gx + 1) * np.float32((W - 1) * 0.5), (gy + 1) * np.float32((H - 1) * 0.5)
    else:
        ix, iy = ((gx + 1) * W - 1) / 2, ((gy + 1) * H - 1) / 2
    fx, fy = ix.floor(), iy.floor()
    wx, wy = ((fx + 1) - ix, ix - fx), ((fy + 1) - iy, iy - fy)
    idx, w = [], []
    for dy, dx in ((0, 0), (0, 1), (1, 0), (1, 1)):
        xi, yi = fx + dx, fy + dy
        ok = (xi >= 0) & (xi < W) & (yi >= 0) & (yi < H)
        idx.append(torch.where(ok, yi.clamp(0, H - 1).long() * W + xi.clamp(0, W - 1).long(), -1))
        w.append(torch.where(ok, wx[dx] * wy[dy], 0.0).double())
    return torch.stack(idx, 1), torch.stack(w, 1)


def _sttf_ref(src, theta, fault=None):
    """src (n,H,W,C) float64, theta (n,2,3) fp32 -> y, A = sum_t w_t |v_t| (n,H,W,C)."""
    n, H, W, C = src.shape
    idx, w = _sttf_taps(theta, H, W, align=fault != "align")
    X = src.reshape(n, H * W, C)
    y, A = torch.zeros_like(X), torch.zeros_like(X)
    for t in range(4):
        v = torch.gather(X, 1, idx[:, t].clamp_min(0).unsqueeze(-1).expand(-1, -1, C))
        y += w[:, t].unsqueeze(-1) * v
        A += w[:, t].unsqueeze(-1) * v.abs()
    return y.reshape(n, H, W, C), A.reshape(n, H, W, C)


def _reference(case, inp, vals, fault=None):
    """float64 output (N,H,W,C) and its bound for one case.  vals: the float64 value of each activation input the kernel
    reads.  `fault` restates a plausible kernel bug (test_bound_rejects_plausible_kernel_bugs)."""
    p, k = case.p, case.kernel
    if k == "window":
        o, t1, t2 = _window_ref(vals["qkv"], p["heads"], p["dh"], p["ws"], inp["bias"].double(), fault, p["special"])
        a_s, a_p = (WIN_BF16_S, WIN_BF16_P) if case.fmt == "bf16" else (WIN_SPLIT, WIN_SPLIT)
        return o, a_s * t1 + a_p * t2 + REL * o.abs()
    if k == "cav":
        o, t1, t2 = _cav_ref(vals["qkv"], p["rl"], p["ego_only"], fault)
        return o, ALPHA * (t1 + t2) + REL * o.abs()
    if k == "swap":
        o, t1, t2 = _swap_ref(vals["qkv"], p["rl"], p["L"], p["w"], p["grid"], inp["bias"].double(), fault)
        return o, ALPHA * (t1 + t2) + REL * o.abs()
    if k == "split":
        d = {s: inp[s].double() for s in ("fc1", "fc2", "lw", "lb")}
        return _split_ref(vals["o"], vals["x"], d["fc1"], d["lw"], d["lb"], inp["eps"], d["fc2"], fault)
    y, A = _sttf_ref(vals["src"], inp["theta"], fault)
    return y, ALPHA * A + REL * y.abs()


# ------------------------------------------------------------------------------------------------ the bound is sharp (CPU)
def _faults(case):
    p, k = case.p, case.kernel
    f = ["lo"] if case.fmt == "split" else []
    if k == "window" and p["special"] != "zero_q":          # zero q and bias: every score is 0
        f.append("bias_t")
        if p["ws"] * p["ws"] > KC and p["special"] != "first":     # with a dominant first key later chunks weigh e^-30
            f += ["skip_rescale", "drop_last"]
    elif k == "cav":
        if len(p["rl"]) > 1:
            f.append("image_of")
        if len(p["rl"]) > CAV_SCENES and not p["ego_only"]:
            f.append("restart")
    elif k == "swap":
        if p["L"] * p["w"] ** 2 > 1:
            f.append("bias_t")
        if any(r < p["L"] for r in p["rl"]):
            f.append("pad_keys")
        if p["w"] > 1:
            f.append("mode")
    elif k == "split":
        f.append("gate_channels")
        if (p["H"] * p["W"]) % 32 and p["small"]:
            f.append("hw_slab")
        if p["xfmt"] == "split" and "lo" not in f:
            f.append("lo")
    elif k == "sttf" and min(p["H"], p["W"]) > 1:
        f.append("align")
    return f


def _ratio(got, y, bound):
    err = (got - y).abs()
    return torch.where(err == 0, 0.0, err / bound).nan_to_num(nan=math.inf).max().item()


@pytest.mark.parametrize("name", list(CASE))
def test_bound_rejects_plausible_kernel_bugs(name):
    """Each plausible kernel bug, restated on the float64 reference of the case, leaves the bound on some element: the lo
    plane of split input ignored; window attention with the bias read transposed (key-major instead of query-major), the last
    online-softmax chunk's rescale skipped, or the last chunk dropped; cav attention with image_of off by one scene, or each
    launch restarting the scene table's image counter; swap attention with the bias read query-major, padded agents' keys
    included, or window and grid token orders swapped; the split-attention gate softmaxed over channels instead of branches,
    or the pooled sum divided by HW rounded up to the 32 slabs; STTF with align_corners off."""
    case = CASE[name]
    inp = INPUTS[case.kernel](case)
    st = _storage(case, inp)
    vals = {s: _value(t, _fmt_of(case, s)) for s, t in st.items()}
    y, bound = _reference(case, inp, vals)
    assert bool(torch.isfinite(y).all()) and bool((bound > 0).any())
    faults = _faults(case)
    if not faults:
        pytest.skip("no plausible bug applies to this case's shape")
    for fault in faults:
        v = {s: _value(t, _fmt_of(case, s), drop_lo=True) for s, t in st.items()} if fault == "lo" else vals
        yf = _reference(case, inp, v, fault)[0]
        ratio = _ratio(yf, y, bound)
        assert ratio > 1, f"{name}: the bound does not reject '{fault}' (max err / bound {ratio:.3f})"


def test_every_fault_is_exercised_and_every_instantiation_has_a_case():
    """Each simulated bug applies to at least one case, and the cases together reach every instantiation the dispatch can
    launch (the names in the case ids)."""
    faults = {f for c in CASES for f in _faults(c)}
    assert faults == {"lo", "bias_t", "skip_rescale", "drop_last", "image_of", "restart", "pad_keys", "mode",
                      "gate_channels", "hw_slab", "align"}
    reached = {r for c in CASES for r in c.reaches}
    assert reached == REACHABLE, sorted(REACHABLE - reached)
    for c in CASES:
        assert c.reaches[0].split("<")[0] in c.name.replace("+gate+combine", "")


def test_reference_matches_the_modules():
    """The float64 restatements above agree in float64 with the functional restatements of the reference's modules in oracle/
    (pinned against the unmodified reference by its goldens), fed the package's own parameter containers:
    mswin.BaseWindowAttention (dense_bias, the scale folded into q), hmsa.HGTCavAttention with agent types 0 (relation_att[0]
    and relation_msg[0] folded into q and v as V2XViTFusion does), split_attn.SplitAttn plus the residual,
    swap_fusion_modules.Attention with CoBEVT's agent mask (key-major bias as CoBEVT builds it), and the STTF warp_affine
    chain (fp32 grid_sample, so to fp32 rounding)."""
    from heal_b200.models.fuse_modules.swap_fusion_modules import Attention
    from heal_b200.models.sub_modules.hmsa import HGTCavAttention
    from heal_b200.models.sub_modules.mswin import BaseWindowAttention
    from heal_b200.models.sub_modules.split_attn import SplitAttn
    from oracle import cobevt as cb, v2xvit as vx
    torch.manual_seed(3)
    g = torch.Generator().manual_seed(5)

    def close(a, b, what):
        err = (a - b).abs().max().item()
        assert err <= 1e-12 * max(1.0, b.abs().max().item()), f"{what}: {err:.3e}"

    # window attention
    for heads, dh, ws in ((16, 16, 4), (8, 32, 8), (2, 64, 16)):
        inner = heads * dh
        m = BaseWindowAttention(inner, heads, dh, 0.0, ws, True).double()
        with torch.no_grad():
            m.to_out[0].weight.copy_(torch.eye(inner))
            m.to_out[0].bias.zero_()
        sd = {"a." + k: v for k, v in m.state_dict().items()}
        x = torch.randn(1, 2, 2 * ws, 3 * ws, inner, generator=g, dtype=torch.float64)
        ref = vx.base_window_attention(x, sd, "a", heads, dh, ws)[0]
        w = m.to_qkv.weight.detach()
        qkv = F.linear(x[0], torch.cat([w[:inner] * m.scale, w[inner:]]))
        close(_window_ref(qkv, heads, dh, ws, m.dense_bias())[0], ref, f"window {heads}/{dh}/{ws}")

    # cav attention: two scenes of 3 and 1 agents in 3 slots
    C, heads, rl, L = 64, 2, [3, 1], 3
    m = HGTCavAttention(C, heads, dim_head=32).double()
    with torch.no_grad():
        m.a_linears[0].weight.copy_(torch.eye(C))
        m.a_linears[0].bias.zero_()
    sd = {"h." + k: v for k, v in m.state_dict().items()}
    x = torch.randn(2, L, 3, 5, C, generator=g, dtype=torch.float64)
    mask = torch.zeros(2, 3, 5, 1, L, dtype=torch.float64)
    for b, n in enumerate(rl):
        mask[b, ..., :n] = 1
    ref = vx.hgt_cav_attention(x, mask, torch.zeros(2, L, dtype=torch.long), sd, "h", heads, 32)
    imgs = [x[b, 0] for b in range(2)] + [x[b, i] for b, n in enumerate(rl) for i in range(1, n)]
    lin = lambda t, s: F.linear(t, sd[f"h.{s}_linears.0.weight"], sd[f"h.{s}_linears.0.bias"])
    X = torch.stack(imgs)
    q, k, v = (lin(X, s).reshape(*X.shape[:3], heads, 32) for s in ("q", "k", "v"))
    q = torch.einsum("nhwmp,mpq->nhwmq", q, m.relation_att.detach()[0]) * m.scale
    v = torch.einsum("nhwmp,mpc->nhwmc", v, m.relation_msg.detach()[0])
    got = _cav_ref(torch.cat([t.reshape(*X.shape[:3], C) for t in (q, k, v)], -1), rl, False)[0]
    close(got[[0, 2, 3]], ref[0], "cav scene 0")
    close(got[1], ref[1, 0], "cav scene 1")

    # SplitAttn + residual
    m = SplitAttn(256).double()
    with torch.no_grad():
        m.bn1.weight.uniform_(0.5, 1.5)
        m.bn1.bias.normal_()
    sd = {"s." + k: v for k, v in m.state_dict().items()}
    wl = [torch.randn(2, 1, 3, 7, 256, generator=g, dtype=torch.float64) for _ in range(3)]
    xr = torch.randn(2, 1, 3, 7, 256, generator=g, dtype=torch.float64)
    ref = vx.split_attn(wl, sd, "s") + xr
    got = _split_ref(torch.cat([t[:, 0] for t in wl], -1), xr[:, 0], m.fc1.weight.detach(), m.bn1.weight.detach(),
                     m.bn1.bias.detach(), m.bn1.eps, m.fc2.weight.detach())[0]
    close(got, ref[:, 0], "split_attn")

    # CoBEVT window and grid attention: scenes of 3 and 1 agents in 3 slots
    C, L, w, rl = 64, 3, 2, [3, 1]
    m = Attention(C, 32, 0.0, L, w).double()
    with torch.no_grad():
        m.to_out[0].weight.copy_(torch.eye(C))
    sd = {"a." + k: v for k, v in m.state_dict().items()}
    bias = m.relative_position_bias_table.weight.detach()[m.relative_position_index].permute(2, 1, 0)   # key-major
    x = torch.randn(2, L, 6, 8, C, generator=g, dtype=torch.float64)
    wq = m.to_qkv.weight.detach()
    qkv = F.linear(x.reshape(2 * L, 6, 8, C), torch.cat([wq[:C] * m.scale, wq[C:]]))
    for grid in (False, True):
        X, Y = 6 // w, 8 // w
        if grid:      # 'b m (w1 x) (w2 y) d -> b m x y w1 w2 d'
            xt = x.reshape(2, L, w, X, w, Y, C).permute(0, 1, 3, 5, 2, 4, 6)
        else:         # 'b m (x w1) (y w2) d -> b m x y w1 w2 d'
            xt = x.reshape(2, L, X, w, Y, w, C).permute(0, 1, 2, 4, 3, 5, 6)
        mask = torch.zeros(2, X, Y, w, w, 1, L, dtype=torch.float64)
        for b, n in enumerate(rl):
            mask[b, ..., :n] = 1
        ref = cb.attention(xt, sd, "a", 32, L, w, mask)                    # (b, l, x, y, w1, w2, d)
        ref = ref.permute(0, 1, 4, 2, 5, 3, 6) if grid else ref.permute(0, 1, 2, 4, 3, 5, 6)
        close(_swap_ref(qkv, rl, L, w, grid, bias)[0], ref.reshape(2 * L, 6, 8, C), f"swap grid={grid}")

    # STTF: the reference's warp_affine chain (fp32 affine_grid and grid_sample) against _sttf_ref on the same theta
    H, W = 20, 36
    src = torch.randn(3, 8, H, W, generator=g)
    M = vx.sttf_matrix(torch.eye(4).expand(1, 4, 4, 4), H, W, 0.4, 4)
    c, s = math.cos(0.3), math.sin(0.3)
    M[1] = torch.tensor([[c, -s, 2.5], [s, c, -1.25]])
    M[2] = torch.tensor([[c, s, -3.75], [-s, c, 0.6]])
    ref = vx.warp_affine(src, M, (H, W))
    theta = vx.warp_affine_matrix(M, (H, W), (H, W)).float().contiguous()
    y, A = _sttf_ref(src.permute(0, 2, 3, 1).double(), theta)
    ratio = ((y.permute(0, 3, 1, 2) - ref.double()).abs() / (2.0 ** -21 * A.permute(0, 3, 1, 2) + 1e-30)).max().item()
    assert ratio <= 1, f"sttf: F.grid_sample differs from _sttf_ref by {ratio:.3f} x 2^-21 A"


def test_split_attn_refuses_more_than_65535_images():
    """heal_split_attn launches with gridDim.y = n_img: 65536 images are refused with HEAL_ERR_UNSUPPORTED before the
    workspace size is looked at and before anything is launched (a 256-byte workspace; the pointers are never read)."""
    from heal_b200._lib import HealAct, lib
    fake = 1 << 20                                                    # 16-byte aligned, never dereferenced
    o, x, out = HealAct(fake, 0, 768, 0, 0), HealAct(fake, 0, 256, 0, 0), HealAct(fake, 0, 256, 0, 0)
    vp = ctypes.c_void_p
    before = lib.heal_launch_count()
    code = lib.heal_split_attn(ctypes.byref(o), ctypes.byref(x), 65536, 1, 1, 256, vp(fake), vp(fake), vp(fake), 1e-5, vp(fake), vp(fake), 256,
                               ctypes.byref(out), vp(0))
    assert code == -4, f"heal_split_attn(n_img = 65536) returned {code}, expected HEAL_ERR_UNSUPPORTED (-4)"
    assert lib.heal_launch_count() == before


# ------------------------------------------------------------------------------------------------ the kernels (GPU)
def _put(st, sl):
    """A CUDA buffer holding storage tensor `st` in channels [coff, coff + C) and SENTINEL elsewhere (lo plane 0), the view of
    the slice, and the channel offset."""
    width, coff = sl or (st.shape[-1], 0)
    buf = torch.full(st.shape[:-1] + (width,), SENTINEL, dtype=st.dtype)
    if st.dtype == torch.bfloat16 and st.shape[0] == 2:
        buf[1] = 0
    buf[..., coff:coff + st.shape[-1]] = st
    buf = buf.cuda()
    return buf, buf[..., coff:coff + st.shape[-1]], coff


def _out_buffer(N, H, W, width, fmt, sliced):
    fill = SENTINEL if sliced else float("nan")
    if fmt == "f32":
        return torch.full((N, H, W, width), fill, dtype=torch.float32, device="cuda")
    buf = torch.full((2 if fmt == "split" else 1, N, H, W, width), fill, dtype=torch.bfloat16, device="cuda")
    if fmt == "split" and sliced:
        buf[1] = 0
    return buf


def _launch(case, inp, st, runs=(("A", "f32"), ("B", None))):
    """Runs the case's kernels with fp32 output (A) and in the input's format (B).  Returns the input buffers (with the
    slice offsets) and the output buffers."""
    from heal_b200 import ops
    p, k = case.p, case.kernel
    bufs = {}
    for i, (s, t) in enumerate(st.items()):
        bufs[s] = _put(t, case.in_slice if i == 0 else None)
    acts = {s: ops.Act(v, _fmt_of(case, s)) for s, (_, v, _) in bufs.items()}
    if k == "window":
        N, H, W, cout = p["N"], p["H"], p["W"], p["heads"] * p["dh"]
    elif k == "cav":
        N, H, W, cout = len(p["rl"]) if p["ego_only"] else sum(p["rl"]), p["H"], p["W"], p["C"]
    elif k == "swap":
        N, H, W, cout = len(p["rl"]) * p["L"], p["H"], p["W"], p["C"]
    elif k == "split":
        N, H, W, cout = p["N"], p["H"], p["W"], 256
    else:
        N, H, W, cout = len(p["thetas"]), p["H"], p["W"], p["C"]
    width, oco = case.out_slice or (cout, 0)
    outs = {}
    for run, fmt in runs:
        fmt = fmt or case.fmt
        buf = _out_buffer(N, H, W, width, fmt, case.out_slice is not None)
        view = ops.Act(buf[..., oco:oco + cout], fmt)
        if k == "window":
            whole, _, coff = bufs["qkv"]
            ops.window_attention(ops.Act(whole, case.fmt), p["heads"], p["dh"], p["ws"], inp["bias"].cuda(), qkv_coffset=coff,
                                 out=ops.Act(buf, fmt), out_coffset=oco)
        elif k == "cav":
            ops.cav_attention(acts["qkv"], list(p["rl"]), p["ego_only"], out=view)
        elif k == "swap":
            ops.swap_attention(acts["qkv"], list(p["rl"]), p["L"], p["w"], p["grid"], inp["bias"].cuda(), out=view)
        elif k == "split":
            ops.split_attn(acts["o"], acts["x"], inp["fc1"].t().contiguous().cuda(), inp["lw"].cuda(), inp["lb"].cuda(),
                           inp["eps"], inp["fc2"].t().contiguous().cuda(), out=view)
        else:
            ops.sttf_resample(acts["src"], inp["theta"].cuda(), out=view)
        outs[run] = buf
    return bufs, outs, oco, cout


def _bits(t):
    t = t.contiguous()
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASE))
def test_attention_kernel(name):
    case = CASE[name]
    inp = INPUTS[case.kernel](case)
    st = _storage(case, inp)
    runs = (("A", "f32"), ("B", None)) + ((("A2", "f32"),) if case.kernel == "split" else ())
    bufs, outs, oco, cout = _launch(case, inp, st, runs)
    torch.cuda.synchronize()
    # 1. the inputs as the kernel read them (read back from the device); the buffers around an input slice are untouched
    vals = {}
    for s, (whole, _, coff) in bufs.items():
        b = whole.cpu()
        c_in = st[s].shape[-1]
        vals[s] = _value(b[..., coff:coff + c_in], _fmt_of(case, s))
        assert torch.equal(_bits(b[..., coff:coff + c_in]), _bits(st[s])), f"{name}: input {s} changed"
        if b.shape[-1] != c_in:
            around = torch.cat([b[..., :coff].flatten(), b[..., coff + c_in:].flatten()]).double()
            assert bool(((around == SENTINEL) | (around == 0)).all()), f"{name}: the input buffer around the slice changed"
    # 2. run A against float64
    y, bound = _reference(case, inp, vals)
    a_full = outs["A"].cpu()
    a = a_full[..., oco:oco + cout]
    err = (a.double() - y).abs()
    ok = err <= bound
    ratio = _ratio(a.double(), y, bound)
    print(f"{name}: max err / bound {ratio:.4f}  (max err {err.max().item():.3e}, max|y| {y.abs().max().item():.3f})")
    assert bool(ok.all()), f"{name}: {int((~ok).sum())} elements outside the bound, max err / bound {ratio:.3f}"
    if case.kernel == "sttf":
        for j, kind in enumerate(case.p["thetas"]):
            if kind in ("outside", "clamp+", "clamp-"):
                assert bool((a[j] == 0).all()), f"{name}: image {j} ({kind}) samples nothing but is not 0"
    if case.kernel == "split":
        assert torch.equal(_bits(outs["A2"].cpu()), _bits(a_full)), f"{name}: a second run differs"
    # 3. run B is the rounding of run A
    b_full = outs["B"].cpu()
    b = b_full[..., oco:oco + cout]
    if case.fmt == "f32":
        assert torch.equal(_bits(b), _bits(a)), f"{name}: the two fp32 runs differ"
    else:
        hi = a.to(torch.bfloat16)
        assert torch.equal(_bits(b[0]), _bits(hi)), f"{name}: hi plane != bf16(fp32 output)"
        if case.fmt == "split":
            assert torch.equal(_bits(b[1]), _bits((a - hi.float()).to(torch.bfloat16))), f"{name}: lo plane != bf16(fp32 - hi)"
    # 4. the channels around an output slice keep their sentinel
    if case.out_slice:
        for run, t in (("A", a_full), ("B", b_full)):
            v = t.double() if t.dtype == torch.float32 else t[0].double()
            around = torch.cat([v[..., :oco].flatten(), v[..., oco + cout:].flatten()])
            assert bool((around == SENTINEL).all()), f"{name} run {run}: a write spilled out of channels [{oco}, {oco + cout})"
            if case.fmt == "split" and run == "B":
                lo = torch.cat([t[1][..., :oco].flatten(), t[1][..., oco + cout:].flatten()])
                assert bool((lo == 0).all()), f"{name}: a lo-plane write spilled out of the slice"


@pytest.mark.gpu
def test_swap_attention_checks_every_count_before_launching():
    """65 scenes need two launches; a bad count in the 65th (0, or more than L) must raise before the first launch and leave
    the output as it was."""
    from heal_b200 import ops
    from heal_b200._lib import lib
    L = 2
    qkv = ops.Act(torch.ones(65 * L, 4, 4, 3 * 32, device="cuda"), "f32")
    bias = torch.zeros(1, L * 4, L * 4, device="cuda")
    for bad in (0, L + 1):
        out = ops.Act(torch.full((65 * L, 4, 4, 32), 7.0, device="cuda"), "f32")
        before = lib.heal_launch_count()
        with pytest.raises(RuntimeError, match="HEAL_ERR_ARG"):
            ops.swap_attention(qkv, [1] * 64 + [bad], L, 2, False, bias, out=out)
        torch.cuda.synchronize()
        assert lib.heal_launch_count() == before
        assert bool((out.t == 7.0).all()), f"count {bad}: the output changed"


def _misaligned_call(kernel, where, fmt):
    """One call of `kernel` whose activation input (where='in') or output (where='out') view starts one element past a
    16-byte boundary (channel 1 of a buffer whose pixel stride is a multiple of 4).  Every other argument is well formed."""
    from heal_b200 import ops
    H, W = 4, 8

    def act(N, c, bad):
        t = torch.zeros((N, H, W, c + 4)) if fmt == "f32" else torch.zeros((1, N, H, W, c + 4), dtype=torch.bfloat16)
        t = t.cuda()
        return ops.Act(t[..., 1:1 + c] if bad else t[..., :c], fmt)

    bi, bo = where == "in", where == "out"
    if kernel == "window":
        bias = torch.zeros(16, 16, device="cuda")
        return lambda: ops.window_attention(act(1, 3 * 32, bi), 2, 16, 4, bias, out=act(1, 32, bo))
    if kernel == "cav":
        return lambda: ops.cav_attention(act(3, 3 * 64, bi), [2, 1], False, out=act(3, 64, bo))
    if kernel == "swap":
        bias = torch.zeros(2, 8, 8, device="cuda")
        return lambda: ops.swap_attention(act(4, 3 * 64, bi), [2, 1], 2, 2, False, bias, out=act(4, 64, bo))
    if kernel == "split":
        C = 256
        return lambda: ops.split_attn(act(1, 3 * C, bi), act(1, C, False), torch.zeros(C, C, device="cuda"),
                                      torch.ones(C, device="cuda"), torch.zeros(C, device="cuda"), 1e-5,
                                      torch.zeros(C, 3 * C, device="cuda"), out=act(1, C, bo))
    th = torch.tensor([[[1.0, 0.0, 0.0], [0.0, 1.0, 0.0]]] * 2, device="cuda")
    return lambda: ops.sttf_resample(act(2, 32, bi), th, out=act(2, 32, bo))


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["f32", "bf16"])
@pytest.mark.parametrize("where", ["in", "out"])
@pytest.mark.parametrize("kernel", ["window", "cav", "swap", "split", "sttf"])
def test_misaligned_view_is_refused(kernel, where, fmt):
    """A qkv (or input) or output view whose data pointer is one element past a 16-byte boundary is refused
    (HEAL_ERR_UNSUPPORTED -> RuntimeError) and nothing is launched: the kernels' paired and 4-channel vector accesses could
    not use it."""
    from heal_b200._lib import lib
    call = _misaligned_call(kernel, where, fmt)
    torch.cuda.synchronize()
    before = lib.heal_launch_count()
    with pytest.raises(RuntimeError, match="HEAL_ERR_UNSUPPORTED"):
        call()
    torch.cuda.synchronize()
    assert lib.heal_launch_count() == before
