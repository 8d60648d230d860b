"""The fusion kernels of csrc/fuse.cu against a float64 reference, one case per kernel instantiation the dispatch can reach.

heal_pyramid_fuse_level (k_pyramid_fuse<FUSE_PIX>, k_pyramid_fuse_split8<FUSE_PIX>), heal_att_fuse (k_att_fuse<Q>,
k_att_fuse_split8<NA>), heal_max_fuse, heal_warp_affine, heal_v2v_aggregate and heal_gru_gate.  Every case runs its kernel
twice: with fp32 output (run A) and with the product's output format, the format of the input (run B).  The checks:
  - A is within a per-element bound of a float64 reference computed on the exact input the kernel read (hi + lo for split
    input, the bf16 value for bf16 input);
  - B is bit for bit the rounding of A: bf16(A); for split, hi = bf16(A) and lo = bf16(A - hi); for fp32, A itself;
  - the channels around an output slice (out_coffset, or an `out=` view into a wider buffer) and around an input slice keep
    their sentinel, and a pixel where every agent is masked comes out exactly 0.

Reference geometry.  warp_affine_simple is F.affine_grid on the fp64 theta, the grid cast to fp32, then F.grid_sample: taps
and bilinear weights are decided in fp32.  The reference does the same (fp64 affine_grid, the grid cast to fp32, fp32 ix / iy,
floor and weights wx * wy) and then works in float64: sigmoid, the warped sums, softmax, the weighted sums, tanh.
grid_sample rounds the unnormalisation ((gx + 1) W - 1) / 2 once (its (gx + 1) * W - 1 compiles to an FMA, as it does in the
kernels), so _taps evaluates it exactly in float64 and rounds once; test_reference_taps_follow_grid_sample pins that.
oracle/nets.warp_affine_simple casts the grid to the input's dtype, so fed float64 it would compute other taps; _taps and
_sample below are the fp32-taps / float64-arithmetic form of it.
  The masked softmax of PyramidFusion is discontinuous where a warped score is exactly 0, and a tap changes where ix or iy
crosses an integer.  The kernels evaluate theta . (xb, yb, 1) in fp64 in their own order, affine_grid in another; the two
can differ in the last fp64 bit and then, rarely, cast to neighbouring fp32 values.  So generic poses keep every tap
coordinate at least MIN_FRAC px from an integer (asserted for every case): there such a one-ulp shift keeps the taps and the
zero weights and moves the result by a first-order amount inside the bound.  Exact edges are tested separately: whole-pixel
translations and quarter / half turns on power-of-two maps with align_corners off, where every fp32 and fp64 step is exact
and every tap lands on a pixel centre.

The bound is first order in the reference's own quantities.  With a_j the softmax weights, w_jk the fp32 tap weights, x_jk the
sampled values, Xw_j = sum_k w_jk x_jk the warped feature and A_j = sum_k w_jk |x_jk| the warp of |x|:
  pyramid  |err| <= ALPHA sum_j a_j A_j + REL |y|.  Each warped feature carries a relative error of a few 2^-24 of A_j (fp32
           FMAs over four taps, the sum over agents, the one-ulp shift of ix); the weights a_j carry a few 2^-24 from the fp32
           sigmoid, warped score and softmax, which moves y by at most sum_j a_j |Xw_j| <= sum_j a_j A_j times that.
  att      the same plus the softmax's sensitivity to the scores d_j = Xw_0 . Xw_j / sqrt(C): da_j = a_j (dd_j - sum_k a_k dd_k)
           and |dd_j| <= ALPHA D_j with D_j = A_0 . A_j / sqrt(C), so
           |err| <= ALPHA [sum_j a_j A_j + sum_j a_j |Xw_j| (D_j + sum_k a_k D_k)] + REL |y|.
  max      |err| <= ALPHA max_j A_j + REL |y| (the max is 1-Lipschitz);   warp  |err| <= ALPHA A + REL |y|.
  v2v      element-wise: |err| <= ALPHA (agg_j m_j (|q_j| + |p|) + |x|) + REL |y|, agg the mean or max over the neighbours,
           m_j the summed in-bounds tap weights, |x| only when the output is x + agg (the [x | agg] copy of x is exact).
  gru_gate element-wise: |err| <= (ALPHA + REL) |y|: expf, the add, the division, tanhf and the product each contribute a
           relative error of a few 2^-24.
REL = 2^-22 covers the final fp32 rounding.  test_bound_rejects_plausible_kernel_bugs (no GPU) shows that the bound rejects
each plausible kernel bug on these cases.

Calibration, on an H100 80GB HBM3 at a 400 W power limit: largest err / bound per case at ALPHA = 2^-20 (a ratio of 0 means
the output was exact)
  pyramid  split_c64_n5 0.229, split_c128_n3_align 0.174, split_c256_n6_rows 0.166, split_c32_n1 0.089,
           split_c128_n8_gathered 0.144, split_edges 0.161, split_c36 0.147, split_slice4 0.168, bf16_c64_n5_masked 0.156,
           bf16_c128_n6_rows_last 0.134, bf16_c256_n3_align 0.199, bf16_c512_n1 0.093, f32_c128_n8_gathered 0.182,
           f32_c32_n6_rows_last 0.147, f32_c384_n3_align 0.166, f32_edges 0.172
  att      split_c256_n5 0.125, split_c128_n8 0.115, split_c128_n3_slice4 0.111, split_c512_n3 0.117, f32_c128_n1 0.072,
           bf16_c256_n6 0.109, f32_c384_n3 0.103, bf16_c512_n8 0.092, f32_edges 0.083
  max      f32_n4 0.133, bf16_n3 0.079, split_n6 0.118, bf16_edges 0
  warp     f32 0.121, bf16 0.148, split 0.160, split_edges 0
  v2v      split_mean_gru 0.140, bf16_max_gru 0.086, f32_mean 0.127, split_max 0.100
  gru      split 0.243, bf16 0.208, f32 0.248
so ALPHA = 2^-20 leaves 4x of headroom over the largest (gru_f32)."""
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

# Calibrated on an H100 80GB HBM3 at a 400 W power limit: the largest err / bound of any case was 0.248 (gru_f32), so these
# kernels need ALPHA >= 2^-22; 2^-20 leaves 4x of headroom.  The module docstring lists every case; test_fuse_kernel prints them.
ALPHA = 2.0 ** -20
REL = 2.0 ** -22
MIN_FRAC = 1e-3            # least distance of a generic tap coordinate from an integer, in pixels
SENTINEL = -1000.0         # finite and exact in bf16: fills the channels around a slice

# Exact rotations in pixel space (entries multiples of 1/5).  Rotating about the map centre (W-1)/2, (H-1)/2, a pixel lands on
# a multiple of 1/10 plus the pose's translation, so translations of k + 0.35 (x) and k + 0.65 (y) keep every tap coordinate
# 0.05 px from an integer.
ROT = [((1.0, 0.0), (0.0, 1.0)), ((0.6, -0.8), (0.8, 0.6)), ((-0.8, -0.6), (0.6, -0.8)), ((0.0, 1.0), (-1.0, 0.0)),
       ((-1.0, 0.0), (0.0, -1.0)), ((0.8, 0.6), (-0.6, 0.8)), ((-0.6, 0.8), (-0.8, -0.6))]
# exact edges: identity, whole-pixel shifts, a quarter and a half turn
EDGE_POSES = [(ROT[0], (0, 0)), (ROT[0], (3, -2)), (ROT[3], (1, 2)), (ROT[4], (-2, 1))]


@dataclass(frozen=True)
class Case:
    name: str
    kernel: str                                   # pyramid | att | max | warp | v2v | gru
    fmt: str                                      # input storage format: f32 | bf16 | split
    n: int                                        # agents (pyramid, att, max), output images (warp), neighbours (v2v), images (gru)
    C: int
    H: int
    W: int
    reaches: Tuple[str, ...]                      # the instantiations runs A and B launch
    align: bool = False                           # align_corners (pyramid only; the others are align_corners=False)
    edges: bool = False                           # EDGE_POSES instead of generic poses
    out_of_view: Tuple[int, ...] = ()             # agents / images translated fully outside the map
    crop: Optional[Tuple[Tuple[int, int, int, int], ...]] = None   # per agent (h0, h1, w0, w1) in eighths of H and W
    rows: Optional[Tuple[int, int]] = None        # (row0, rows) output slab; row0 < 0 counts from the last row
    gathered: bool = False                        # agents in a shuffled order with gaps in one buffer (agent offsets)
    in_slice: Optional[Tuple[int, int]] = None    # (buffer width, channel offset) the input is read from
    out_slice: Optional[Tuple[int, int]] = None   # (buffer width, channel offset) the output is written to
    agg_max: bool = False                         # v2v: max instead of mean
    gru: bool = True                              # v2v: output [x | agg] (the GRU conv input) instead of x + agg
    all_masked: bool = False                      # some pixels have every agent masked (asserted)


FULL = (0, 8, 0, 8)
CASES = [
    # ---- heal_pyramid_fuse_level.  Split input (tc32, C2's three levels): the 8-channel kernel
    Case("pyr_split_c64_n5", "pyramid", "split", 5, 64, 33, 47, ("k_pyramid_fuse_split8<32>",), out_of_view=(4,),
         crop=(FULL, FULL, (1, 7, 2, 8), FULL, FULL)),
    Case("pyr_split_c128_n3_align", "pyramid", "split", 3, 128, 17, 25, ("k_pyramid_fuse_split8<16>",), align=True,
         out_slice=(192, 32)),
    Case("pyr_split_c256_n6_rows", "pyramid", "split", 6, 256, 19, 21, ("k_pyramid_fuse_split8<8>",), rows=(5, 7),
         out_of_view=(2,)),
    Case("pyr_split_c32_n1", "pyramid", "split", 1, 32, 15, 17, ("k_pyramid_fuse_split8<32>",), crop=((1, 6, 2, 7),)),
    Case("pyr_split_c128_n8_gathered", "pyramid", "split", 8, 128, 11, 13, ("k_pyramid_fuse_split8<16>",), gathered=True,
         out_of_view=(7,)),
    Case("pyr_split_edges", "pyramid", "split", 4, 128, 16, 32, ("k_pyramid_fuse_split8<16>",), edges=True,
         crop=(FULL, (2, 6, 1, 5), FULL, (0, 4, 4, 8))),
    # split input the 8-channel kernel must not take: C % 8 != 0, and a view at channel 4 (an 8-byte aligned pointer)
    Case("pyr_split_c36", "pyramid", "split", 3, 36, 13, 19, ("k_pyramid_fuse<32>",), out_of_view=(1,)),
    Case("pyr_split_slice4", "pyramid", "split", 3, 64, 13, 19, ("k_pyramid_fuse<16>",), in_slice=(72, 4),
         crop=((1, 7, 1, 7), FULL, FULL)),
    # bf16 input (C4 and the 'bf16' mode): the generic kernel
    Case("pyr_bf16_c64_n5_masked", "pyramid", "bf16", 5, 64, 21, 27, ("k_pyramid_fuse<16>",), out_of_view=(3, 4),
         crop=((2, 6, 2, 6), (0, 4, 0, 8), (4, 8, 0, 8), FULL, FULL), all_masked=True),
    Case("pyr_bf16_c128_n6_rows_last", "pyramid", "bf16", 6, 128, 13, 17, ("k_pyramid_fuse<8>",), rows=(-3, 3),
         out_of_view=(5,)),
    Case("pyr_bf16_c256_n3_align", "pyramid", "bf16", 3, 256, 15, 19, ("k_pyramid_fuse<4>",), align=True,
         out_slice=(320, 32)),
    Case("pyr_bf16_c512_n1", "pyramid", "bf16", 1, 512, 9, 11, ("k_pyramid_fuse<4>",), crop=((0, 5, 3, 8),)),
    # fp32 input
    Case("pyr_f32_c128_n8_gathered", "pyramid", "f32", 8, 128, 13, 15, ("k_pyramid_fuse<8>",), gathered=True,
         crop=((1, 7, 1, 7),) + (FULL,) * 7),
    Case("pyr_f32_c32_n6_rows_last", "pyramid", "f32", 6, 32, 17, 23, ("k_pyramid_fuse<32>",), rows=(-4, 4),
         out_of_view=(1,)),
    Case("pyr_f32_c384_n3_align", "pyramid", "f32", 3, 384, 9, 13, ("k_pyramid_fuse<4>",), align=True, out_slice=(448, 64)),
    Case("pyr_f32_edges", "pyramid", "f32", 4, 64, 16, 32, ("k_pyramid_fuse<16>",), edges=True,
         crop=((0, 8, 2, 6), FULL, (1, 5, 0, 8), FULL), rows=(4, 8)),
    # ---- heal_att_fuse.  Split input with C <= 256 (tc32, C3): the 8-channel kernel, register file sized for <= 5 or 8 agents
    Case("att_split_c256_n5", "att", "split", 5, 256, 15, 21, ("k_att_fuse_split8<5>",), out_of_view=(4,)),
    Case("att_split_c128_n8", "att", "split", 8, 128, 11, 13, ("k_att_fuse_split8<8>",), out_slice=(192, 64)),
    Case("att_split_c128_n3_slice4", "att", "split", 3, 128, 11, 13, ("k_att_fuse<1>",), in_slice=(136, 4)),
    Case("att_split_c512_n3", "att", "split", 3, 512, 7, 9, ("k_att_fuse<4>",)),
    Case("att_f32_c128_n1", "att", "f32", 1, 128, 9, 11, ("k_att_fuse<1>",)),
    Case("att_bf16_c256_n6", "att", "bf16", 6, 256, 11, 13, ("k_att_fuse<2>",), out_slice=(320, 64), out_of_view=(5,)),
    Case("att_f32_c384_n3", "att", "f32", 3, 384, 9, 11, ("k_att_fuse<3>",), in_slice=(392, 8)),
    Case("att_bf16_c512_n8", "att", "bf16", 8, 512, 5, 7, ("k_att_fuse<4>",)),
    Case("att_f32_edges", "att", "f32", 3, 128, 16, 16, ("k_att_fuse<1>",), edges=True),
    # ---- heal_max_fuse (F-Cooper)
    Case("max_f32_n4", "max", "f32", 4, 64, 21, 37, ("k_max_fuse",), out_of_view=(3,)),
    Case("max_bf16_n3", "max", "bf16", 3, 32, 13, 17, ("k_max_fuse",), out_of_view=(2,), out_slice=(48, 8)),
    Case("max_split_n6", "max", "split", 6, 128, 11, 15, ("k_max_fuse",), out_of_view=(1,), in_slice=(136, 4)),
    Case("max_bf16_edges", "max", "bf16", 4, 32, 16, 16, ("k_max_fuse",), edges=True),
    # ---- heal_warp_affine (V2VNet, CoBEVT, V2X-ViT): n output images from 3 source images
    Case("warp_f32", "warp", "f32", 5, 32, 19, 26, ("k_warp_affine",), out_of_view=(3,)),
    Case("warp_bf16", "warp", "bf16", 4, 64, 13, 21, ("k_warp_affine",), out_slice=(96, 16)),
    Case("warp_split", "warp", "split", 6, 128, 11, 13, ("k_warp_affine",), in_slice=(132, 4), out_of_view=(0,)),
    Case("warp_split_edges", "warp", "split", 4, 32, 8, 16, ("k_warp_affine",), edges=True),
    # ---- heal_v2v_aggregate: two updated nodes with n and n - 1 neighbours
    Case("v2v_split_mean_gru", "v2v", "split", 3, 64, 13, 17, ("k_v2v_aggregate",), out_of_view=(1,)),
    Case("v2v_bf16_max_gru", "v2v", "bf16", 5, 32, 11, 15, ("k_v2v_aggregate",), agg_max=True, out_slice=(80, 8)),
    Case("v2v_f32_mean", "v2v", "f32", 2, 128, 9, 11, ("k_v2v_aggregate",), gru=False, in_slice=(136, 4)),
    Case("v2v_split_max", "v2v", "split", 4, 32, 13, 15, ("k_v2v_aggregate",), agg_max=True, gru=False, out_of_view=(2,)),
    # ---- heal_gru_gate: n images of (update gate | candidate), 2C channels
    Case("gru_split", "gru", "split", 2, 64, 13, 17, ("k_gru_gate",)),
    Case("gru_bf16", "gru", "bf16", 1, 128, 9, 11, ("k_gru_gate",), out_slice=(136, 4)),
    Case("gru_f32", "gru", "f32", 3, 32, 11, 13, ("k_gru_gate",), in_slice=(80, 8)),
]
CASE = {c.name: c for c in CASES}

# every instantiation the six launchers can dispatch to
REACHABLE = {"k_pyramid_fuse<4>", "k_pyramid_fuse<8>", "k_pyramid_fuse<16>", "k_pyramid_fuse<32>",
             "k_pyramid_fuse_split8<8>", "k_pyramid_fuse_split8<16>", "k_pyramid_fuse_split8<32>",
             "k_att_fuse<1>", "k_att_fuse<2>", "k_att_fuse<3>", "k_att_fuse<4>", "k_att_fuse_split8<5>", "k_att_fuse_split8<8>",
             "k_max_fuse", "k_warp_affine", "k_v2v_aggregate", "k_gru_gate"}


# ------------------------------------------------------------------------------------------------ inputs
def _norm(size, align):
    """d(normalised coordinate) / d(pixel) of affine_grid / grid_sample."""
    return 2.0 / (size - 1) if align else 2.0 / size


def _theta(H, W, align, R, t):
    """theta of the pixel-space map  source = R (p - c) + c + t  about the map centre c = ((W-1)/2, (H-1)/2), p = (x, y)."""
    aw, ah = _norm(W, align), _norm(H, align)
    return [[R[0][0], R[0][1] * aw / ah, aw * t[0]], [R[1][0] * ah / aw, R[1][1], ah * t[1]]]


def _thetas(case, H, W, count):
    rng = np.random.default_rng(zlib.crc32(f"poses/{case.name}".encode()))
    th = []
    for j in range(count):
        if case.edges:
            R, t = EDGE_POSES[j % len(EDGE_POSES)]
            if j in case.out_of_view:
                t = (t[0] + 3 * W, t[1])
        else:
            R = ROT[0] if j == 0 else ROT[1 + int(rng.integers(len(ROT) - 1))]
            tx, ty = (0, 0) if j == 0 else (int(rng.integers(-(W // 4), W // 4 + 1)), int(rng.integers(-(H // 4), H // 4 + 1)))
            t = (tx + 0.35 + (3 * W if j in case.out_of_view else 0), ty + 0.65)
        th.append(_theta(H, W, case.align, R, t))
    return torch.tensor(th, dtype=torch.float64)


def _crop(case, H, W):
    if case.crop is None:
        return None
    return torch.tensor([[h0 * H // 8, h1 * H // 8, w0 * W // 8, w1 * W // 8] for h0, h1, w0, w1 in case.crop], dtype=torch.int32)


def _v2v_nodes(n):
    """(x image, P image, first pair row, neighbours) of the two updated nodes."""
    return [(1, 0, 0, n), (0, 1, n, max(n - 1, 1))]


def _inputs(case, H=None, W=None):
    """The case's fp32 inputs (channels-last) and geometry, seeded by its name."""
    H, W = H or case.H, W or case.W
    g = torch.Generator().manual_seed(zlib.crc32(case.name.encode()))
    n, C = case.n, case.C
    k = case.kernel
    if k == "pyramid":
        return dict(feat=torch.randn(n, H, W, C, generator=g) * 2, occ=torch.randn(n, H, W, generator=g) * 2,
                    theta=_thetas(case, H, W, n), crop=_crop(case, H, W))
    if k in ("att", "max"):
        # attention on |x| ~ 0.3: scores of order 1, so that the softmax weights spread over the agents
        return dict(feat=torch.randn(n, H, W, C, generator=g) * (0.3 if k == "att" else 1.0), theta=_thetas(case, H, W, n))
    if k == "warp":
        return dict(src=torch.randn(3, H, W, C, generator=g), index=[(2 * i + 1) % 3 for i in range(n)],
                    theta=_thetas(case, H, W, n))
    if k == "v2v":
        nodes = _v2v_nodes(n)
        pairs = sum(nd[3] for nd in nodes)
        return dict(q=torch.randn(pairs, H, W, C, generator=g), p=torch.randn(2, H, W, C, generator=g),
                    x=torch.randn(2, H, W, C, generator=g), nodes=nodes, theta=_thetas(case, H, W, pairs))
    z = torch.randn(n, H, W, C, generator=g) * 3
    c = torch.randn(n, H, W, C, generator=g) * 1.5
    return dict(zc=torch.cat([z, c], -1))


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


INPUT_KEYS = {"pyramid": ("feat",), "att": ("feat",), "max": ("feat",), "warp": ("src",), "v2v": ("q", "p", "x"), "gru": ("zc",)}


# ------------------------------------------------------------------------------------------------ float64 reference
def _taps(theta, H, W, align):
    """fp32 tap geometry of warp_affine_simple for thetas (n,2,3): affine_grid in float64, the grid cast to fp32, then
    grid_sample's unnormalisation (gx + 1 in fp32, then (gx + 1) * W - 1 rounded once, as an FMA does), floor and bilinear
    weights in fp32.  Returns idx (n,4,H*W) the source pixel of the
    (nw, ne, sw, se) taps or -1 off the map, w (n,4,H*W) the fp32 weights as float64 (0 off the map), and ix, iy (n,H*W)."""
    n = theta.shape[0]
    grid = F.affine_grid(theta.double(), [n, 1, H, W], align_corners=align).float().reshape(n, H * W, 2)
    gx, gy = grid[..., 0], grid[..., 1]
    if align:
        ix, iy = (gx + 1) / 2 * (W - 1), (gy + 1) / 2 * (H - 1)
    else:
        # (gx + 1) * W - 1 is exact in float64 (24 + log2(W) bits), so one cast rounds it once
        ix = ((gx + 1).double() * W - 1).float() / 2
        iy = ((gy + 1).double() * H - 1).float() / 2
    x0, y0 = ix.floor(), iy.floor()
    wx, wy = (x0 + 1 - ix, ix - x0), (y0 + 1 - iy, iy - y0)
    idx, w = [], []
    for dy, dx in ((0, 0), (0, 1), (1, 0), (1, 1)):
        xi, yi = x0 + dx, y0 + dy
        ok = (xi >= 0) & (xi < W) & (yi >= 0) & (yi < H)
        idx.append(torch.where(ok, yi.clamp(0, H - 1).long() * W + xi.clamp(0, W - 1).long(), -1))
        w.append(torch.where(ok, wx[dx] * wy[dy], 0.0).double())
    return torch.stack(idx, 1), torch.stack(w, 1), ix, iy


def _geometry(case, theta, H, W, align, check=True):
    idx, w, ix, iy = _taps(theta, H, W, align)
    if check:
        if case.edges:
            assert bool((ix == ix.floor()).all() and (iy == iy.floor()).all()), f"{case.name}: an edge tap is not a pixel centre"
        else:
            frac = torch.cat([ix - ix.round(), iy - iy.round()]).abs().min().item()
            assert frac >= MIN_FRAC, f"{case.name}: a tap coordinate lies {frac:.2e} px from an integer"
    return idx, w


def _sample(X, idx, w):
    """Bilinear warp of X (n,HW,C) float64 with fp32 taps: (sum_k w_k x_k, sum_k w_k |x_k|), each (n,HW,C)."""
    C = X.shape[-1]
    out = torch.zeros(idx.shape[0], idx.shape[-1], C, dtype=torch.float64)
    ab = torch.zeros_like(out)
    for k in range(4):
        g = torch.gather(X, 1, idx[:, k].clamp_min(0).unsqueeze(-1).expand(-1, -1, C))
        wk = w[:, k].unsqueeze(-1)
        out += wk * g
        ab += wk * g.abs()
    return out, ab


def _reference(case, inp, vals, H, W, fault=None):
    """float64 output (N,H*W,Cout), its bound, and the pixels where every agent is masked (pyramid) for one case.  vals: the
    float64 value of each input the kernel reads.  `fault` restates a plausible kernel bug (test_bound_rejects_...)."""
    k, C = case.kernel, case.C
    HW = H * W
    dead = None
    if k in ("pyramid", "att", "max", "warp", "v2v"):
        align = case.align != (fault == "align")
        idx, w = _geometry(case, inp["theta"], H, W, align, check=fault != "align")
        if fault == "swap":
            w = w[:, [1, 0, 2, 3]]
    if k == "pyramid":
        n = case.n
        X = vals["feat"].reshape(n, HW, C)
        sc = torch.sigmoid(inp["occ"].double().reshape(n, HW)) + 1e-4
        if inp["crop"] is not None:
            e = 1 if fault == "crop_incl" else 0
            keep = torch.zeros(n, H, W, dtype=torch.float64)
            for j, (h0, h1, w0, w1) in enumerate(inp["crop"].tolist()):
                keep[j, h0:h1 + e, w0:w1 + e] = 1
            sc = sc * keep.reshape(n, HW)
        s = sum(w[:, t] * torch.gather(sc, 1, idx[:, t].clamp_min(0)) for t in range(4))
        if fault != "nomask":
            s = s.masked_fill(s == 0, -math.inf)
        a = torch.softmax(s, 0)
        a = torch.where(torch.isnan(a), 0.0, a).unsqueeze(-1)
        Xw, A = _sample(X, idx, w)
        y = (a * Xw).sum(0, keepdim=True)
        bound = ALPHA * (a * A).sum(0, keepdim=True) + REL * y.abs()
        dead = (a.sum(0) == 0).reshape(1, HW)
    elif k == "att":
        n = case.n
        Xw, A = _sample(vals["feat"].reshape(n, HW, C), idx, w)
        d = (Xw[0] * Xw).sum(-1) / (C if fault == "scale" else math.sqrt(C))
        a = torch.softmax(d, 0).unsqueeze(-1)
        y = (a * Xw).sum(0, keepdim=True)
        D = ((A[0] * A).sum(-1) / math.sqrt(C)).unsqueeze(-1)
        sens = (a * Xw.abs() * (D + (a * D).sum(0, keepdim=True))).sum(0, keepdim=True)
        bound = ALPHA * ((a * A).sum(0, keepdim=True) + sens) + REL * y.abs()
    elif k == "max":
        Xw, A = _sample(vals["feat"].reshape(case.n, HW, C), idx, w)
        if fault == "oov":      # agents with no tap on their map left out of the max
            Xw = torch.where((w.sum(1) > 0).unsqueeze(-1), Xw, -math.inf)
            y = Xw.max(0, keepdim=True).values
            y = torch.where(torch.isinf(y), 0.0, y)
        else:
            y = Xw.max(0, keepdim=True).values
        bound = ALPHA * A.max(0, keepdim=True).values + REL * y.abs()
    elif k == "warp":
        X = vals["src"].reshape(3, HW, C)[inp["index"]]
        y, A = _sample(X, idx, w)
        bound = ALPHA * A + REL * y.abs()
    elif k == "v2v":
        q, p, x = (vals[s].reshape(-1, HW, C) for s in ("q", "p", "x"))
        m = torch.ones_like(w[:, 0]) if fault == "mask1" else w.sum(1)
        ys, bs = [], []
        for xi, pi, r, nn in inp["nodes"]:
            mj = m[r:r + nn].unsqueeze(-1)
            msg, mag = mj * (q[r:r + nn] + p[pi]), mj * (q[r:r + nn].abs() + p[pi].abs())
            if case.agg_max:
                agg, magg = msg.max(0).values, mag.max(0).values
            else:
                agg, magg = msg.sum(0) / (max(nn - 1, 1) if fault == "n_minus_1" else nn), mag.sum(0) / nn
            if case.gru:
                ys.append(torch.cat([x[xi], agg], -1))
                bs.append(torch.cat([REL * x[xi].abs(), ALPHA * magg + REL * agg.abs()], -1))
            else:
                ys.append(x[xi] + agg)
                bs.append(ALPHA * (magg + x[xi].abs()) + REL * ys[-1].abs())
        y, bound = torch.stack(ys), torch.stack(bs)
    else:
        zc = vals["zc"].reshape(case.n, HW, 2 * C)
        z, c = zc[..., :C], zc[..., C:]
        y = torch.tanh(z) * torch.sigmoid(c) if fault == "swap_act" else torch.sigmoid(z) * torch.tanh(c)
        bound = (ALPHA + REL) * y.abs()
    return y, bound, dead


# ------------------------------------------------------------------------------------------------ the bound is sharp (CPU)
def _faults(case):
    f = ["lo"] if case.fmt == "split" else []
    k = case.kernel
    if k in ("pyramid", "att", "max", "warp"):
        f.append("swap")
    if k == "pyramid":
        f.append("nomask")
        if case.crop is not None:
            f.append("crop_incl")
        if case.align:
            f.append("align")
    if k == "att" and case.n > 1:
        f.append("scale")
    if k == "max" and case.out_of_view:
        f.append("oov")
    if k == "v2v":
        f.append("mask1")
        if not case.agg_max:
            f.append("n_minus_1")
    if k == "gru":
        f.append("swap_act")
    return f


def _shrunk(case):
    return min(case.H, 8), min(case.W, 16)


@pytest.mark.parametrize("name", list(CASE))
def test_bound_rejects_plausible_kernel_bugs(name):
    """Each plausible kernel bug, restated on the float64 reference of a shrunken case, leaves the bound on some element: the
    lo plane of split input dropped, the nw / ne taps swapped, a crop end treated as inclusive, zero warped scores not masked,
    align_corners ignored, attention scaled by 1/C instead of 1/sqrt(C), the max without the zeros of out-of-view agents, the
    V2VNet mask set to 1 instead of the sum of the tap weights, the mean over n - 1 neighbours, sigmoid and tanh swapped in the
    GRU gate.  Also checks the tap geometry rule (MIN_FRAC, or pixel centres for the edge cases) at the shrunken size."""
    case = CASE[name]
    H, W = _shrunk(case)
    inp = _inputs(case, H, W)
    st = {s: _store(inp[s], case.fmt) for s in INPUT_KEYS[case.kernel]}
    vals = {s: _value(t, case.fmt) for s, t in st.items()}
    y, bound, _ = _reference(case, inp, vals, H, W)
    assert bool(torch.isfinite(y).all())
    faults = _faults(case)
    assert faults, name
    for fault in faults:
        v = {s: _value(t, case.fmt, drop_lo=True) for s, t in st.items()} if fault == "lo" else vals
        yf = _reference(case, inp, v, H, W, fault)[0]
        d = (yf - y).abs()
        ratio = torch.where(d == 0, 0.0, d / bound).max().item()
        assert ratio > 1, f"{name}: the bound does not reject '{fault}' (max err / bound {ratio:.3f})"


def test_reference_taps_follow_grid_sample():
    """_taps + _sample reproduce F.grid_sample on the fp32 grid of affine_grid (the reference's warp) up to grid_sample's own
    fp32 sums over the four taps, for generic and edge poses with and without align_corners.  With grid_sample's
    unnormalisation rounded twice instead of once, taps move by an fp32 ulp and max_f32_n4 / pyr_split_c64_n5 exceed this
    bound 10 to 20 times over."""
    for case, align in ((CASE["pyr_split_c128_n3_align"], True), (CASE["max_f32_n4"], False), (CASE["pyr_f32_edges"], False),
                        (CASE["pyr_split_c64_n5"], False)):
        H, W = case.H, case.W
        g = torch.Generator().manual_seed(1)
        x = torch.randn(case.n, 8, H, W, generator=g)
        th = _thetas(case, H, W, case.n)
        grid = F.affine_grid(th, [case.n, 8, H, W], align_corners=align).float()
        ref = F.grid_sample(x, grid, align_corners=align)
        idx, w = _geometry(case, th, H, W, align)
        got, A = _sample(x.double().permute(0, 2, 3, 1).reshape(case.n, H * W, 8), idx, w)
        got, A = (t.reshape(case.n, H, W, 8).permute(0, 3, 1, 2) for t in (got, A))
        ratio = ((got - ref.double()).abs() / (2.0 ** -21 * A)).nan_to_num(nan=0.0).max().item()
        assert ratio <= 1, f"{case.name}: F.grid_sample differs from _taps + _sample by {ratio:.3f} x 2^-21 A"


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


def _gathered(st, occ, fmt, H, W, C):
    """Agents in a shuffled order with gaps in one flat buffer, as in the all-gathered buffer of the agent-per-GPU partition:
    (Act of one agent's geometry at the buffer base, feature offsets, occupancy buffer, occupancy offsets).  The gaps hold
    SENTINEL (features) and NaN (occupancy), so a read from a wrong place shows in the result."""
    from heal_b200 import ops
    n, per, gap = occ.shape[0], H * W * C, 24
    order = torch.randperm(n, generator=torch.Generator().manual_seed(7)).tolist()
    foff, ooff = [0] * n, [0] * n
    for slot, j in enumerate(order):
        foff[j] = gap + slot * (per + gap)
        ooff[j] = 3 + slot * (H * W + 5)
    L = gap + n * (per + gap)
    planes = 1 if fmt == "f32" else st.shape[0]
    flat = torch.full((planes, L), SENTINEL, dtype=torch.float32 if fmt == "f32" else torch.bfloat16)
    obuf = torch.full((3 + n * (H * W + 5),), float("nan"))
    for j in range(n):
        flat[:, foff[j]:foff[j] + per] = (st[j][None] if fmt == "f32" else st[:, j]).reshape(planes, per)
        obuf[ooff[j]:ooff[j] + H * W] = occ[j].flatten()
    flat, obuf = flat.cuda(), obuf.cuda()
    if fmt == "f32":
        act = ops.Act(flat[0, :per].view(1, H, W, C), fmt)
    else:
        act = ops.Act(torch.as_strided(flat, (planes, 1, H, W, C), (L, per, W * C, C, 1)), fmt)
    return act, foff, obuf, ooff


def _launch(case):
    """Runs A (fp32 output) and B (the input's format) of a case.  Returns the inputs as the kernel read them (storage
    tensors, on the CPU), the input buffers, and both outputs."""
    from heal_b200 import ops
    inp = _inputs(case)
    H, W, C, n = case.H, case.W, case.C, case.n
    st = {s: _store(inp[s], case.fmt) for s in INPUT_KEYS[case.kernel]}
    first = INPUT_KEYS[case.kernel][0]
    bufs, acts = {}, {}
    for s, t in st.items():
        bufs[s], acts[s] = _put(t, case.fmt, case.in_slice if s == first else None)
    theta = inp.get("theta").cuda() if "theta" in inp else None
    width, oco = case.out_slice or ((2 * C if case.kernel == "v2v" and case.gru else C), 0)
    cout = 2 * C if case.kernel == "v2v" and case.gru else C
    row0, nrows = case.rows or (0, H)
    row0 = row0 % H
    N_out = {"pyramid": 1, "att": 1, "max": 1, "warp": n, "v2v": 2, "gru": n}[case.kernel]
    H_out = nrows if case.kernel == "pyramid" else H
    outs = {}
    gathered = _gathered(st["feat"], inp["occ"], case.fmt, H, W, C) if case.gathered else None
    for run, fmt in (("A", "f32"), ("B", case.fmt)):
        buf = _out_buffer(N_out, H_out, W, width, fmt, case.out_slice is not None)
        view = ops.Act(buf[..., oco:oco + cout], fmt)
        if case.kernel == "pyramid":
            crop = inp["crop"].cuda() if inp["crop"] is not None else None
            if gathered:
                act, foff, obuf, ooff = gathered
                ops.pyramid_fuse_level(act, obuf, theta, case.align, crop, out=ops.Act(buf, fmt), out_coffset=oco,
                                       agent_offsets=(foff, ooff), n_agents=n, rows=(row0, nrows))
            else:
                ops.pyramid_fuse_level(acts["feat"], inp["occ"].cuda().contiguous(), theta, case.align, crop,
                                       out=ops.Act(buf, fmt), out_coffset=oco, rows=(row0, nrows))
        elif case.kernel == "att":
            ops.att_fuse(acts["feat"], theta, out=view)
        elif case.kernel == "max":
            ops.max_fuse(acts["feat"], theta, out=view)
        elif case.kernel == "warp":
            ops.warp_affine(acts["src"], inp["index"], theta, out=view)
        elif case.kernel == "v2v":
            ops.v2v_aggregate(acts["q"], acts["p"], acts["x"], theta, inp["nodes"], case.agg_max, case.gru, out=view)
        else:
            ops.gru_gate(acts["zc"], out=view)
        outs[run] = buf
    return dict(inp=inp, st=st, bufs=bufs, outs=outs, oco=oco, cout=cout, rows=(row0, nrows))


def _bits(t):
    t = t.contiguous()
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASE))
def test_fuse_kernel(name):
    case = CASE[name]
    r = _launch(case)
    torch.cuda.synchronize()
    H, W, oco, cout = case.H, case.W, r["oco"], r["cout"]
    row0, nrows = r["rows"]
    # 1. the inputs as the kernel read them (read back from the device), and the sentinels around an input slice
    vals = {}
    for s, buf in r["bufs"].items():
        b = buf.cpu()
        width, coff = case.in_slice if (case.in_slice and s == INPUT_KEYS[case.kernel][0]) else (b.shape[-1], 0)
        c_in = r["st"][s].shape[-1]
        vals[s] = _value(b[..., coff:coff + c_in], case.fmt)
        if width != c_in:
            whole = _value(b, case.fmt)
            around = torch.cat([whole[..., :coff].flatten(), whole[..., coff + c_in:].flatten()])
            assert bool((around == SENTINEL).all()), f"{name}: the input buffer around the slice changed"
    # 2. run A against float64
    y, bound, dead = _reference(case, r["inp"], vals, H, W)
    Nn = y.shape[0]
    y = y.reshape(Nn, H, W, cout)[:, row0:row0 + nrows]
    bound = bound.reshape(Nn, H, W, cout)[:, row0:row0 + nrows]
    a_full = r["outs"]["A"].cpu()
    a = a_full[..., oco:oco + cout]
    err = (a.double() - y).abs()
    ok = err <= bound
    ratio = torch.where(err == 0, 0.0, err / bound).max().item()
    print(f"{name}: max err / bound {ratio:.4f}  (max err {err.max().item():.3e}, max|y| {y.abs().max().item():.3f}, "
          f"ALPHA 2^{math.log2(ALPHA):.0f})")
    assert bool(ok.all()), f"{name}: {int((~ok).sum())} elements outside the bound, max err / bound {ratio:.3f}"
    if dead is not None:
        dead = dead.reshape(1, H, W)[:, row0:row0 + nrows]
        assert bool((a[dead] == 0).all()), f"{name}: a pixel with every agent masked is not 0"
        if case.all_masked:
            assert bool(dead.any()), f"{name}: no pixel has every agent masked"
    # 3. run B is the rounding of run A
    b_full = r["outs"]["B"].cpu()
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


_KERNEL = re.compile(r"\b(k_(?:pyramid_fuse_split8|pyramid_fuse|att_fuse_split8|att_fuse|max_fuse|warp_affine|v2v_aggregate|gru_gate))"
                     r"\b(?:<\s*(?:\(int\))?\s*(\d+)\s*>)?")


def _launched_name(key):
    """`k_name<N>` for a fuse.cu kernel's profiler name, None for any other kernel (torch's fills and copies)."""
    m = _KERNEL.search(key)
    return m.group(1) + (f"<{m.group(2)}>" if m.group(2) else "") if m else None


def _launched(prof):
    return {n for n in (_launched_name(e.key) for e in prof.key_averages()) if n}


def _profiled_kernels():
    """Runs every case under one torch.profiler session and returns the fuse.cu kernels it recorded, in launch order (each case is
    two library launches, runs A and B, so the list holds the cases' pairs in case order).  A session that recorded none of the
    launches the library counted is repeated once (a wrong kernel never is)."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    from heal_b200._lib import lib
    for _ in range(2):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for case in CASES:
                before = lib.heal_launch_count()
                _launch(case)
                torch.cuda.synchronize()
                assert lib.heal_launch_count() - before == 2, f"{case.name}: runs A and B are one launch each"
        ours = sorted((e.time_range.start, _launched_name(e.name)) for e in prof.events()
                      if e.device_type == DeviceType.CUDA and _launched_name(e.name))
        if ours:
            break
    return [n for _, n in ours]


@pytest.mark.gpu
def test_each_case_launches_its_instantiations():
    """Each case runs the instantiations its row names (kernel names from torch.profiler), and together the cases run all of
    REACHABLE: a change to a dispatch predicate cannot quietly move a case off what it exists to test.

    The profiler session runs in a child process.  torch.profiler's CUDA records travel through activity buffers that live for
    the whole process, so a short session late in a long process can come back without any kernel record, depending on every
    session and CUDA call the process made before it.  In a process of its own the session does not depend on what ran
    earlier in the suite."""
    tests_dir = os.path.dirname(os.path.abspath(__file__))
    code = ("import json, sys; sys.path[:0] = [%r, %r]; import test_gpu_fuse_kernels as t; "
            "print('KERNELS ' + json.dumps(t._profiled_kernels()))" % (tests_dir, os.path.dirname(tests_dir)))
    r = subprocess.run([sys.executable, "-s", "-c", code], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stdout[-4000:]
    names = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("KERNELS ")][-1][len("KERNELS "):])
    assert len(names) == 2 * len(CASES), f"the session recorded {len(names)} fuse.cu kernels for {2 * len(CASES)} launches"
    for i, case in enumerate(CASES):
        assert set(names[2 * i:2 * i + 2]) == set(case.reaches), \
            f"{case.name}: ran {names[2 * i:2 * i + 2]}, expected {sorted(case.reaches)}"
    print(f"instantiations reached: {len(set(names) & REACHABLE)} of {len(REACHABLE)}")
    assert set(names) == REACHABLE


def _misaligned_call(kernel, where, fmt):
    """One call of `kernel` whose input (where='in') or output (where='out') view starts at channel 2 of a wider buffer:
    an 8-byte aligned pointer for fp32, 4-byte aligned for bf16.  Every other argument is well formed."""
    from heal_b200 import ops
    H, W, C, n = 5, 7, 128, 2
    th = _thetas(CASE["max_f32_n4"], H, W, n).cuda()

    def act(N, c, bad):
        t = torch.zeros((N, H, W, c + 4)) if fmt == "f32" else torch.zeros((1, N, H, W, c + 4), dtype=torch.bfloat16)
        t = t.cuda()
        return ops.Act(t[..., 2:2 + c] if bad else t[..., :c], fmt)

    bad_in, bad_out = where == "in", where == "out"
    if kernel == "pyramid":
        occ = torch.zeros(n, H, W, device="cuda")
        return lambda: ops.pyramid_fuse_level(act(n, C, bad_in), occ, th, False, out=act(1, C, bad_out))
    if kernel == "att":
        return lambda: ops.att_fuse(act(n, C, bad_in), th, out=act(1, C, bad_out))
    if kernel == "max":
        return lambda: ops.max_fuse(act(n, C, bad_in), th, out=act(1, C, bad_out))
    if kernel == "warp":
        return lambda: ops.warp_affine(act(n, C, bad_in), [0, 1], th, out=act(n, C, bad_out))
    if kernel == "v2v":
        return lambda: ops.v2v_aggregate(act(n, C, bad_in), act(1, C, False), act(1, C, False), th, [(0, 0, 0, 2)], False,
                                         True, out=act(1, 2 * C, bad_out))
    return lambda: ops.gru_gate(act(n, 2 * C, bad_in), out=act(n, C, bad_out))


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["f32", "bf16"])
@pytest.mark.parametrize("where", ["in", "out"])
@pytest.mark.parametrize("kernel", ["pyramid", "att", "max", "warp", "v2v", "gru"])
def test_misaligned_view_is_refused(kernel, where, fmt):
    """A view whose data pointer the 4-channel loads or stores cannot use is refused (HEAL_ERR_UNSUPPORTED ->
    RuntimeError) and nothing is launched.  (A split view at channel 4 is accepted and takes the generic kernel: the
    pyr_split_slice4 and att_split_c128_n3_slice4 cases.)"""
    from torch.profiler import ProfilerActivity, profile
    from heal_b200._lib import lib
    call = _misaligned_call(kernel, where, fmt)
    torch.cuda.synchronize()
    before = lib.heal_launch_count()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        with pytest.raises(RuntimeError, match="HEAL_ERR_UNSUPPORTED"):
            call()
        torch.cuda.synchronize()
    assert lib.heal_launch_count() == before
    assert not _launched(prof), f"{kernel}: launched {sorted(_launched(prof))}"
