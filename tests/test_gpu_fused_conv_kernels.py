"""The fused ResNeXt bottleneck kernels against float64, one case per tile schedule: heal_bottleneck_tc (PyramidFusion level 0,
64 -> 128 -> 64) and the expand + heal_gconv_reduce_tc of levels 1 and 2 (C -> 2C -> C, C = 128 or 256).

Both kernels are persistent: a grid of min(work, 132) CTAs walks the work list with a stride of the grid, so a CTA runs
several tiles exactly when the work exceeds 132.  Work is N * ceil(H / 16) * ceil(W / 8) tiles of 16 x 8 pixels for the
bottleneck, and that times Cout / 128 items for gconv_reduce (level 2's two 128-channel n-tiles of one pixel tile are two
items).  The cases are chosen by that schedule: one tile, exactly one tile per CTA, one CTA with two, ragged maps, the product
frame at 19-20 tiles per CTA, channel slices of wider maps, and back-to-back blocks on one stream with no synchronisation (every
launch uses programmatic dependent launch).

Each case runs in both activation modes, 'split' (hi + lo bf16 planes) and 'bf16' (one plane), and checks:
  (a) the fused output is bit-identical to the chain of heal_conv2d_tc launches it replaces (expand, grouped 3x3, reduce with
      the residual), block by block;
  (b) every chain stage, run again with an f32 output, is within |got - y64| <= ALPHA * (|W| (*) |u|) + REL * (|y64| + |b| + |r|)
      of float64 computed from the nn modules themselves (so the BN fold and the packing are covered) on the exact stored
      input u (and residual r) it read; its split / bf16 output is exactly the rounding of that f32 output and equals the
      product call's output bit for bit.  With (a) this checks the fused kernels' internal mid and g maps without reading them;
  (c) the fused output is within a propagated bound of the whole block computed in float64 from the unrounded input: each
      stage's bound (b) plus the rounding of its stored output, carried through the absolute-value convolutions of the later
      stages (ReLU is 1-Lipschitz).  This catches an error the fused and the chained paths share.
test_chain_grouped_conv_runs_the_kernel_each_case_names checks from torch.profiler's kernel names that the chain's grouped
3x3 runs the kernel each case names: the row-ring kernel on maps a multiple of 128 pixels wide, the grouped tile kernel on the
others.  test_bounds_reject_plausible_kernel_bugs (no GPU) restates plausible bugs of these kernels in float64 on the same cases and
shows each one outside the bound by a stated margin.

The products are split-bf16: the dropped lo x lo product and the weights' two-plane rounding each carry up to 2^-16 of
|a| |w|, so ALPHA is their sum, 2^-15, with the fp32 accumulation inside it.  Measured on an H100 80GB HBM3 (700 W power
limit): at the epilogue test's ALPHA = 2^-16 the largest err / bound of (b) was 0.93 (bt_chain3 [split], block 2, grouped
3x3).  At ALPHA = 2^-15 it is 0.47 (0.22 in the 'bf16' mode), 2.1x of headroom.  The largest of (c) is 0.18 (bt_chain3
[bf16], block 2), and 0.007 in the split mode.  test_fused_conv_kernels prints err / bound for every stage and block."""
import json
import math
import os
import re
import subprocess
import sys
import zlib
from dataclasses import dataclass
from typing import Optional, Tuple

import pytest
import torch
import torch.nn.functional as F

ALPHA = 2.0 ** -15
REL = 2.0 ** -22
SENTINEL = -1000.0                        # finite and exact in bf16: fills the channels around a slice
MODES = {"split": 2, "bf16": 1}           # activation format -> planes; the packed weights always carry 2 planes
STORE_U = {2: 2.0 ** -16, 1: 2.0 ** -8}   # relative error of storing an fp32 value as bf16 hi + lo / as bf16 (round to nearest)
NUM_SMS = 132                             # HEAL_NUM_SMS: the persistent grids are min(work, 132) CTAs
TILE_H, TILE_W, NT = 16, 8, 128           # the fused kernels' output tile, and gconv_reduce's output channels per item
GROUPS = 32


@dataclass(frozen=True)
class Case:
    name: str
    C: int                                       # 64: bottleneck_tc; 128 / 256: expand + gconv_reduce_tc
    shape: Tuple[int, int, int]                  # N, H, W
    work: int                                    # tiles (bottleneck) or items (gconv_reduce), as the comment states
    grouped: str                                 # the chain's grouped 3x3: 'ring' (k_gconv3x3_ring) or 'tile' (k_conv2d_tc)
    blocks: int = 1                              # blocks run back to back, each reading the previous output
    in_slice: Optional[Tuple[int, int]] = None   # (buffer width, channel offset) x and the residual are read from
    out_slice: Optional[Tuple[int, int]] = None  # (buffer width, channel offset) the fused output is written into
    mid_slice: Optional[Tuple[int, int]] = None  # gconv_reduce: (buffer width, channel offset) of the expand's output

    @property
    def n_tiles(self):
        return 1 if self.C == 64 else self.C // NT

    @property
    def tiles(self):
        N, H, W = self.shape
        return N * math.ceil(H / TILE_H) * math.ceil(W / TILE_W)

    @property
    def grid(self):
        return min(self.tiles * self.n_tiles, NUM_SMS)


CASES = [
    # ---- heal_bottleneck_tc (level 0); the chain's grouped 3x3 is 'ring' when W % 128 == 0
    # 1 tile: one CTA, one tile (the chain's grouped conv: 8-wide tiles, a box per tap)
    Case("bt_1tile", 64, (1, 5, 7), 1, "tile"),
    # 3 x 44 = 132 tiles: every CTA runs exactly one
    Case("bt_132", 64, (1, 48, 352), 132, "tile"),
    # 7 x 1 x 19 = 133 tiles: CTA 0 runs two (tiles 0 and 132), the cross-tile x prefetch and the second bar_xfull phase
    Case("bt_133", 64, (7, 16, 152), 133, "tile"),
    # 5 x 3 x 11 = 165 ragged tiles (37 = 2 x 16 + 5 rows, 83 = 10 x 8 + 3 columns): CTAs 0-32 run two
    Case("bt_ragged_165", 64, (5, 37, 83), 165, "tile"),
    # the product's level-0 frame (5 agents, 256 x 256 after the 512 x 512 pillar grid's stride-2 backbone):
    # 5 x 16 x 32 = 2560 tiles, 19 per CTA and 20 on CTAs 0-51
    Case("bt_frame", 64, (5, 256, 256), 2560, "ring"),
    # x and the residual read from channels [64, 128) of a 192-wide map: 3 x 3 x 16 = 144 tiles, CTAs 0-11 run two
    Case("bt_in_slice", 64, (3, 48, 128), 144, "ring", in_slice=(192, 64)),
    # output written into channels [64, 128) of a 192-wide map: 2 x 3 x 25 = 150 tiles, CTAs 0-17 run two
    Case("bt_out_slice", 64, (2, 33, 200), 150, "tile", out_slice=(192, 64)),
    # three blocks back to back: 2 x 4 x 48 = 384 tiles each, 2 per CTA and 3 on CTAs 0-119
    Case("bt_chain3", 64, (2, 64, 384), 384, "ring", blocks=3),
    # ---- expand + heal_gconv_reduce_tc (levels 1 and 2): items = tiles x Cout / 128
    # the product's level-1 frame: 5 x 8 x 16 = 640 items, 4 per CTA and 5 on CTAs 0-111
    Case("gr1_frame", 128, (5, 128, 128), 640, "ring"),
    # the product's level-2 frame: 5 x 4 x 8 = 160 tiles x 2 n-tiles = 320 items, 2 per CTA and 3 on CTAs 0-55
    Case("gr2_frame", 256, (5, 64, 64), 320, "tile"),
    # an odd number of pixel tiles, 3 x 3 x 9 = 81: 162 items, CTAs 0-29 run two; the n-tile pairs of tiles 66-80 are the
    # second items of CTAs 2k and 2k + 1
    Case("gr2_odd_tiles", 256, (3, 40, 72), 162, "tile"),
    # the expand writes mid into channels [64, 320) of a 384-wide map, gconv_reduce reads it there: 2 x 3 x 25 = 150 items
    Case("gr1_mid_slice", 128, (2, 48, 200), 150, "tile", mid_slice=(384, 64)),
    # x and the residual read from channels [64, 320) of a 384-wide map: 2 x 3 x 16 x 2 = 192 items, CTAs 0-59 run two
    Case("gr2_res_slice", 256, (2, 40, 128), 192, "ring", in_slice=(384, 64)),
    # two level-1 blocks back to back: 3 x 2 x 32 = 192 items each, CTAs 0-59 run two
    Case("gr1_chain2", 128, (3, 32, 256), 192, "ring", blocks=2),
]
CASE = {c.name: c for c in CASES}


def _grouped_path(case):
    """Which kernel heal_conv2d_tc runs for the chain's grouped 3x3 (its dispatch, conv2d_tc.cu): the row-ring kernel when the
    staging epilogue applies (no f32 output, no residual), the map is a multiple of 128 pixels wide and Cin == Cout; else the
    64-wide grouped tile kernel."""
    return "ring" if case.shape[2] % 128 == 0 else "tile"


def test_case_table_states_the_kernels_schedules():
    """The counts in the table are the kernels' own tile arithmetic, and the table reaches what it exists to reach."""
    for c in CASES:
        assert c.tiles * c.n_tiles == c.work, f"{c.name}: the kernel's work list has {c.tiles * c.n_tiles} entries"
        assert _grouped_path(c) == c.grouped, c.name
        assert c.blocks == 1 or not (c.in_slice or c.out_slice or c.mid_slice)
    for lvl in (64, 128, 256):
        cs = [c for c in CASES if c.C == lvl]
        assert any(c.work > NUM_SMS for c in cs), f"C {lvl}: no case runs two or more tiles per CTA"
        assert {c.grouped for c in cs} == {"ring", "tile"}, f"C {lvl}: the chain's grouped 3x3 does not run both kernels"
    assert any(c.work == NUM_SMS + 1 for c in CASES) and any(c.work == NUM_SMS for c in CASES)


# ------------------------------------------------------------------------------------------------ float64 reference
def _modules(case, b):
    """Block b of the case: PyramidFusion's bottleneck C -> 2C -> C (32 groups) with random BN statistics.  The BN shifts are
    mostly positive, so ReLU(b1) is not 0 where the grouped conv zero-pads its input."""
    gen = torch.Generator().manual_seed(zlib.crc32(f"{case.name}/{b}".encode()))
    C, width = case.C, 2 * case.C
    convs = [torch.nn.Conv2d(C, width, 1, bias=False), torch.nn.Conv2d(width, width, 3, padding=1, groups=GROUPS, bias=False),
             torch.nn.Conv2d(width, C, 1, bias=False)]
    bns = [torch.nn.BatchNorm2d(c).eval() for c in (width, width, C)]
    with torch.no_grad():
        for conv in convs:
            conv.weight.copy_(torch.randn(conv.weight.shape, generator=gen) * math.sqrt(2.0 / conv.weight[0].numel()))
        for bn in bns:
            c = bn.num_features
            bn.weight.copy_(torch.rand(c, generator=gen) + 0.5)
            bn.bias.copy_(torch.randn(c, generator=gen) * 0.1 + 0.3)
            bn.running_mean.copy_(torch.randn(c, generator=gen) * 0.1)
            bn.running_var.copy_(torch.rand(c, generator=gen) + 0.5)
    return convs, bns


def _folded(conv, bn, device):
    """Eval BatchNorm folded into the conv's weight and bias, in float64."""
    s = bn.weight.detach().double() / torch.sqrt(bn.running_var.detach().double() + bn.eps)
    b = bn.bias.detach().double() - bn.running_mean.detach().double() * s
    return (conv.weight.detach().double() * s.view(-1, 1, 1, 1)).to(device), b.to(device)


def _params(case, device):
    """[(w, b, groups) x 3] per block, float64."""
    out = []
    for b in range(case.blocks):
        convs, bns = _modules(case, b)
        out.append([(*_folded(c, n, device), c.groups) for c, n in zip(convs, bns)])
    return out


def _conv(w, u, groups):
    return F.conv2d(u, w, padding=w.shape[-1] // 2, groups=groups)


def _stage(w, b, groups, u, r=None):
    """ReLU(conv(u) + b (+ r)) in float64."""
    v = _conv(w, u, groups) + b.view(1, -1, 1, 1)
    return (v if r is None else v + r).clamp_min(0)


def _stage_bound(w, b, groups, u, y, r=None):
    extra = b.abs().view(1, -1, 1, 1) + (0 if r is None else r.abs())
    return ALPHA * _conv(w.abs(), u.abs(), groups) + REL * (y.abs() + extra)


def _store(y, planes):
    """The value a kernel stores for float64 `y` (through fp32) as bf16 hi + lo (planes 2) or bf16 (planes 1), in float64."""
    y32 = y.float()
    hi = y32.to(torch.bfloat16)
    if planes == 1:
        return hi.double()
    return hi.double() + (y32 - hi.float()).to(torch.bfloat16).double()


def _block_bound(blk, z, E, planes):
    """One block in float64 from its exact input z, and an elementwise bound on |stored output - exact| given |input - z| <= E:
    per stage the input error through |W| (plus the residual's error), that stage's bound (b) and the rounding of its stored
    output."""
    U = STORE_U[planes]
    xz, xE = z, E
    for s, (w, b, g) in enumerate(blk):
        res = s == 2
        zn = _stage(w, b, g, z, xz if res else None)
        prop = _conv(w.abs(), E, g) + (xE if res else 0)
        mag = zn + prop                                        # >= |stage(u)| for every input u within E of z
        extra = b.abs().view(1, -1, 1, 1) + (xz.abs() + xE if res else 0)
        bs = ALPHA * _conv(w.abs(), z.abs() + E, g) + REL * (mag + extra)
        E = prop + bs + U * (mag + bs)
        z = zn
    return z, E


# ------------------------------------------------------------------------------------------------ the bound is sharp (CPU)
def _untile(t, case, H, W):
    N, Hp, Wp = case.shape[0], math.ceil(H / TILE_H) * TILE_H, math.ceil(W / TILE_W) * TILE_W
    th, tw = Hp // TILE_H, Wp // TILE_W
    c = t.shape[1]
    return t.view(N, th, tw, c, TILE_H, TILE_W).permute(0, 3, 1, 4, 2, 5).reshape(N, c, Hp, Wp)[..., :H, :W]


def _tiles(r, case):
    """(N, C, H, W) -> (tiles, C, 16, 8) in the kernels' tile order (image, tile row, tile column), zero outside the image."""
    N, c, H, W = r.shape
    th, tw = math.ceil(H / TILE_H), math.ceil(W / TILE_W)
    p = F.pad(r, (0, tw * TILE_W - W, 0, th * TILE_H - H))
    return p.view(N, c, th, TILE_H, tw, TILE_W).permute(0, 2, 4, 1, 3, 5).reshape(N * th * tw, c, TILE_H, TILE_W)


def _stale(r, case):
    """The residual each work item would add if it read the x tile of the item its CTA ran before it (item - grid): the next
    tile's prefetch landing in the resident tile too early.  A CTA's first item keeps its own."""
    t = _tiles(r, case)
    out = t.clone()
    n = case.n_tiles
    cb = r.shape[1] // n
    assert case.grid % n == 0                          # so the item before an n-tile-nt item is an n-tile-nt item too
    for nt in range(n):
        items = torch.arange(t.shape[0]) * n + nt
        m = items >= case.grid
        out[m, nt * cb:(nt + 1) * cb] = t[(items[m] - case.grid) // n, nt * cb:(nt + 1) * cb]
    return _untile(out, case, r.shape[2], r.shape[3])


STAGE_NAMES = ("expand", "grouped", "reduce")
# bug -> (the stage it corrupts, the bound it is held to, what it restates).  A bug a chain stage can have too (a dropped cross
# product, a shifted halo) is held to that stage's bound (b) in both modes.  The others exist only inside a fused kernel, where
# (a) pins it to the chain; they are held to the block bound (c), which is what would catch them if the chain shared them, in
# the split mode.  In the bf16 mode (c) carries each stored map's 2^-8 rounding through the absolute-value convolutions of the
# later stages and is printed only: a 128-channel reduce over a 3x3 grouped conv widens it about a hundredfold.
BUGS = {
    "stale_residual": (2, "c", "the residual read from the x tile the CTA ran before (a stale cross-tile prefetch)"),
    "mid_pad": (1, "c", "mid pixels outside the image holding ReLU(b1) instead of 0 (the bottleneck's expand over the halo)"),
    "nt_bias": (2, "c", "level 2: the second 128-channel n-tile adding the first one's bias"),
    "drop_cross_expand": (0, "b", "one split cross product dropped: a_lo x b_hi (split) / a_hi x b_lo (bf16)"),
    "drop_cross_grouped": (1, "b", "one split cross product dropped: a_lo x b_hi (split) / a_hi x b_lo (bf16)"),
    "drop_cross_reduce": (2, "b", "one split cross product dropped: a_lo x b_hi (split) / a_hi x b_lo (bf16)"),
    "halo_shift": (1, "b", "the grouped conv's taps one pixel to the right at the last column of every tile"),
}
MARGIN = 8.0             # each held bug leaves its bound by at least this factor on every case it can occur on (closest:
                         # nt_bias, 9.1 x (c); every other one 20 x or more)


def _applies(bug, case):
    if bug == "stale_residual":
        return case.tiles * case.n_tiles > NUM_SMS          # only a CTA's second item can read a stale tile
    if bug == "mid_pad":
        return case.C == 64
    if bug == "nt_bias":
        return case.C == 256
    if bug == "halo_shift":
        return case.shape[2] >= TILE_W
    return True


def _bugged_stage(bug, case, blk, s, u, r, planes):
    """Stage s of block `blk` on input u (residual r) in float64, with `bug`."""
    w, b, g = blk[s]
    if bug.startswith("drop_cross"):
        if planes == 2:
            u = u.float().to(torch.bfloat16).double()              # the activations' lo plane
        else:
            w = w.float().to(torch.bfloat16).double()              # the weights' lo plane
    elif bug == "stale_residual":
        r = _stale(r, case)
    elif bug == "nt_bias":
        b = b.clone()
        b[NT:2 * NT] = b[:NT].clone()
    elif bug == "mid_pad":
        N, _, H, W = u.shape
        ring = 1 - F.pad(torch.ones(1, 1, H, W, dtype=u.dtype), (1, 1, 1, 1))
        relu_b1 = _store(blk[0][1].clamp_min(0), planes).view(1, -1, 1, 1)
        return (F.conv2d(F.pad(u, (1, 1, 1, 1)) + ring * relu_b1, w, groups=g) + b.view(1, -1, 1, 1)).clamp_min(0)
    elif bug == "halo_shift":
        y = _stage(w, b, g, u)
        y[..., TILE_W - 1::TILE_W] = _stage(w, b, g, F.pad(u[..., 1:], (0, 1)))[..., TILE_W - 1::TILE_W]
        return y
    return _stage(w, b, g, u, r)


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("name", list(CASE))
def test_bounds_reject_plausible_kernel_bugs(name, mode):
    """Block 0 of each case as the kernels compute it when every stage is exact and every stored map is rounded as the mode
    stores it: inside the block bound (c).  Each plausible bug that can occur on the case, restated in that computation, leaves
    the bound it is held to by MARGIN.  Prints err / bound for every bug."""
    case, planes = CASE[name], MODES[mode]
    blk = _params(case, "cpu")[0]
    gen = torch.Generator().manual_seed(zlib.crc32(case.name.encode()))
    x = torch.randn(case.shape[0], case.C, *case.shape[1:], generator=gen).double()
    z, E = _block_bound(blk, x, (_store(x, planes) - x).abs(), planes)
    u, ins = _store(x, planes), []
    for s, (w, b, g) in enumerate(blk):
        r = ins[0][0] if s == 2 else None
        ins.append((u, r))
        u = _store(_stage(w, b, g, u, r), planes)
    ratio = ((u - z).abs() / E).max().item()
    print(f"{name} [{mode}] exactly rounded: err / bound (c) {ratio:.3f}")
    assert ratio <= 1, f"{name} [{mode}]: the block bound does not hold for the exactly rounded computation ({ratio:.3f})"
    for bug, (s, held, what) in BUGS.items():
        if not _applies(bug, case):
            continue
        u, r = ins[s]
        y = _bugged_stage(bug, case, blk, s, u, r, planes)
        if held == "b":
            w, b, g = blk[s]
            y64 = _stage(w, b, g, u, r)
            ratio = ((y - y64).abs() / _stage_bound(w, b, g, u, y64, r)).max().item()
        else:
            for t in range(s + 1, 3):
                w, b, g = blk[t]
                y = _stage(w, b, g, _store(y, planes), ins[0][0] if t == 2 else None)
            ratio = ((_store(y, planes) - z).abs() / E).max().item()
        print(f"{name} [{mode}] {bug:20s} err / bound ({held}) {ratio:10.2f}")
        if held == "b" or planes == 2:
            assert ratio > MARGIN, f"{name} [{mode}]: '{bug}' ({what}) is only {ratio:.2f} x its bound ({held})"


# ------------------------------------------------------------------------------------------------ the kernels (GPU)
def _slice(a, off, c):
    from heal_b200 import ops
    return ops.Act(a.t[..., off:off + c], a.fmt)


def _filled(planes, N, H, W, width, fill, fmt):
    from heal_b200 import ops
    return ops.Act(torch.full((planes, N, H, W, width), fill, dtype=torch.bfloat16, device="cuda"), fmt)


def _inputs(case, mode):
    """The case's packed weights per block, its input (fp32, and the stored map it is read from), and the buffers around its
    input slice."""
    from heal_b200 import ops
    N, H, W = case.shape
    C = case.C
    pcs = [[ops.pack_conv_tc(c, b, True, planes=2).to("cuda") for c, b in zip(*_modules(case, i))] for i in range(case.blocks)]
    gen = torch.Generator().manual_seed(zlib.crc32(case.name.encode()))
    x32 = torch.randn(N, C, H, W, generator=gen)
    width, off = case.in_slice or (C, 0)
    xb = torch.full((N, width, H, W), SENTINEL)
    xb[:, off:off + C] = x32
    xfull = ops.convert(ops.to_act(xb.cuda()), mode)
    return pcs, x32, _slice(xfull, off, C), {"in": (xfull, off, C, xfull.t.clone())}


def _chain(x, pcs):
    """The heal_conv2d_tc launches the fused blocks replace (expand, grouped 3x3, reduce with the residual), one record per
    stage."""
    from heal_b200 import ops
    stages, cur = [], x
    for pc1, pc2, pc3 in pcs:
        mid, _ = ops.conv2d_tc(cur, pc1)
        g, _ = ops.conv2d_tc(mid, pc2)
        y, _ = ops.conv2d_tc(g, pc3, residual=cur)
        stages += [dict(u=cur, pc=pc1, r=None, a=mid), dict(u=mid, pc=pc2, r=None, a=g), dict(u=g, pc=pc3, r=cur, a=y)]
        cur = y
    return stages


def _launch(case, mode):
    """The case's fused blocks back to back, then the chain of heal_conv2d_tc launches they replace, then one call per chain
    stage that also writes f32; no synchronisation in between.  Returns (the fp32 input, fused outputs per block, chain stage
    records, buffers around slices)."""
    from heal_b200 import ops
    fmt, planes = mode, MODES[mode]
    N, H, W = case.shape
    C = case.C
    pcs, x32, x, bufs = _inputs(case, mode)
    fused, cur = [], x
    for pc1, pc2, pc3 in pcs:
        out, oco = None, 0
        if case.out_slice:
            ow, oco = case.out_slice
            out = _filled(planes, N, H, W, ow, SENTINEL, fmt)
            bufs["out"] = (out, oco, C, None)
        if C == 64:
            y = ops.bottleneck_tc(cur, pc1, pc2, pc3, out=out, out_coffset=oco)
        else:
            if case.mid_slice:
                mw, mo = case.mid_slice
                mbuf = _filled(planes, N, H, W, mw, SENTINEL, fmt)
                ops.conv2d_tc(cur, pc1, out=mbuf, out_coffset=mo)
                bufs["mid"] = (mbuf, mo, 2 * C, None)
                mid = _slice(mbuf, mo, 2 * C)
            else:
                mid, _ = ops.conv2d_tc(cur, pc1)
            y = ops.gconv_reduce_tc(mid, pc2, pc3, cur, out=out, out_coffset=oco)
        cur = _slice(y, oco, C)
        fused.append(cur)
    stages = _chain(x, pcs)
    for st in stages:
        st["ob"] = ops.act_empty(N, H, W, st["pc"].cout, fmt, "cuda")
        st["of"] = ops.act_empty(N, H, W, st["pc"].cout, "f32", "cuda")
        ops.conv2d_tc(st["u"], st["pc"], residual=st["r"], out=st["ob"], out_f32=st["of"], want_f32=True)
    return x32, fused, stages, bufs


def _bits(t):
    t = t.contiguous()
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


def _nchw64(a):
    """An Act's exact values as a float64 (N, C, H, W) tensor."""
    t = a.t.double() if a.fmt == "f32" else a.t.double().sum(0)
    return t.permute(0, 3, 1, 2)


# k_conv2d_tc<BLOCK_N, STAGES, STG, GELU, GROUPED> with GROUPED set: the 64-wide grouped tile kernel
_GROUPED_TILE = re.compile(r"k_conv2d_tc<\s*(?:\(int\))?64,\s*(?:\(int\))?\d+,\s*(?:\(int\))?\d+,\s*(?:false|\(bool\)0),"
                           r"\s*(?:true|\(bool\)1)\s*>")


@pytest.mark.gpu
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("name", list(CASE))
def test_fused_conv_kernels(name, mode):
    case, planes = CASE[name], MODES[mode]
    x32, fused, stages, bufs = _launch(case, mode)
    torch.cuda.synchronize()
    tag = f"{name} [{mode}]"
    params = _params(case, "cuda")
    worst_b = worst_c = 0.0
    for bi in range(case.blocks):
        chain = stages[3 * bi + 2]["a"]
        # (a) the fused block and the chain agree bit for bit
        assert torch.equal(_bits(fused[bi].t), _bits(chain.t)), f"{tag} block {bi}: the fused output differs from the chain"
        # (b) each chain stage against float64 on the exact input it read
        for s in range(3):
            st = stages[3 * bi + s]
            w, b, g = params[bi][s]
            u = _nchw64(st["u"])
            r = None if st["r"] is None else _nchw64(st["r"])
            y64 = _stage(w, b, g, u, r)
            bound = _stage_bound(w, b, g, u, y64, r)
            of = st["of"].t
            err = (_nchw64(st["of"]) - y64).abs()
            ratio = (err / bound).max().item()
            worst_b = max(worst_b, ratio)
            print(f"{tag} block {bi} {STAGE_NAMES[s]:8s}: (b) max err / bound {ratio:.4f}  (max err {err.max().item():.3e})")
            assert bool((err <= bound).all()), f"{tag} block {bi} {STAGE_NAMES[s]}: {int((err > bound).sum())} elements outside (b)"
            hi = of.to(torch.bfloat16)
            assert torch.equal(_bits(st["ob"].t[0]), _bits(hi)), f"{tag} block {bi} {STAGE_NAMES[s]}: hi plane != bf16(f32)"
            if planes == 2:
                assert torch.equal(_bits(st["ob"].t[1]), _bits((of - hi.float()).to(torch.bfloat16))), \
                    f"{tag} block {bi} {STAGE_NAMES[s]}: lo plane != bf16(f32 - hi)"
            assert torch.equal(_bits(st["ob"].t), _bits(st["a"].t)), \
                f"{tag} block {bi} {STAGE_NAMES[s]}: the product call and the f32 call differ"
        # (c) the fused block against float64 from its unrounded input (block 0) or from the stored input it read
        if bi == 0:
            z = x32.double().cuda()
            E = (_nchw64(stages[0]["u"]) - z).abs()
        else:
            z = _nchw64(fused[bi - 1])
            E = torch.zeros_like(z)
        z, E = _block_bound(params[bi], z, E, planes)
        err = (_nchw64(fused[bi]) - z).abs()
        ratio = (err / E).max().item()
        worst_c = max(worst_c, ratio)
        print(f"{tag} block {bi} fused   : (c) max err / bound {ratio:.4f}  (max err {err.max().item():.3e})")
        assert bool((err <= E).all()), f"{tag} block {bi}: {int((err > E).sum())} elements outside the block bound (c)"
    print(f"{tag}: largest err / bound (b) {worst_b:.4f}, (c) {worst_c:.4f}  (ALPHA 2^{math.log2(ALPHA):.0f})")
    # the channels around a slice that is read keep their values, and those around a written slice their sentinel
    for key, (a, off, c, before) in bufs.items():
        t = a.t.cpu()
        around = torch.cat([t[..., :off].flatten(), t[..., off + c:].flatten()])
        if before is None:
            assert bool((around.float() == SENTINEL).all()), f"{tag}: a write spilled out of the {key} slice [{off}, {off + c})"
        else:
            b0 = before.cpu()
            assert torch.equal(_bits(around), _bits(torch.cat([b0[..., :off].flatten(), b0[..., off + c:].flatten()]))), \
                f"{tag}: the {key} buffer around the slice changed"


def _grouped_kernel(key):
    """'ring' / 'tile' for the profiler name of a grouped 3x3 kernel, None for any other kernel."""
    if "k_gconv3x3_ring" in key:
        return "ring"
    return "tile" if _GROUPED_TILE.search(key) else None


def _profiled_grouped_kernels():
    """Runs every case's chain under one torch.profiler session and returns the grouped 3x3 kernels it recorded, in launch
    order.  The dispatch does not depend on the activation mode: the split mode stands for both."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    from heal_b200._lib import lib
    inputs = [_inputs(case, "split") for case in CASES]
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for case, (pcs, _, x, _) in zip(CASES, inputs):
            before = lib.heal_launch_count()
            _chain(x, pcs)
            torch.cuda.synchronize()
            assert lib.heal_launch_count() - before == 3 * case.blocks, f"{case.name}: the chain is three launches per block"
    return [n for _, n in sorted((e.time_range.start, _grouped_kernel(e.name)) for e in prof.events()
                                 if e.device_type == DeviceType.CUDA and _grouped_kernel(e.name))]


@pytest.mark.gpu
def test_chain_grouped_conv_runs_the_kernel_each_case_names():
    """The chain's grouped 3x3 runs the row-ring kernel on the cases marked 'ring' and the grouped tile kernel on the others
    (kernel names from torch.profiler), so a change to the dispatch cannot quietly move a case off the path it covers.

    The profiler session runs in a child process: torch.profiler's CUDA records travel through activity buffers that live
    for the whole process, so a short session late in a long test process can come back without any kernel record."""
    tests_dir = os.path.dirname(os.path.abspath(__file__))
    code = ("import json, sys; sys.path[:0] = [%r, %r]; import test_gpu_fused_conv_kernels as t; "
            "print('KERNELS ' + json.dumps(t._profiled_grouped_kernels()))" % (tests_dir, os.path.dirname(tests_dir)))
    r = subprocess.run([sys.executable, "-s", "-c", code], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stdout[-4000:]
    names = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("KERNELS ")][-1][len("KERNELS "):])
    want = [k for case in CASES for k in [case.grouped] * case.blocks]
    assert len(names) == len(want), f"the session recorded {len(names)} grouped 3x3 kernels for {len(want)} launches"
    i = 0
    for case in CASES:
        assert names[i:i + case.blocks] == [case.grouped] * case.blocks, \
            f"{case.name}: the grouped 3x3 ran {names[i:i + case.blocks]}, expected {case.grouped}"
        i += case.blocks
