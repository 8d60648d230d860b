"""The Lift-Splat-Shoot kernels of csrc/lss.cu against float64 references, on inputs built for the places they can go wrong.

heal_lss_pool_sorted (k_lss_keys, k_lss_prob, the CUB sort, k_lss_pool_chunks, k_lss_pool_fixup), heal_lss_pool (the atomic
kernel), heal_lss_cell_index and heal_lss_camera_matrices, all through their wrappers in heal_b200/ops.py.

Pooling.  `cell` is an input of both pooling kernels, so a case hands them the BEV cell of every frustum point.  What
k_lss_pool_chunks does with a cell depends on how the cell-sorted points fall on chunks of 128: a cell inside one chunk is
written directly, a cell that runs past the chunk's end leaves a tail partial, one that began earlier a head partial, one that
covers a whole chunk uses the head slot again, and k_lss_pool_fixup adds the heads of the following chunks to the tail.  The
constructed maps of _runs place cells on those boundaries on purpose; _census sorts a case's keys as the kernel does and
names the situations that occur, each case declares the ones it exists for (test_case_produces_its_situations), and
together the cases produce every name in SITUATIONS.  One case has the product's size (4 cameras of 704x256, D = 48, C = 128,
256x256 cells) with `cell` from heal_lss_cell_index.

Reference: softmax over D in float64 of the fp32 logits, then per (agent, cell, channel) the float64 sum of prob * feat over
the points with cell >= 0.  A cell nobody hits is exactly 0.

Bound, first order, per output element.  With u = 2^-24, x_d = logit_d - max over d (<= 0), p_d the exact probability and
n the number of points of the cell:
  p_d as computed carries a relative error of at most u (9 + s + |x_d| + sum_k p_k |x_k|):  the subtraction rounds x_d (its
        relative error u turns into an error u |x_d| of the exponent), expf is within 2 ulp = 4u; the sum of the exponentials
        inherits their weighted mean error, 4u + u sum_k p_k |x_k|, and adds s roundings of its own; the division rounds once.
        s = 6 for k_lss_prob (one add per lane and five shuffle steps), s = D - 1 for the serial sum of k_lss_pool.
  the sum carries at most n + ceil(n / 128) + 2 roundings of a partial sum no larger than S = sum |p f|: one per fma of
        the chain (k_lss_pool: one for the product and one per atomicAdd), and one per head partial added by the fix-up.
  so |err| <= u [(n + ceil(n / 128) + 2) S + sum_points (9 + s + |x| + E|x|) |p f|] + n 2^-126 (1 + max |f|);
the last term covers probabilities below the normal range (a spread of 160 in the logits gives exp(-160)).  The bound does
not depend on the order of the sum, so the atomic kernel is held to the same one.  A cell with one point and a cell with 3000
get different bounds.  test_bound_rejects_plausible_kernel_bugs (no GPU) shows that the bound rejects each plausible kernel bug.

Every pooling case also checks that NCHW inputs and the fused channels-last heads layout (BN, fH, fW, D + C) give the same
bits, that a second run gives the same bits, that out_fmt 'bf16' is bf16(fp32 run) and 'split' is hi = bf16(A),
lo = bf16(A - hi).  Every case's logits hold a pixel of equal logits, one spread over +-80 and one with a single dominant bin.

Cell index.  With post_rots^-1 = combine = I and post_trans = 0 a coordinate is one fp32 multiply (u d), one add (+ trans), one
subtract (- lower) and one division, whatever the compiler contracts (a product with an exact 0 or 1 is exact), so numpy float32
reproduces it bit for bit: test_cell_index_exact places points on cell edges, in (-1, 0), at nx, one ulp below nx, at <= -1, on
each axis with nz = 3.  For general cameras test_cell_index_vs_float64 requires every index to be the truncation of the
float64 coordinate moved by at most eps per axis, eps = 16 u (the magnitude of the terms summed) / dx.  The roundings on the
way from the frustum point to the cell coordinate: the subtraction of post_trans (1), the three terms of post_rots^-1 (3), the
product q_xy q_z (both factors' 4, and its own: 9), the three terms of combine (12), + trans, - lower and the division (15).

What the GPU tests printed on an H100 80GB HBM3 at a 700 W power limit is kept in MEASURED below."""
import dataclasses
import math
import zlib
from dataclasses import dataclass
from typing import Tuple

import numpy as np
import pytest
import torch

U = 2.0 ** -24
TINY = 2.0 ** -126
CH = 128                   # LSS_CH of lss.cu: sorted points per block of k_lss_pool_chunks
PROB_SUM_ROUNDINGS = 6     # k_lss_prob: e0 + e1, then five shuffle steps

# What the GPU tests print, on an H100 80GB HBM3 at a 700 W power limit (err / bound of 0 means an exact output).
MEASURED = """
heal_lss_pool_sorted, 20 cases, largest err / bound 0.528 (softmax_d64); per case
    long_d48_c128 0.153, long_d64_c256 0.069, cut_d16_c32 0.142, cut_d32_c33 0.104, both_d33_c33 0.161, both_d48_c128 0.103,
    k128_d32_c64 0.040, few_d1_c1 0.015, none_d16_c200 0, all_d31_c256 0.193, agents_d64_c128 0.134, agents_d16_c1 0.015,
    pow2_d48_c32 0.185, pow2m1_d32_c64 0.468, skewed_d48_c200 0.165, softmax_d31 0.455, softmax_d32 0.455, softmax_d33 0.418,
    softmax_d64 0.528, c4 0.198 (max err 4.5e-06 at max |y| 13.0)
heal_lss_pool, the same 20 cases, largest err / bound 0.361 (softmax_d31); c4 0.122 (max err 1.4e-05)
c4 census (camera_rig(2, 4, 256, 704), D = 48, 32x88 feature map, 256x256 cells): 1081344 points, 1054486 valid, 8448 chunks,
    19476 cells hit, at most 1536 points in one cell, 1353 whole-chunk head partials, longest fix-up 12 chunks
heal_lss_cell_index, augmented rig, 1081344 points, 84 % inside the grid: 8 differ from the float64 truncation (7.4e-06), all
    within eps (largest eps inside the grid 5.8e-04 cells); hand-placed and random identity-camera points: equal to numpy float32
heal_lss_camera_matrices, n = 1 / 64 / 65: post_rots^-1 err / bound 0.356 / 0.455 / 0.445, combine 0.220 / 0.398 / 0.383
"""

SITUATIONS = (
    "direct",             # a cell begins and ends inside one chunk
    "tail",               # a cell runs past the end of its chunk
    "head",               # a cell that began in an earlier chunk ends in this one
    "whole",              # a chunk lies wholly inside one cell (head slot)
    "fixup2",             # a tail collects the heads of two or more following chunks
    "head_and_tail",      # one chunk writes both of its partial slots
    "clean_cut",          # a cell ends at slot 127 and another begins at slot 0 of the next chunk
    "tail_of_one",        # a cell begins at slot 127 and continues
    "agent_edge",         # agent a's cell (cells - 1) ends a chunk, agent a + 1's cell 0 begins the next
    "mixed_chunk",        # a chunk holds valid points and part of the invalid tail
    "full_then_invalid",  # the valid points end exactly at a chunk's end and invalid ones follow
    "invalid_chunk",      # a chunk lies wholly in the invalid tail
    "partial_last",       # the point count is not a multiple of 128
    "no_valid",           # every point is invalid
    "no_invalid",         # every point is valid
    "key_pow2",           # agents * cells is a power of two, its top cell is hit and invalid points exist
    "key_pow2m1",         # agents * cells is one less than a power of two, likewise
)


@dataclass(frozen=True)
class Case:
    name: str
    map: str                      # which cell map (_cell)
    D: int
    C: int
    fH: int
    fW: int
    BN: int                       # images
    cams: int                     # cameras per agent
    nx: int
    ny: int
    situations: Tuple[str, ...]   # what the case is there for (asserted by test_case_produces_its_situations)

    @property
    def HW(self):
        return self.fH * self.fW

    @property
    def cells(self):
        return self.nx * self.ny

    @property
    def agents(self):
        return self.BN // self.cams


CASES = [
    # the nastiest constructed map at the product's depth and channel counts, four cameras feeding one agent
    Case("long_d48_c128", "long", 48, 128, 4, 8, 4, 4, 8, 8, ("tail", "whole", "head", "fixup2", "direct", "invalid_chunk")),
    Case("long_d64_c256", "long", 64, 256, 2, 4, 2, 1, 8, 8, ("tail", "whole", "head", "fixup2")),
    Case("cut_d16_c32", "cut", 16, 32, 4, 8, 2, 2, 8, 8, ("clean_cut", "tail_of_one", "head", "direct")),
    Case("cut_d32_c33", "cut", 32, 33, 2, 8, 2, 1, 5, 3, ("clean_cut", "tail_of_one")),
    Case("both_d33_c33", "both", 33, 33, 3, 5, 2, 1, 8, 8, ("head_and_tail", "direct", "partial_last")),
    Case("both_d48_c128", "both", 48, 128, 2, 4, 4, 2, 8, 8, ("head_and_tail", "direct")),
    Case("k128_d32_c64", "k128", 32, 64, 2, 4, 2, 2, 8, 8, ("full_then_invalid", "invalid_chunk")),
    Case("few_d1_c1", "few", 1, 1, 8, 16, 2, 2, 8, 8, ("mixed_chunk", "invalid_chunk")),
    Case("none_d16_c200", "none", 16, 200, 2, 4, 2, 2, 8, 8, ("no_valid", "invalid_chunk")),
    Case("all_d31_c256", "all", 31, 256, 3, 5, 2, 2, 7, 9, ("no_invalid", "partial_last", "tail", "head")),
    Case("agents_d64_c128", "agents", 64, 128, 2, 4, 4, 2, 8, 8, ("agent_edge", "clean_cut")),
    Case("agents_d16_c1", "agents", 16, 1, 4, 8, 2, 1, 16, 16, ("agent_edge",)),
    Case("pow2_d48_c32", "skewed", 48, 32, 4, 8, 8, 4, 16, 8, ("key_pow2", "whole", "fixup2")),
    Case("pow2m1_d32_c64", "skewed", 32, 64, 2, 4, 3, 1, 17, 5, ("key_pow2m1",)),
    Case("skewed_d48_c200", "skewed", 48, 200, 4, 8, 8, 4, 12, 10, ("whole", "fixup2", "head_and_tail", "direct")),
    # the depth softmax on its own: every point of image 0 in a cell of its own and feat = 1, so the output is prob
    Case("softmax_d31", "softmax", 31, 1, 2, 4, 2, 1, 32, 16, ("direct",)),
    Case("softmax_d32", "softmax", 32, 32, 2, 4, 2, 1, 32, 16, ("direct",)),
    Case("softmax_d33", "softmax", 33, 1, 2, 4, 2, 1, 32, 16, ("direct",)),
    Case("softmax_d64", "softmax", 64, 33, 2, 4, 2, 1, 32, 16, ("direct", "full_then_invalid")),
    # the product's size: camera_rig(2, 4, 256, 704) on the +-51.2 m / 0.4 m grid, cell from heal_lss_cell_index (GPU only)
    Case("c4", "c4", 48, 128, 32, 88, 8, 4, 256, 256, ("direct", "tail", "head", "whole", "fixup2", "head_and_tail")),
]
CASE = {c.name: c for c in CASES}
CONSTRUCTED = [c.name for c in CASES if c.map != "c4"]
C4_GRID = {"xbound": [-51.2, 51.2, 0.4], "ybound": [-51.2, 51.2, 0.4], "zbound": [-10, 10, 20.0], "ddiscr": [2, 50, 48], "mode": "LID"}


# ------------------------------------------------------------------------------------------------ inputs
def _rng(case, what):
    return np.random.default_rng(zlib.crc32(f"{what}/{case.name}".encode()))


def _runs(case):
    """Per agent, the (cell, points) runs of a constructed map in ascending cell order: the sorted point list is agent 0's runs,
    then agent 1's, then every other point (invalid).  Positions count from 0; a chunk is 128 positions."""
    last = case.cells - 1
    return {
        # cell 2 begins at slot 70 of chunk 0: a tail of 58, chunks 1 and 2 whole, a head of 7 in chunk 3
        "long": [[(1, 70), (2, 3 * CH + 7), (3, 20), (5, 9)]],
        # cell 1 ends at slot 127 and cell 2 begins at slot 0; cell 4 begins at position 255 = slot 127 of chunk 1
        "cut": [[(0, 100), (1, 28), (2, 50), (3, 77), (4, 41), (9, 3)]],
        # chunk 1 = head of cell 3 (5 points), cells 4 and 5 written directly, tail of cell 6 (53 points)
        "both": [[(2, 120), (3, 13), (4, 30), (5, 40), (6, 63), (7, 5)], [(0, 17), (3, 200)]],
        "k128": [[(0, 100), (3, 100), (4, 56)]],
        "few": [[(c, 10) for c in (0, 2, 3, 7, last)]],
        "none": [[]],
        # agent 0 ends with its last cell at slot 127 of chunk 0, agent 1 begins with cell 0 at slot 0 of chunk 1
        "agents": [[(0, 60), (last, 68)], [(0, 30), (1, 140), (last, 9)]],
    }[case.map]


def _cell(case):
    """int32 (BN, D, fH, fW): the BEV cell of every frustum point, -1 for none."""
    rng = _rng(case, "cell")
    per_agent = case.cams * case.D * case.HW
    cell = np.full((case.agents, per_agent), -1, dtype=np.int32)
    if case.map == "all":
        cell[:] = rng.integers(0, case.cells, cell.shape)
    elif case.map == "skewed":
        # most points in a few low cells, as next to a camera; a third invalid; the top cell of the last agent is hit
        c = np.floor(rng.random(cell.shape) ** 4 * case.cells).astype(np.int32)
        cell[:] = np.where(rng.random(cell.shape) < 0.33, -1, c)
        cell[-1, 5] = case.cells - 1
    elif case.map == "softmax":
        n = case.D * case.HW
        assert n <= case.cells and case.cams == 1
        cell[0] = rng.permutation(case.cells)[:n]
    else:
        for a, runs in enumerate(_runs(case)):
            # the points of a run are scattered over the agent's cameras, pixels and depth bins
            perm, pos = rng.permutation(per_agent), 0
            for c, count in runs:
                cell[a, perm[pos:pos + count]] = c
                pos += count
            assert pos <= per_agent, case.name
    return torch.from_numpy(cell.reshape(case.BN, case.D, case.fH, case.fW))


def _c4_cell():
    """The product-size cell map, from heal_lss_cell_index on the synthetic rig (needs the GPU)."""
    from heal_b200 import ops, synth
    from oracle import lss
    fr = lss.create_frustum(C4_GRID, [256, 704], 8)
    dx, bx, nx = lss.gen_dx_bx(C4_GRID["xbound"], C4_GRID["ybound"], C4_GRID["zbound"])
    rots, trans, intr, post_rots, post_trans = [torch.from_numpy(a).cuda() for a in synth.camera_rig(2, 4, 256, 704)]
    post_inv, combine = ops.lss_camera_matrices(rots, intr, post_rots)
    cell = ops.lss_cell_index(fr.cuda(), post_inv, post_trans.reshape(-1, 3), combine, trans.reshape(-1, 3),
                              (bx - dx / 2.).tolist(), dx.tolist(), nx.tolist())
    return cell.cpu()


def _inputs(case):
    """fp32 depth logits (BN, D, fH, fW) and features (BN, C, fH, fW), seeded by the case's name."""
    g = torch.Generator().manual_seed(zlib.crc32(case.name.encode()))
    logits = torch.randn(case.BN, case.D, case.fH, case.fW, generator=g) * 3
    feat = torch.randn(case.BN, case.C, case.fH, case.fW, generator=g)
    if case.map == "softmax":
        feat = torch.ones_like(feat)
    flat = logits.view(case.BN, case.D, case.HW)
    flat[0, :, 0] = 0.75                                             # all equal
    flat[0, :, 1] = torch.linspace(-80, 80, case.D) if case.D > 1 else 80.0   # the max subtraction matters
    flat[0, :, 2] = 0.0
    flat[0, case.D // 2, 2] = 30.0                                   # one dominant bin
    return logits, feat


# ------------------------------------------------------------------------------------------------ the chunk census (CPU)
def _keys(cell, cams, cells):
    """The sort keys of k_lss_keys: agent * cells + cell, or agents * cells for an invalid point."""
    BN = cell.shape[0]
    c = cell.reshape(BN, -1).numpy().astype(np.int64)
    total = (BN // cams) * cells
    agent = (np.arange(BN) // cams)[:, None]
    return np.where(c < 0, total, agent * cells + c).reshape(-1), total


def _census(cell, cams, cells):
    """Sorts the keys as heal_lss_pool_sorted does and walks the chunks as k_lss_pool_chunks does.  Returns the situations
    that occur (names of SITUATIONS) and the counts a reader optimising the kernel wants."""
    keys, total = _keys(cell, cams, cells)
    sk = np.sort(keys, kind="stable")
    n = sk.size
    found, whole_heads = set(), 0
    for base in range(0, n, CH):
        k = sk[base:base + CH]
        nvalid = int((k < total).sum())
        if len(k) < CH:
            found.add("partial_last")
        if nvalid == 0:
            found.add("invalid_chunk")
            continue
        if nvalid < len(k):
            found.add("mixed_chunk")
        v = k[:nvalid]
        started_here = base == 0 or sk[base - 1] != v[0]
        continues = nvalid == CH and base + CH < n and sk[base + CH] == v[-1]
        first_of_run = np.flatnonzero(np.r_[True, v[1:] != v[:-1]])
        whole = len(first_of_run) == 1 and not started_here and continues
        head, tail = not started_here and not whole, continues and not whole
        whole_heads += whole
        found.update(s for s, on in (("whole", whole), ("head", head), ("tail", tail), ("head_and_tail", head and tail)) if on)
        if len(first_of_run) - (not started_here) - continues + whole > 0:
            found.add("direct")
        if tail and nvalid - first_of_run[-1] == 1:
            found.add("tail_of_one")
        if nvalid == CH and not continues and base + CH < n:
            nxt = sk[base + CH]
            found.add("clean_cut" if nxt < total else "full_then_invalid")
            if nxt < total and nxt == v[-1] + 1 and nxt % cells == 0:
                found.add("agent_edge")
    valid = sk[sk < total]
    stats = dict(points=n, valid=valid.size, chunks=-(-n // CH), whole_heads=int(whole_heads), cells_hit=0, max_points=0,
                 longest_fixup=0)
    if valid.size:
        begin = np.flatnonzero(np.r_[True, valid[1:] != valid[:-1]])
        end = np.r_[begin[1:], valid.size]
        stats.update(cells_hit=begin.size, max_points=int((end - begin).max()),
                     longest_fixup=int(((end - 1) // CH - begin // CH).max()))
    if stats["longest_fixup"] >= 2:
        found.add("fixup2")
    if valid.size in (0, n):
        found.add("no_valid" if valid.size == 0 else "no_invalid")
    elif valid[-1] == total - 1:
        if total & (total - 1) == 0:
            found.add("key_pow2")
        if total & (total + 1) == 0:
            found.add("key_pow2m1")
    return found, stats


@pytest.mark.parametrize("name", CONSTRUCTED)
def test_case_produces_its_situations(name):
    case = CASE[name]
    found, stats = _census(_cell(case), case.cams, case.cells)
    assert set(case.situations) <= set(SITUATIONS)
    assert set(case.situations) <= found, f"{name}: {sorted(set(case.situations) - found)} do not occur ({stats})"


def test_cases_cover_every_situation_and_shape():
    found = set()
    for name in CONSTRUCTED:
        found |= _census(_cell(CASE[name]), CASE[name].cams, CASE[name].cells)[0]
    assert found == set(SITUATIONS), sorted(set(SITUATIONS) - found)
    assert {c.D for c in CASES} >= {1, 16, 31, 32, 33, 48, 64}
    assert {c.C for c in CASES} >= {1, 32, 33, 64, 128, 200, 256}
    assert {c.cams for c in CASES} >= {1, 2, 4}


# ------------------------------------------------------------------------------------------------ float64 reference
FAULTS = ("head2", "tail", "nvalid-1", "softmax32", "agent_image", "transposed")


def _dropped(fault, keys, total):
    """The points a summation fault loses: `head2` the head partial of the second chunk after a tail, `tail` a tail
    partial, `nvalid-1` the last valid point of every chunk."""
    order = np.argsort(keys, kind="stable")
    sk = keys[order]
    pos = np.arange(sk.size)
    valid = sk < total
    if fault == "nvalid-1":
        last = np.r_[valid[:-1] & ((pos[1:] % CH == 0) | ~valid[1:]), valid[-1]]
        return order[last]
    begin = np.flatnonzero(valid & np.r_[True, sk[1:] != sk[:-1]])
    end = np.r_[begin[1:], int(valid.sum())]
    span = (end - 1) // CH - begin // CH
    i = int(np.argmax(span >= (2 if fault == "head2" else 1)))
    chunk = begin[i] // CH + (2 if fault == "head2" else 0)
    lost = pos[max(begin[i], chunk * CH):min(end[i], (chunk + 1) * CH)]
    return order[lost]


def _reference(case, logits, feat, cell, sum_roundings=PROB_SUM_ROUNDINGS, fault=None):
    """float64 output (agents * cells, C), its bound (None with a fault), the points per cell.  `fault` restates a plausible
    kernel bug (test_bound_rejects_plausible_kernel_bugs)."""
    BN, D, HW, C, cells = case.BN, case.D, case.HW, case.C, case.cells
    total = case.agents * cells
    lg = logits.double().reshape(BN, D, HW)
    if fault == "softmax32":                       # the second register of k_lss_prob (bins 32..63) left out
        lg = lg.clone()
        lg[:, 32:] = -math.inf
    x = lg - lg.max(1, keepdim=True).values
    p = torch.softmax(x, 1)
    if fault == "transposed":                      # prob stored [pixel][D], read as [D][pixel]
        p = p.permute(0, 2, 1).reshape(BN, D, HW)
    c = cell.reshape(BN, -1).long()
    image = torch.arange(BN)[:, None].expand_as(c)
    key = (image if fault == "agent_image" else image // case.cams) * cells + c
    keep = (c >= 0) & (key < total)
    if fault in ("head2", "tail", "nvalid-1"):
        keep.view(-1)[torch.from_numpy(_dropped(fault, _keys(cell, case.cams, cells)[0], total))] = False
    pix = torch.arange(HW).repeat(D)
    F = feat.double().reshape(BN, C, HW).permute(0, 2, 1)

    def pooled(w, f):
        out = torch.zeros(total, C, dtype=torch.float64)
        w = w.reshape(BN, -1)
        for bn in range(BN):
            k = keep[bn]
            out.index_add_(0, key[bn][k], w[bn][k][:, None] * f[bn][pix[k]])
        return out

    y = pooled(p, F)
    n = torch.bincount(key[keep], minlength=total).double()
    if fault is not None:
        return y, None, n
    ax = x.abs()
    soft = 9 + sum_roundings + ax + (p * ax).sum(1, keepdim=True)
    roundings = n + torch.ceil(n / CH) + 2
    bound = U * (roundings[:, None] * pooled(p, F.abs()) + pooled(p * soft, F.abs())) \
        + n[:, None] * TINY * (1 + F.abs().max().item())
    return y, bound, n


def _ratio(err, bound):
    return torch.where(err == 0, 0.0, err / bound).max().item()


def _faults(case, found, stats):
    f = []
    if stats["valid"]:
        f.append("nvalid-1")
        if case.D > 1:
            f.append("transposed")
        if case.cams > 1:
            f.append("agent_image")
        if case.D > 32:
            f.append("softmax32")
    if "tail" in found:
        f.append("tail")
    if stats["longest_fixup"] >= 2:
        f.append("head2")
    return f


def test_bound_rejects_plausible_kernel_bugs():
    """Each plausible kernel bug, restated on the float64 reference of every constructed case (at 8 channels) it applies to,
    leaves the bound on some element: the head partial of the second chunk after a tail dropped (a fix-up that stops one chunk
    early), a tail partial dropped, the last valid point of a chunk dropped (nvalid - 1), the softmax over the first 32 depth
    bins only, the agent of a point taken as its image instead of image / cams, the probability read with D and pixel
    transposed."""
    applied = set()
    for name in CONSTRUCTED:
        case = dataclasses.replace(CASE[name], C=min(CASE[name].C, 8))
        logits, feat = _inputs(case)
        cell = _cell(case)
        y, bound, _ = _reference(case, logits, feat, cell)
        assert bool(torch.isfinite(y).all() and torch.isfinite(bound).all())
        for fault in _faults(case, *_census(cell, case.cams, case.cells)):
            d = (_reference(case, logits, feat, cell, fault=fault)[0] - y).abs()
            assert _ratio(d, bound) > 1, f"{name}: the bound does not reject '{fault}' (max err / bound {_ratio(d, bound):.3f})"
            applied.add(fault)
    assert applied == set(FAULTS)


def test_reference_is_the_oracle_pooling():
    """_reference is the per-cell sum oracle/lss.py pins to the unmodified model: softmax (x) features, summed per cell."""
    from oracle import lss
    case = dataclasses.replace(CASE["both_d48_c128"], C=8)
    logits, feat = _inputs(case)
    cell = _cell(case)
    y = _reference(case, logits, feat, cell)[0].reshape(case.agents, case.cells, case.C)
    x = lss.outer_product(logits.double(), feat.double())                                 # (BN, C, D, fH, fW)
    for a in range(case.agents):
        xa = x[a * case.cams:(a + 1) * case.cams].permute(0, 2, 3, 4, 1).reshape(-1, case.C)
        ca = cell[a * case.cams:(a + 1) * case.cams].reshape(-1).long()
        ref = torch.zeros(case.cells, case.C, dtype=torch.float64).index_add_(0, ca[ca >= 0], xa[ca >= 0])
        torch.testing.assert_close(y[a], ref, rtol=1e-12, atol=1e-14)


# ------------------------------------------------------------------------------------------------ pooling kernels (GPU)
def _bits(t):
    t = t.contiguous()
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


def _where(case, cell, flat_index):
    """The failing element's key, its point count and where its points lie in the sorted list."""
    keys, total = _keys(cell, case.cams, case.cells)
    key = flat_index // case.C
    pos = np.flatnonzero(np.sort(keys, kind="stable") == key)
    span = f"sorted positions {pos[0]}..{pos[-1]} (chunks {pos[0] // CH}..{pos[-1] // CH})" if pos.size else "no point"
    return f"key {key} (agent {key // case.cells}, cell {key % case.cells}), channel {flat_index % case.C}, {pos.size} points, {span}"


def _check(case, cell, got, y, bound, what):
    err = (got.double().reshape(y.shape) - y).abs()
    bad = ~(err <= bound)                         # NaN is bad
    ratio = _ratio(err, bound)
    print(f"{case.name} {what}: max err / bound {ratio:.4f} (max err {err.max().item():.3e}, max |y| {y.abs().max().item():.3f})")
    if bool(bad.any()):
        worst = int(torch.where(bad, err / bound.clamp_min(TINY), -1.0).argmax())
        pytest.fail(f"{case.name} {what}: {int(bad.sum())} elements outside the bound, worst at {_where(case, cell, worst)}: "
                    f"got {got.reshape(-1)[worst].item()!r}, expected {y.reshape(-1)[worst].item()!r}")
    return ratio


def _case_tensors(case):
    logits, feat = _inputs(case)
    cell = _c4_cell() if case.map == "c4" else _cell(case)
    return logits, feat, cell


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASE))
def test_pool_sorted(name):
    from heal_b200 import ops
    case = CASE[name]
    D, C, HW = case.D, case.C, case.HW
    logits, feat, cell = _case_tensors(case)
    found, stats = _census(cell, case.cams, case.cells)
    if case.map == "c4":
        print(f"c4 census: {stats}; situations {sorted(found)}")
        assert set(case.situations) <= found
    lg, ft, cl = logits.cuda(), feat.cuda(), cell.cuda()

    def run(out_fmt="f32"):
        return ops.lss_pool_sorted(lg, (D * HW, HW, 1), ft, (C * HW, HW, 1), cl, case.cams, D, C, case.fH, case.fW, case.nx,
                                   case.ny, out_fmt=out_fmt)

    a = run().t.cpu()
    assert a.shape == (case.agents, case.ny, case.nx, C)
    y, bound, n = _reference(case, logits, feat, cell)
    _check(case, cell, a, y, bound, "heal_lss_pool_sorted")
    assert bool((a.reshape(y.shape)[n == 0] == 0).all()), f"{name}: a cell nobody hits is not 0"
    # the fused channels-last heads (BN, fH, fW, D + C): the same sums in the same order
    S = D + C
    fused = torch.cat([lg.permute(0, 2, 3, 1), ft.permute(0, 2, 3, 1)], -1).contiguous()
    b = ops.lss_pool_sorted(fused, (HW * S, 1, S), fused[..., D:], (HW * S, 1, S), cl, case.cams, D, C, case.fH, case.fW,
                            case.nx, case.ny)
    assert torch.equal(_bits(b.t.cpu()), _bits(a)), f"{name}: NCHW and channels-last inputs differ"
    assert torch.equal(_bits(run().t.cpu()), _bits(a)), f"{name}: a second run differs"
    hi = a.to(torch.bfloat16)
    assert torch.equal(_bits(run("bf16").t.cpu()[0]), _bits(hi)), f"{name}: bf16 output != bf16(fp32 output)"
    s = run("split").t.cpu()
    assert torch.equal(_bits(s[0]), _bits(hi)), f"{name}: hi plane != bf16(fp32 output)"
    assert torch.equal(_bits(s[1]), _bits((a - hi.float()).to(torch.bfloat16))), f"{name}: lo plane != bf16(fp32 - hi)"


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASE))
def test_pool_atomic(name):
    """heal_lss_pool (atomicAdd, sum order not fixed) against the same reference and bound; its softmax sums D terms serially."""
    from heal_b200 import ops
    case = CASE[name]
    logits, feat, cell = _case_tensors(case)
    a = ops.lss_pool(logits.cuda(), feat.cuda(), cell.cuda(), case.cams, case.nx, case.ny).t.cpu()
    y, bound, n = _reference(case, logits, feat, cell, sum_roundings=case.D - 1)
    _check(case, cell, a, y, bound, "heal_lss_pool")
    assert bool((a.reshape(y.shape)[n == 0] == 0).all()), f"{name}: a cell nobody hits is not 0"


@pytest.mark.gpu
@pytest.mark.parametrize("what, symbol, error", [
    ("D65", "heal_lss_pool_sorted", "HEAL_ERR_UNSUPPORTED"), ("C257", "heal_lss_pool_sorted", "HEAL_ERR_ARG"),
    ("cams", "heal_lss_pool_sorted", "HEAL_ERR_ARG"), ("row_over_200KiB", "heal_lss_pool", "HEAL_ERR_UNSUPPORTED")])
def test_pool_refusals(what, symbol, error):
    """More than 64 depth bins, more than 256 channels, an image count the cameras per agent do not divide, and an image row
    beyond the atomic kernel's 200 KiB of shared memory are refused by name, and nothing is launched."""
    from heal_b200 import ops
    from heal_b200._lib import lib
    D, C, fH, fW, BN, cams = {"D65": (65, 32, 2, 4, 2, 2), "C257": (16, 257, 2, 4, 2, 2), "cams": (16, 32, 2, 4, 3, 2),
                              "row_over_200KiB": (48, 128, 1, 512, 1, 1)}[what]
    lg = torch.zeros(BN, D, fH, fW, device="cuda")
    ft = torch.zeros(BN, C, fH, fW, device="cuda")
    cl = torch.zeros(BN, D, fH, fW, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    before = lib.heal_launch_count()
    with pytest.raises(RuntimeError, match=f"{symbol} failed: {error}"):
        if symbol == "heal_lss_pool":
            ops.lss_pool(lg, ft, cl, cams, 8, 8)
        else:
            ops.lss_pool_sorted(lg, (D * fH * fW, fH * fW, 1), ft, (C * fH * fW, fH * fW, 1), cl, cams, D, C, fH, fW, 8, 8)
    torch.cuda.synchronize()
    assert lib.heal_launch_count() == before


# ------------------------------------------------------------------------------------------------ heal_lss_cell_index
def _cell_index_f32(fr, trans, lower, dx, nx):
    """numpy float32 restatement of k_lss_cell_index for post_rots^-1 = combine = I, post_trans = 0: every step is one fp32
    operation.  fr (P, 3) = (u, v, d), trans (BN, 3) -> (cell (BN, P), v (BN, P, 3) the cell coordinates)."""
    fr, trans, lower, dx = (np.asarray(a, dtype=np.float32) for a in (fr, trans, lower, dx))
    r = np.stack([fr[:, 0] * fr[:, 2], fr[:, 1] * fr[:, 2], fr[:, 2]], -1)
    v = ((r[None] + trans[:, None]) - lower) / dx
    assert v.dtype == np.float32
    tr = np.trunc(v)
    ok = ((tr >= 0) & (tr < np.asarray(nx, dtype=np.float32))).all(-1)
    i = np.where(ok[..., None], tr, 0).astype(np.int64)
    return np.where(ok, (i[..., 2] * nx[1] + i[..., 1]) * nx[0] + i[..., 0], -1), v


def _run_cell_index(fr, trans, lower, dx, nx):
    from heal_b200 import ops
    BN = len(trans)
    eye = torch.eye(3).repeat(BN, 1, 1).cuda()
    frustum = torch.from_numpy(np.asarray(fr, dtype=np.float32)).reshape(1, 1, -1, 3).cuda()
    cell = ops.lss_cell_index(frustum, eye, torch.zeros(BN, 3).cuda(), eye, torch.from_numpy(np.asarray(trans, dtype=np.float32)).cuda(),
                              list(lower), list(dx), list(nx))
    return cell.cpu().numpy().reshape(BN, -1)


@pytest.mark.gpu
def test_cell_index_exact():
    # 1. a dyadic grid, points placed by hand: d = 2, u = (x - 1) / 2, v = (y + 0.5) / 2 and one image per z, all exact
    lower, dx, nx = (-4.0, -2.0, 0.0), (0.5, 0.25, 1.0), (16, 12, 3)

    def targets(j):
        below = float(np.nextafter(np.float32(nx[j]), np.float32(0)))
        vs = [0.0, 3.0, 2.5, -0.5, -2.0 ** -20, -1.0, -1.25, float(nx[j]), below, nx[j] - 0.5, nx[j] + 3.0]
        return vs, [lower[j] + v * dx[j] for v in vs]

    (vx, xs), (vy, ys), (vz, zs) = targets(0), targets(1), targets(2)
    fr = [((x - 1.0) / 2, (y + 0.5) / 2, 2.0) for y in ys for x in xs]
    trans = [(1.0, -0.5, z - 2.0) for z in zs]
    want, v = _cell_index_f32(fr, trans, lower, dx, nx)
    expect_v = np.array([[(a, b, c) for b in vy for a in vx] for c in vz])
    assert np.array_equal(v.astype(np.float64), expect_v), "the hand-placed points are not where they were meant to be"
    inside = lambda t, n: (t > -1) & (t < n)                           # truncation toward zero keeps (-1, 0) in cell 0
    ok = np.all([inside(expect_v[..., j], nx[j]) for j in range(3)], 0)
    assert np.array_equal(want >= 0, ok)
    for j in range(3):                                                  # out on one axis only, for each axis
        others = np.all([inside(expect_v[..., k], nx[k]) for k in range(3) if k != j], 0)
        assert bool((others & ~inside(expect_v[..., j], nx[j])).any())
    zero_cell = np.all((expect_v > -1) & (expect_v < 0), -1)
    assert bool(zero_cell.any()) and bool((want[zero_cell] == 0).all())
    got = _run_cell_index(fr, trans, lower, dx, nx)
    assert np.array_equal(got, want), f"{int((got != want).sum())} of {want.size} hand-placed points differ"
    assert got.max() == (2 * nx[1] + nx[1] - 1) * nx[0] + nx[0] - 1      # (z ny + y) nx + x at the far corner
    # 2. the product's grid spacing with three z slices, random points: still one rounding per step
    rng = np.random.default_rng(11)
    lower, dx, nx = (-51.2, -51.2, -10.0), (0.4, 0.4, 20.0 / 3), (256, 256, 3)
    fr = np.stack([rng.uniform(-1.5, 1.5, 20000), rng.uniform(-1.5, 1.5, 20000), rng.uniform(2, 50, 20000)], -1)
    trans = [(0.0, 0.0, -20.0), (1.5, -0.25, -30.0), (-3.1, 7.7, -8.0), (0.4, 0.8, -12.0)]
    want, _ = _cell_index_f32(fr, trans, lower, dx, nx)
    got = _run_cell_index(fr, trans, lower, dx, nx)
    print(f"cell index, random points: {(want >= 0).mean():.2f} inside the grid")
    assert 0.2 < (want >= 0).mean() < 0.9
    assert np.array_equal(got, want), f"{int((got != want).sum())} of {want.size} random points differ"


def _augmented_rig(n_agents, seed):
    """camera_rig with what the data augmentation and real calibrations add: post_rots = resize 0.3..0.5 x optional horizontal flip
    x a rotation of up to 5.4 degrees, the matching crop offsets, ego rotations off the axes, focal lengths that follow the resize, and rigs 15 to 30 m off the grid's centre."""
    from heal_b200 import synth
    rots, trans, intr, post_rots, post_trans = [torch.from_numpy(a).double() for a in synth.camera_rig(n_agents, 4, 256, 704)]
    rng = np.random.default_rng(seed)
    for a in range(n_agents):
        shift = np.r_[rng.uniform(15, 30, 2) * rng.choice([-1, 1], 2), 0]   # off centre: part of every frustum leaves the grid
        for c in range(4):
            s, flip, th = rng.uniform(0.3, 0.5), rng.random() < 0.5, rng.uniform(-0.094, 0.094)
            R2 = np.array([[np.cos(th), -np.sin(th)], [np.sin(th), np.cos(th)]]) @ np.diag([-s if flip else s, s])
            post_rots[a, c, :2, :2] = torch.from_numpy(R2)
            post_trans[a, c, :2] = torch.tensor([704.0 if flip else rng.uniform(-40, 0), rng.uniform(-60, 0)])
            intr[a, c, :2] /= s                                         # the original image is 1 / s times larger
            w = rng.uniform(-0.05, 0.05, 3)                             # a small rotation of the camera in the ego frame
            K = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
            rots[a, c] = torch.linalg.matrix_exp(torch.from_numpy(K)) @ rots[a, c]
            trans[a, c] += torch.from_numpy(shift + rng.uniform(-0.3, 0.3, 3))
    return [t.float() for t in (rots, trans, intr, post_rots, post_trans)]


@pytest.mark.gpu
def test_cell_index_vs_float64():
    """Rotated, scaled and flipped cameras at the product's size, all 8 images.  The reference is the same chain in float64 on the
    fp32 matrices the kernel reads.  Every index must be the truncation of the float64 cell coordinate moved by at most eps
    on each axis, eps = 16 u (sum of the magnitudes of the terms) / dx (15 roundings, module docstring): a point that differs from the float64 truncation lies
    within eps of a cell edge and lands in the neighbouring cell on that axis, or flips valid / invalid at the grid's edge."""
    from heal_b200 import ops
    from oracle import lss
    fr = lss.create_frustum(C4_GRID, [256, 704], 8)
    dx, bx, nx = lss.gen_dx_bx(C4_GRID["xbound"], C4_GRID["ybound"], C4_GRID["zbound"])
    lower = bx - dx / 2.
    rots, trans, intr, post_rots, post_trans = [t.cuda() for t in _augmented_rig(2, 5)]
    post_inv, combine = ops.lss_camera_matrices(rots, intr, post_rots)
    cell = ops.lss_cell_index(fr.cuda(), post_inv, post_trans.reshape(-1, 3), combine, trans.reshape(-1, 3), lower.tolist(),
                              dx.tolist(), nx.tolist()).cpu().reshape(8, -1)
    A, Cm = post_inv.cpu().double()[:, None], combine.cpu().double()[:, None]            # (8, 1, 3, 3)
    pt, t = post_trans.cpu().double().reshape(8, 1, 3), trans.cpu().double().reshape(8, 1, 3)
    f = fr.double().reshape(1, -1, 3)
    p = f - pt
    q = (A * p[..., None, :]).sum(-1)
    q_mag = (A.abs() * (f.abs() + pt.abs())[..., None, :]).sum(-1)
    r = torch.cat([q[..., :2] * q[..., 2:], q[..., 2:]], -1)
    r_mag = torch.cat([q_mag[..., :2] * q_mag[..., 2:], q_mag[..., 2:]], -1)
    e = (Cm * r[..., None, :]).sum(-1) + t
    mag = (Cm.abs() * r_mag[..., None, :]).sum(-1) + t.abs() + lower.double().abs()
    v = (e - lower.double()) / dx.double()                                                # (8, P, 3) cell coordinates
    eps = 16 * U * mag / dx.double()
    n3 = nx.double()
    lo, hi, mid = torch.trunc(v - eps), torch.trunc(v + eps), torch.trunc(v)
    out = lambda tr: (tr < 0) | (tr >= n3)
    exact_ok = ~out(mid).any(-1)
    exact = torch.where(exact_ok, (mid[..., 2] * n3[1] + mid[..., 1]) * n3[0] + mid[..., 0], -1.0).long()
    mism = cell.long() != exact
    in_grid = exact_ok | (cell >= 0)
    print(f"cell index, augmented rig: {int(mism.sum())} of {mism.numel()} differ from the float64 truncation "
          f"({mism.double().mean().item():.2e}); {exact_ok.double().mean().item():.2f} inside the grid; "
          f"largest eps in the grid {eps[in_grid].max().item():.2e} cells")
    assert 0.2 < exact_ok.double().mean().item() < 0.95
    assert mism.double().mean().item() < 2e-4
    c = cell.long()
    got = torch.stack([c % nx[0], (c // nx[0]) % nx[1], c // (nx[0] * nx[1])], -1).double()
    valid_fits = ((got >= lo) & (got <= hi)).all(-1)
    invalid_fits = (out(lo) | out(hi)).any(-1)
    fits = torch.where(cell >= 0, valid_fits, invalid_fits)
    assert bool(fits.all()), f"{int((~fits).sum())} indices are not the float64 coordinate moved by eps"
    assert bool((eps[in_grid] < 1e-2).all())


# ------------------------------------------------------------------------------------------------ heal_lss_camera_matrices
@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 64, 65])
def test_camera_matrices(n):
    """Against the float64 inverse of the fp32 inputs, for post_rots with a resize of 0.3..0.5, a horizontal flip (negative
    determinant) and a small rotation, focal lengths from 200 to 3000 px, and image counts on either side of the 64-thread
    block.  post_rots^-1 is the float64 adjugate rounded once: within 2 u of the exact entry, stated against the largest entry
    (a zero entry of the exact inverse may come out as rounding noise of the float64 adjugate).  combine = rots @ K^-1 is an
    fp32 product of the rounded inverse: one rounding of each K^-1 entry and three of the fma chain, so entry (r, k) is within
    4 u sum_j |rots_rj| |K^-1_jk| of the exact product."""
    from heal_b200 import ops
    rng = np.random.default_rng(100 + n)
    rots, intr, post = np.zeros((n, 3, 3)), np.zeros((n, 3, 3)), np.zeros((n, 3, 3))
    for i in range(n):
        rots[i] = np.linalg.qr(rng.normal(size=(3, 3)))[0]
        f = 200.0 * 15.0 ** (i / max(n - 1, 1)) if n > 1 else 1266.4
        intr[i] = [[f, 0, rng.uniform(300, 900)], [0, f * rng.uniform(0.98, 1.02), rng.uniform(150, 500)], [0, 0, 1]]
        s, th, flip = rng.uniform(0.3, 0.5), rng.uniform(-0.094, 0.094), i % 2 == 1
        post[i] = np.eye(3)
        post[i, :2, :2] = np.array([[np.cos(th), -np.sin(th)], [np.sin(th), np.cos(th)]]) @ np.diag([-s if flip else s, s])
    rots, intr, post = (torch.from_numpy(a).float() for a in (rots, intr, post))
    assert n == 1 or bool((torch.linalg.det(post.double())[1::2] < 0).all())
    pi, cb = ops.lss_camera_matrices(rots.cuda(), intr.cuda(), post.cuda())
    pi_ref = torch.inverse(post.double())
    k_inv = torch.inverse(intr.double())
    cb_ref = rots.double() @ k_inv
    e_pi = (pi.cpu().double() - pi_ref).abs() / (2 * U * pi_ref.abs().amax((1, 2), keepdim=True))
    e_cb = (cb.cpu().double() - cb_ref).abs() / (4 * U * (rots.double().abs() @ k_inv.abs()))
    print(f"camera matrices, n = {n}: post_rots^-1 err / bound {e_pi.max().item():.3f}, combine err / bound {e_cb.max().item():.3f}")
    assert pi.shape == (n, 3, 3) and cb.shape == (n, 3, 3)
    assert e_pi.max().item() <= 1 and e_cb.max().item() <= 1
