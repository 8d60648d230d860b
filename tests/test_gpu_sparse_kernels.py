"""The sparse kernels of csrc/spconv.cu, csrc/spconv_tc.cu and csrc/sparse_stem.cu against float64 or exact references, on
inputs built for the places they can go wrong.

Rulebooks (exact).  The specification is restated in numpy and compared integer for integer:
  SubM   nbr[i][k] = row of the live site coords[i] + (k - centre), else -1; rows at or beyond the live count are not written.
  strided: an output site exists where some live (row i, offset k) proposes it (c + pad - d divisible by the stride and
         inside the output grid, out = floor((in + 2 pad - k) / stride) + 1); sites are ordered by their smallest proposer id
         i K + k; nbr[row][k] = the proposing input row, -1 elsewhere and on every row beyond the output count; the output
         count is the number of sites even past the capacity (rows >= capacity are dropped, the count reports them).
  the hash tables: the occupied slots are those of a sequential linear-probing insertion of the same keys (the set of
         occupied slots of linear probing does not depend on the insertion order), each holding one live key and its row.
sp_hash is restated (multiplicative hash, 2^max(10, ceil(log2 2 capacity)) slots) so that constructed sites can aim at chosen
slots: _sites places keys whose home is the table's last slot (a probe that wraps) and a run of homes across the table's end
(a long cluster); _rulebook_census names what occurs.  The dead rows behind a live count hold valid but wrong sites
(duplicates of live sites, other in-range sites, row 0's site), so a kernel that ignores the count fails an assertion
instead of reading out of bounds.

Gather-GEMMs (float64, per element).  y[r] = bias + sum_k a[nbr[r][k]] . W[k], then ReLU; n_r = hits of row r.
  heal_spconv_gather_gemm (fp32 FMA chain per output, then one add of the bias):
        |err| <= u (n_r Cin + 1) (sum |a w| + |b|),  u = 2^-24 (first order: each of the n_r Cin + 1 roundings is at most u
        times a partial sum no larger than sum |a w| + |b|; ReLU does not increase an error).
  heal_spconv_gather_gemm_tc (split bf16 operands, three bf16 products per pair, fp32 accumulation in the tensor cores):
        |err| <= ALPHA sum |a| |w| + REL |y|, ALPHA = 2^-16, REL = 2^-22, the bound of test_gpu_conv_epilogue.py.  The input a
        is hi + lo of the split rows the kernel reads, the weights are the fp32 weights (their split is part of what is tested).
        The split output is exactly hi = bf16(v), lo = bf16(v - hi) of the same run's fp32 output v.
  The tensor-core kernel skips every K-block (64 / Cin offsets side by side) no row of a 128-row tile hits and runs tiles
  persistently on min(ceil(capacity / 128), 132) CTAs; _tc_census walks that tiling on the CPU and names what occurs: empty
  tiles, a tile whose only active K-block is not block 0, gaps, padding offsets, three tiles per CTA, a tile whose active
  K-block count leaves the stage ring mid-way for the next tile.
Sparse stem (3x3 stride-2 pad-1 conv + folded BN + ReLU and the 1x1 stride-2 downsample from a cell -> pillar-row id map):
  heal_sparse_stem starts from the bias and chains fp32 FMAs: the same u (n 64 + 1) (sum |a w| + |b|) bound, n = hits of the
  pixel.  heal_sparse_stem_tc (mma.sync, split operands): the ALPHA / REL bound.  A pixel with no centre hit has the
  downsample's bias exactly; a pixel with no hit at all ReLU(bias) exactly.  bf16 and split outputs are the rounding of the
  same kernel's f32 output, bit for bit, written into channel views (even offset, wider stride) whose other channels keep
  their sentinel.
Helpers (exact): heal_rows_to_split against a numpy round-to-nearest-even emulation, heal_sparse_to_bev, heal_pillar_idmap,
heal_stem_rulebook.

test_bound_rejects_plausible_kernel_bugs (no GPU) restates each plausible kernel bug on the float64 reference and shows that
the bound rejects it.  What the GPU tests printed on an H100 80GB HBM3 at a 700 W power limit is kept in MEASURED below."""
import math
import re
import zlib
from dataclasses import dataclass
from pathlib import Path
from typing import Tuple

import numpy as np
import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]
CSRC = ROOT / "heal_b200" / "csrc"

U = 2.0 ** -24
ALPHA = 2.0 ** -16
REL = 2.0 ** -22
NUM_SMS = 132              # HEAL_NUM_SMS: CTAs of the persistent tensor-core kernel
SPT_M = 128                # rows per tile of k_spconv_tc
SP_SCAN = 1024             # rows per block of the strided rulebook's scan
SP_BLOCK = 32              # rows per block of k_sp_gather_gemm
EMPTY = 0xFFFFFFFF
SENT = 0x5A5A5A5A          # int32 / fp32 sentinel bits of outputs that must stay untouched (fp32: 1.5e16, finite)
SENT16 = 0x5A5A            # bf16 sentinel bits

# What the GPU tests print, on an H100 80GB HBM3 at a 700 W power limit (err / bound of 0 means an exact output).
MEASURED = """
rulebooks, 13 cases (SubM (3,3,3) (3,1,1) (1,3,3) (1,1,1); strided (3,3,3)/2/(1,1,1), (3,3,3)/2/(0,1,1), (3,1,1)/(2,1,1)/0):
    exact; e.g. strided_p111_hash 2389 live of 2509 -> 7676 sites, 7903 pairs; strided_one_over 887 sites on a capacity of 886
heal_spconv_gather_gemm, 7 instantiations x bias x ReLU, largest err / bound 0.246 ((4,16), no bias, no ReLU); per
    instantiation (4,16) 0.246, (16,16) 0.090, (16,32) 0.082, (32,32) 0.044, (32,64) 0.068, (64,64) 0.032, (64,128) K 3 0.065
heal_spconv_gather_gemm_tc, 11 cases, largest err / bound 0.544 (tc16x32_k27_big: 399 tiles on 132 CTAs); per case
    tc16x16_k27 0.346, tc16x32_k27_big 0.544, tc32x32_k27 0.292, tc32x64_k27 0.382, tc64x64_k27 0.248, tc64x128_k27 0.214,
    tc64x128_k3_big 0.292, tc64x64_k9_planar 0.192, tc64x64_k1_planar 0.229, tc16x32_k5 0.424, tc32x64_k3 0.360
    (max err 1.8e-05 at max |y| 6.3); split outputs equal the rounding of the fp32 output bit for bit
heal_sparse_stem (conv / down): taps 0.128 / 0.045, border_b3 0.104 / 0.070, hi_only 0.053 / 0.053, empty 0 / 0,
    random_nx44 0.074 / 0.068
heal_sparse_stem_tc (conv / down): taps 0.193 / 0.174, border_b3 0.268 / 0.245, hi_only 0.142 / 0.195, empty 0 / 0
helpers (heal_rows_to_split, heal_sparse_to_bev, heal_pillar_idmap, heal_stem_rulebook): exact; 19 refusals, nothing launched
"""


def _rng(name, what):
    return np.random.default_rng(zlib.crc32(f"{what}/{name}".encode()))


def _ratio(err, bound):
    err, bound = np.asarray(err, dtype=np.float64), np.asarray(bound, dtype=np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(err == 0, 0.0, err / bound)
    return float(np.nanmax(np.where(np.isnan(r), np.inf, r))) if r.size else 0.0


# ================================================================================================ hash and rulebooks
def table_log2(n):
    lg = 10
    while (1 << lg) < 2 * n:
        lg += 1
    return lg


def sp_hash(keys, lg):
    """sp_hash of spconv.cu: (key * 2654435761 mod 2^32) >> (32 - lg)."""
    return ((np.asarray(keys, dtype=np.uint64) * np.uint64(2654435761)) & np.uint64(EMPTY)) >> np.uint64(32 - lg)


def sp_key(c, shape):
    c = np.asarray(c, dtype=np.int64).reshape(-1, 4)
    return ((c[:, 0] * shape[0] + c[:, 1]) * shape[1] + c[:, 2]) * shape[2] + c[:, 3]


def _decode(keys, shape):
    k = np.asarray(keys, dtype=np.int64)
    x = k % shape[2]; k = k // shape[2]
    y = k % shape[1]; k = k // shape[1]
    z = k % shape[0]
    return np.stack([k // shape[0], z, y, x], 1).astype(np.int32)


def _occupancy(keys, lg):
    """Occupied slots after inserting `keys` by linear probing, and the longest run of occupied slots (circular)."""
    T = 1 << lg
    occ = np.zeros(T, dtype=bool)
    for h in sp_hash(keys, lg).tolist():
        s = h
        while occ[s]:
            s = (s + 1) & (T - 1)
        occ[s] = True
    if occ.all():
        return occ, T
    d = np.r_[occ, occ].astype(np.int8)
    edges = np.flatnonzero(np.diff(np.r_[0, d, 0]))
    return occ, int(min((edges[1::2] - edges[0::2]).max(initial=0), T))


def _oshape(shape, ks, st, pd):
    return [(shape[i] + 2 * pd[i] - ks[i]) // st[i] + 1 for i in range(3)]


def _offsets(ks):
    K = ks[0] * ks[1] * ks[2]
    k = np.arange(K)
    return np.stack([k // (ks[1] * ks[2]), (k // ks[2]) % ks[1], k % ks[2]], 1)


def _lookup(sorted_keys, rows_of_sorted, q):
    pos = np.clip(np.searchsorted(sorted_keys, q), 0, max(len(sorted_keys) - 1, 0))
    if len(sorted_keys) == 0:
        return np.full(q.shape, -1, dtype=np.int32)
    return np.where(sorted_keys[pos] == q, rows_of_sorted[pos], -1).astype(np.int32)


def subm_ref(live, shape, ks):
    """nbr (n, K): row of the site live[i] + (offset - centre), else -1."""
    keys = sp_key(live, shape)
    order = np.argsort(keys)
    off = _offsets(ks) - np.array(ks) // 2
    c = live[:, None, 1:].astype(np.int64) + off[None]
    inside = ((c >= 0) & (c < np.array(shape))).all(-1)
    q = ((live[:, None, 0].astype(np.int64) * shape[0] + c[..., 0]) * shape[1] + c[..., 1]) * shape[2] + c[..., 2]
    r = _lookup(keys[order], order, q)
    return np.where(inside, r, -1).astype(np.int32)


def _proposals(live, shape, ks, st, pd):
    """Every (proposer id t = i K + k, output key) of the live rows, and whether some proposal left the output grid on the high
    side (a last plane the output extent drops)."""
    osh = _oshape(shape, ks, st, pd)
    K = ks[0] * ks[1] * ks[2]
    n = live.shape[0]
    num = live[:, None, 1:].astype(np.int64) + np.array(pd) - _offsets(ks)[None]
    ok = ((num >= 0) & (num % np.array(st) == 0)).all(-1)
    o = num // np.array(st)
    inside = ok & (o < np.array(osh)).all(-1)
    dropped = bool((ok & ~inside).any())
    t = np.arange(n * K, dtype=np.int64).reshape(n, K)
    b = np.broadcast_to(live[:, None, 0].astype(np.int64), (n, K))
    okey = ((b * osh[0] + o[..., 0]) * osh[1] + o[..., 1]) * osh[2] + o[..., 2]
    return t[inside], okey[inside], osh, dropped


def strided_ref(live, shape, ks, st, pd):
    """(output coords in the kernel's order, nbr (n_out, K), output keys in row order, rows generated first per input row)."""
    K = ks[0] * ks[1] * ks[2]
    t, okey, osh, _ = _proposals(live, shape, ks, st, pd)
    sites, inv = np.unique(okey, return_inverse=True)
    first = np.full(len(sites), np.iinfo(np.int64).max)
    np.minimum.at(first, inv, t)
    order = np.argsort(first, kind="stable")
    row = np.empty(len(sites), dtype=np.int64)
    row[order] = np.arange(len(sites))
    nbr = np.full((len(sites), K), -1, dtype=np.int32)
    nbr[row[inv], t % K] = t // K
    gen = np.bincount(first[order] // K, minlength=live.shape[0]) if len(sites) else np.zeros(live.shape[0], dtype=np.int64)
    return _decode(sites[order], osh), nbr, sites[order], gen


RULEBOOK_SITUATIONS = (
    "probe_wrap",          # two or more keys whose home slot is the last slot of the table
    "long_cluster",        # 32 or more consecutive occupied slots
    "batch_alias",         # equal (z, y, x) under different batch indices
    "grid_edge",           # live sites on z = 0 and Z - 1, y = 0 and Y - 1, x = 0 and X - 1
    "many_proposers",      # an output site proposed by 8 or more (row, offset) pairs
    "scan_block_edge",     # more than 1024 input rows, rows 1023 and 1024 both generate an output site
    "exact_capacity",      # output rows = capacity
    "one_over",            # output rows = capacity + 1
    "dead_tail",           # a live count below the capacity, the rows behind it poisoned
    "empty",               # a live count of 0
    "plane_dropped",       # a live site proposes a site beyond the output grid (the output extent drops a last plane)
)


@dataclass(frozen=True)
class RCase:
    name: str
    kind: str                     # 'subm' | 'strided'
    shape: Tuple[int, int, int]
    batch: int
    ksize: Tuple[int, int, int]
    stride: Tuple[int, int, int]
    pad: Tuple[int, int, int]
    n_rand: int                   # random live sites (before the constructed ones)
    tail: int                     # poisoned rows behind the live count
    out_cap: object               # strided: an int, 'exact' (= output rows) or 'one_over' (= output rows - 1)
    build: Tuple[str, ...]        # constructions: 'hash' (wrap + cluster), 'alias', 'edges', 'block' (27 proposers)
    situations: Tuple[str, ...]

    @property
    def K(self):
        return self.ksize[0] * self.ksize[1] * self.ksize[2]


S1 = (1, 1, 1)
RCASES = [
    RCase("subm333_hash", "subm", (21, 40, 40), 2, (3, 3, 3), S1, (0, 0, 0), 1400, 150, None, ("hash", "alias", "edges"),
          ("probe_wrap", "long_cluster", "batch_alias", "grid_edge", "dead_tail")),
    RCase("subm311", "subm", (11, 16, 16), 3, (3, 1, 1), S1, (0, 0, 0), 900, 40, None, ("alias", "edges"),
          ("batch_alias", "grid_edge", "dead_tail")),
    RCase("subm133", "subm", (5, 40, 40), 2, (1, 3, 3), S1, (0, 0, 0), 1100, 33, None, ("hash", "edges"),
          ("probe_wrap", "long_cluster", "grid_edge", "dead_tail")),
    RCase("subm111", "subm", (7, 9, 11), 4, (1, 1, 1), S1, (0, 0, 0), 600, 1, None, ("alias", "edges"),
          ("batch_alias", "grid_edge", "dead_tail")),
    RCase("subm_empty", "subm", (11, 16, 16), 1, (3, 3, 3), S1, (0, 0, 0), 0, 64, None, (), ("empty", "dead_tail")),
    # conv2.0 / conv3.0 of VoxelBackBone8x: y and x drop a last plane (160 and 140 are even), z does not (41)
    RCase("strided_p111_hash", "strided", (41, 160, 140), 2, (3, 3, 3), (2, 2, 2), (1, 1, 1), 2300, 120, 12000,
          ("hash", "alias", "edges", "block"),
          ("probe_wrap", "long_cluster", "batch_alias", "grid_edge", "many_proposers", "scan_block_edge", "dead_tail",
           "plane_dropped")),
    RCase("strided_p111_odd", "strided", (21, 41, 39), 1, (3, 3, 3), (2, 2, 2), (1, 1, 1), 1500, 0, 6000, ("edges", "block"),
          ("grid_edge", "many_proposers", "scan_block_edge")),
    # conv4.0: no z padding
    RCase("strided_p011", "strided", (11, 200, 160), 3, (3, 3, 3), (2, 2, 2), (0, 1, 1), 1200, 77, 8000, ("hash", "alias", "edges"),
          ("probe_wrap", "long_cluster", "batch_alias", "grid_edge", "scan_block_edge", "dead_tail", "plane_dropped")),
    # conv_out: (3,1,1) / (2,1,1) / 0 on 5 and on 6 z planes
    RCase("strided_z311", "strided", (5, 32, 32), 3, (3, 1, 1), (2, 1, 1), (0, 0, 0), 1300, 50, 4000, ("alias", "edges"),
          ("batch_alias", "grid_edge", "scan_block_edge", "dead_tail")),
    RCase("strided_z311_even", "strided", (6, 16, 16), 2, (3, 1, 1), (2, 1, 1), (0, 0, 0), 700, 20, 2000, ("edges",),
          ("grid_edge", "dead_tail", "plane_dropped")),
    RCase("strided_exact", "strided", (21, 32, 32), 2, (3, 3, 3), (2, 2, 2), (1, 1, 1), 300, 30, "exact", ("edges", "block"),
          ("exact_capacity", "many_proposers", "dead_tail")),
    RCase("strided_one_over", "strided", (21, 32, 32), 2, (3, 3, 3), (2, 2, 2), (1, 1, 1), 300, 30, "one_over", ("edges",),
          ("one_over", "dead_tail")),
    RCase("strided_empty", "strided", (11, 16, 16), 2, (3, 3, 3), (2, 2, 2), (1, 1, 1), 0, 40, 64, (), ("empty", "dead_tail")),
]
RCASE = {c.name: c for c in RCASES}


def _in_table_geom(case):
    """(shape, batch, table log2, key -> input site) of the table a case's hash construction aims at."""
    if case.kind == "subm":
        return list(case.shape), table_log2(case.n_rand + case.tail + 200), lambda o: o
    osh = _oshape(case.shape, case.ksize, case.stride, case.pad)

    def to_input(o):                 # the input site o * stride proposes o (through the offset d = pad)
        i = o.copy()
        i[:, 1:] = o[:, 1:] * np.array(case.stride)
        return i
    return osh, table_log2(case.out_cap), to_input


def _sites(case):
    """(coords (capacity, 4) int32: the live sites, then the poisoned tail; the live count)."""
    rng = _rng(case.name, "sites")
    shape, B = np.array(case.shape), case.batch
    cells = B * int(np.prod(shape))
    keys = list(rng.choice(cells, size=case.n_rand, replace=False)) if case.n_rand else []
    extra = []
    if "hash" in case.build:
        gshape, lg, to_input = _in_table_geom(case)
        T = 1 << lg
        allk = np.arange(B * int(np.prod(gshape)), dtype=np.int64)
        home = sp_hash(allk, lg).astype(np.int64)
        wrap = allk[home == T - 1]
        pick = list(rng.choice(wrap, min(3, wrap.size), replace=False))                 # probes that wrap
        for s in list(range(T - 24, T)) + list(range(24)):                               # homes across the table's end
            cand = allk[home == s]
            if cand.size:
                pick.append(int(rng.choice(cand)))
        extra.append(to_input(_decode(pick, gshape)))
    block = np.zeros(0, dtype=np.int64)
    if "block" in case.build:                        # a dense 3x3x3 block around an even site: its centre has 27 proposers
        c0 = (shape // 2) & ~1
        g = np.stack(np.meshgrid(*[np.arange(-1, 2)] * 3, indexing="ij"), -1).reshape(-1, 3) + c0
        block = sp_key(np.c_[np.zeros(27, dtype=np.int64), g], shape)
    if "edges" in case.build:
        e = []
        for ax in range(3):
            for v in (0, shape[ax] - 1):
                c = [int(rng.integers(B))] + [int(rng.integers(shape[j])) for j in range(3)]
                c[1 + ax] = int(v)
                e.append(c)
        extra.append(np.array(e, dtype=np.int64))
    if "alias" in case.build and keys:
        a = _decode(keys[:6], shape).astype(np.int64)
        a[:, 0] = (a[:, 0] + 1) % B
        extra.append(a)
    if extra:
        keys += sp_key(np.concatenate(extra), shape).tolist()
    rest = np.setdiff1d(np.asarray(keys, dtype=np.int64), block)
    keys = np.r_[block, rest[rng.permutation(rest.size)]]     # the block's rows first, away from the scan's block boundary
    live = _decode(keys, shape)
    n = live.shape[0]
    tail = []
    for j in range(case.tail):                       # valid but wrong: a live site, another in-range site, row 0's site
        kind = j % 3 if n else 1
        if kind == 0:
            tail.append(live[rng.integers(n)])
        elif kind == 1:
            while True:
                k = int(rng.integers(cells))
                if not np.isin(k, keys):
                    break
            tail.append(_decode([k], shape)[0])
        else:
            tail.append(live[0])
    coords = np.concatenate([live, np.array(tail, dtype=np.int32).reshape(-1, 4)]).astype(np.int32)
    return np.ascontiguousarray(coords), n


def _out_capacity(case, n_out):
    return {"exact": max(n_out, 1), "one_over": n_out - 1}.get(case.out_cap, case.out_cap)


def _rulebook_census(case):
    coords, n = _sites(case)
    live = coords[:n]
    found, stats = set(), dict(live=n, capacity=coords.shape[0])
    if n < coords.shape[0]:
        found.add("dead_tail")
    if n == 0:
        found.add("empty")
    shape = np.array(case.shape)
    if n:
        edge = all(((live[:, 1 + a] == 0).any() and (live[:, 1 + a] == shape[a] - 1).any()) for a in range(3))
        if edge:
            found.add("grid_edge")
        zyx = sp_key(np.c_[np.zeros(n, dtype=np.int64), live[:, 1:]], shape)
        per_site = {}
        for z, b in zip(zyx.tolist(), live[:, 0].tolist()):
            per_site.setdefault(z, set()).add(b)
        if any(len(v) > 1 for v in per_site.values()):
            found.add("batch_alias")
    if case.kind == "subm":
        lg, keys = table_log2(coords.shape[0]), sp_key(live, shape)
    else:
        oc, nbr, okeys, gen = strided_ref(live, list(case.shape), case.ksize, case.stride, case.pad)
        cap = _out_capacity(case, len(okeys))
        lg, keys = table_log2(cap), okeys
        stats.update(out_rows=len(okeys), out_capacity=cap, max_proposers=int((nbr >= 0).sum(1).max(initial=0)))
        if len(okeys) == cap:
            found.add("exact_capacity")
        if len(okeys) == cap + 1:
            found.add("one_over")
        if stats["max_proposers"] >= 8:
            found.add("many_proposers")
        if n > SP_SCAN and gen[SP_SCAN - 1] > 0 and gen[SP_SCAN] > 0:
            found.add("scan_block_edge")
        if _proposals(live, list(case.shape), case.ksize, case.stride, case.pad)[3]:
            found.add("plane_dropped")
    if len(keys):
        T = 1 << lg
        if int((sp_hash(keys, lg) == T - 1).sum()) >= 2:
            found.add("probe_wrap")
        _, run = _occupancy(keys, lg)
        stats["longest_cluster"] = run
        if run >= 32:
            found.add("long_cluster")
    return found, stats


@pytest.mark.parametrize("name", list(RCASE))
def test_rulebook_case_produces_its_situations(name):
    case = RCASE[name]
    found, stats = _rulebook_census(case)
    assert set(case.situations) <= set(RULEBOOK_SITUATIONS)
    assert set(case.situations) <= found, f"{name}: {sorted(set(case.situations) - found)} do not occur ({stats})"


def test_rulebook_cases_cover_every_situation():
    found = set()
    for c in RCASES:
        found |= _rulebook_census(c)[0]
    assert found == set(RULEBOOK_SITUATIONS), sorted(set(RULEBOOK_SITUATIONS) - found)
    assert {c.ksize for c in RCASES if c.kind == "subm"} == {(3, 3, 3), (3, 1, 1), (1, 3, 3), (1, 1, 1)}
    assert {(c.ksize, c.stride, c.pad) for c in RCASES if c.kind == "strided"} == {
        ((3, 3, 3), (2, 2, 2), (1, 1, 1)), ((3, 3, 3), (2, 2, 2), (0, 1, 1)), ((3, 1, 1), (2, 1, 1), (0, 0, 0))}


# ------------------------------------------------------------------------------------------------ rulebooks (GPU)
def _i32(shape, fill=SENT):
    return torch.full(shape, fill, dtype=torch.int32, device="cuda")


def _check_table(keys_t, vals_t, want_keys, want_rows, lg, what):
    keys = keys_t.cpu().numpy().view(np.uint32).astype(np.int64)
    vals = vals_t.cpu().numpy()
    occ = keys != EMPTY
    assert keys.size == 1 << lg, f"{what}: table of {keys.size} slots, expected 2^{lg}"
    assert np.array_equal(occ, _occupancy(want_keys, lg)[0]), f"{what}: the occupied slots are not those of linear probing"
    got = dict(zip(keys[occ].tolist(), vals[occ].tolist()))
    assert got == dict(zip(np.asarray(want_keys).tolist(), np.asarray(want_rows).tolist())), f"{what}: table keys / rows differ"


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(RCASE))
def test_rulebook(name):
    from heal_b200 import ops
    from heal_b200._lib import lib
    case = RCASE[name]
    coords, n = _sites(case)
    cap, K, shape = coords.shape[0], case.K, list(case.shape)
    live = coords[:n]
    cd = torch.from_numpy(coords).cuda()
    rows = torch.tensor([n], dtype=torch.int32, device="cuda")
    st = ops.SparseTensor(None, cd, rows, shape, case.batch)
    if case.kind == "subm":
        keys, vals = ops.sp_build_table(st)
        _check_table(keys, vals, sp_key(live, shape), np.arange(n), table_log2(cap), f"{name} input table")
        nbr = _i32((cap, K))
        ops._call("heal_spconv_subm_neighbors", ops._p(cd), ops._p(rows), cap, ops._host_i32(shape), ops._host_i32(case.ksize),
                  ops._p(keys), ops._p(vals), cap, ops._p(nbr))
        got = nbr.cpu().numpy()
        assert np.array_equal(got[:n], subm_ref(live, shape, case.ksize)), f"{name}: SubM nbr differs"
        assert bool((got[n:] == SENT).all()), f"{name}: rows beyond the live count were written"
        print(f"rulebook {name}: {n} live of {cap}, K {K}, {int((got[:n] >= 0).sum())} hits: exact")
        return
    oc_ref, nbr_ref, okeys, _ = strided_ref(live, shape, case.ksize, case.stride, case.pad)
    n_out = len(okeys)
    ocap = _out_capacity(case, n_out)
    osh = _oshape(shape, case.ksize, case.stride, case.pad)
    lg = table_log2(ocap)
    okt, ovt = _i32((1 << lg,)), _i32((1 << lg,))
    ocoords, orows, nbr = _i32((ocap, 4)), _i32((1,)), _i32((ocap, K))
    wsb = lib.heal_spconv_strided_workspace(cap, ocap, K)
    ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    ops._call("heal_spconv_strided_rulebook", ops._p(cd), ops._p(rows), cap, ops._host_i32(osh), case.batch,
              ops._host_i32(case.ksize), ops._host_i32(case.stride), ops._host_i32(case.pad), ocap,
              ops._p(ocoords), ops._p(orows), ops._p(okt), ops._p(ovt), ops._p(nbr), ops._p(ws), wsb)
    m = min(n_out, ocap)
    assert int(orows.item()) == n_out, f"{name}: output count {int(orows.item())}, expected {n_out}"
    got_c, got_n = ocoords.cpu().numpy(), nbr.cpu().numpy()
    assert np.array_equal(got_c[:m], oc_ref[:m]), f"{name}: output sites or their order differ"
    assert bool((got_c[m:] == SENT).all()), f"{name}: output coords beyond the output count were written"
    assert np.array_equal(got_n[:m], nbr_ref[:m]), f"{name}: nbr differs"
    assert bool((got_n[m:] == -1).all()), f"{name}: nbr rows beyond the output count are not -1"
    row_of = np.where(np.arange(n_out) < ocap, np.arange(n_out), -1)
    _check_table(okt, ovt, okeys, row_of, lg, f"{name} output table")
    out = ops.SparseTensor(None, ocoords, orows, osh, case.batch, (okt, ovt), table_capacity=ocap)
    if n_out > ocap:
        with pytest.raises(RuntimeError, match="exceed the capacity"):
            ops.sp_check_overflow([out])
    else:
        ops.sp_check_overflow([out])
        sub = ops.sp_subm_neighbors(out, (3, 3, 3)).cpu().numpy()       # the new level's table serves SubM lookups
        assert np.array_equal(sub[:m], subm_ref(oc_ref, osh, (3, 3, 3))), f"{name}: SubM lookups in the output table differ"
        assert np.array_equal(sub[:m, 13], np.arange(m))
    print(f"rulebook {name}: {n} live of {cap} -> {n_out} sites (capacity {ocap}), {int((nbr_ref >= 0).sum())} pairs: exact")


# ================================================================================================ gather-GEMMs
SIMT_KERNELS = [(4, 16, 27), (16, 16, 27), (16, 32, 27), (32, 32, 27), (32, 64, 27), (64, 64, 27), (64, 128, 3)]


def _stages(cout):
    return 2 if cout >= 128 else (3 if cout >= 64 else 4)


@dataclass(frozen=True)
class TCase:
    name: str
    cin: int
    cout: int
    K: int
    live: int
    cap: int
    patterns: Tuple[str, ...]     # per-tile active K-block patterns, cycled over the tiles
    relu: bool = True
    bias: bool = True
    planar: bool = False          # split output into a planar view (pitch 80, channel offset 8), as the stem writes it
    situations: Tuple[str, ...] = ()

    @property
    def tpk(self):
        return 64 // self.cin

    @property
    def KB(self):
        return -(-self.K // self.tpk)


TC_SITUATIONS = ("empty_tile", "single_kblock_not_first", "kblock_gap", "all_kblocks", "padding_offsets", "partial_last_tile",
                 "dead_tail", "three_tiles_per_cta", "ring_offset", "late_first_kblock")
BIG = 3 * NUM_SMS * SPT_M + 300          # live rows: every CTA runs three or four tiles
MIX = ("dense", "empty", "last", "gap", "mid", "all", "first")
TCASES = [
    TCase("tc16x16_k27", 16, 16, 27, 2000, 2100, MIX, situations=("empty_tile", "single_kblock_not_first", "kblock_gap",
          "all_kblocks", "padding_offsets", "partial_last_tile", "dead_tail")),
    TCase("tc16x32_k27_big", 16, 32, 27, BIG, BIG + 200, MIX + ("odd",), relu=False, situations=("three_tiles_per_cta",
          "ring_offset", "late_first_kblock", "padding_offsets", "dead_tail", "partial_last_tile", "empty_tile")),
    TCase("tc32x32_k27", 32, 32, 27, 1536, 1536, MIX, bias=False, situations=("all_kblocks", "padding_offsets", "kblock_gap")),
    TCase("tc32x64_k27", 32, 64, 27, 1900, 2000, MIX, situations=("single_kblock_not_first", "dead_tail", "padding_offsets")),
    TCase("tc64x64_k27", 64, 64, 27, 1700, 1800, MIX, relu=False, situations=("kblock_gap", "all_kblocks", "empty_tile")),
    TCase("tc64x128_k27", 64, 128, 27, 1500, 1600, MIX, situations=("kblock_gap", "single_kblock_not_first", "dead_tail")),
    # conv_out of VoxelBackBone8x: (3,1,1), K = 3, on the 2-stage instantiation, fp32 output
    TCase("tc64x128_k3_big", 64, 128, 3, BIG, BIG + 100, ("dense", "first", "gap", "last", "empty", "all", "mid"),
          relu=False, situations=("three_tiles_per_cta", "ring_offset", "late_first_kblock", "kblock_gap", "dead_tail")),
    # the stem as gather-GEMMs: K = 9 (3x3) and K = 1 (downsample) into planar split views
    TCase("tc64x64_k9_planar", 64, 64, 9, 1800, 1800, MIX, planar=True, situations=("single_kblock_not_first", "kblock_gap",
          "empty_tile", "partial_last_tile")),
    TCase("tc64x64_k1_planar", 64, 64, 1, 1000, 1024, ("dense", "empty"), relu=False, planar=True,
          situations=("empty_tile", "all_kblocks", "dead_tail")),
    # padding offsets in the last K-block: Cin 16 with K = 5 (3 padding offsets), Cin 32 with K = 3 (1)
    TCase("tc16x32_k5", 16, 32, 5, 900, 1000, MIX, situations=("padding_offsets", "single_kblock_not_first", "dead_tail")),
    TCase("tc32x64_k3", 32, 64, 3, 700, 700, MIX, situations=("padding_offsets", "single_kblock_not_first", "empty_tile")),
]
TCASE = {c.name: c for c in TCASES}
MIN_ROWS = 3000                  # input rows the rulebooks point into


def _tile_blocks(pattern, KB, rng):
    return {"dense": list(range(KB)), "all": list(range(KB)), "empty": [], "last": [KB - 1], "mid": [KB // 2],
            "first": [0], "gap": sorted({0, KB - 1}) if KB > 2 else [KB - 1],
            "odd": list(range(1, KB, 2)) or [0]}[pattern]


def _tc_nbr(case, rng):
    """A synthetic rulebook (cap, K): tile t follows case.patterns[t % len]; the rows behind the live count hold valid rows."""
    K, tpk = case.K, case.tpk
    nbr = np.full((case.cap, K), -1, dtype=np.int32)
    for t in range(-(-case.live // SPT_M)):
        r0, r1 = t * SPT_M, min(case.live, t * SPT_M + SPT_M)
        pat = case.patterns[t % len(case.patterns)]
        for b in _tile_blocks(pat, case.KB, rng):
            ks = [k for k in range(b * tpk, b * tpk + tpk) if k < K]
            dens = 0.35 if pat == "dense" else 0.15
            hit = rng.random((r1 - r0, len(ks))) < dens
            hit[rng.integers(r1 - r0), rng.integers(len(ks))] = True
            vals = rng.integers(0, MIN_ROWS, (r1 - r0, len(ks)))
            nbr[r0:r1, ks] = np.where(hit, vals, -1)
    dead = nbr[case.live:]
    dead[:] = np.where(rng.random(dead.shape) < 0.5, rng.integers(0, MIN_ROWS, dead.shape), -1)
    return nbr


def _tc_inputs(case):
    rng = _rng(case.name, "tc")
    nbr = _tc_nbr(case, rng)
    x = torch.from_numpy(rng.standard_normal((MIN_ROWS, case.cin)).astype(np.float32))
    w = torch.from_numpy((rng.standard_normal((case.K, case.cin, case.cout)) / math.sqrt(case.K * case.cin)).astype(np.float32))
    b = torch.from_numpy(rng.standard_normal(case.cout).astype(np.float32)) if case.bias else None
    return nbr, x, w, b


def _masks(nbr, live, tpk):
    """Per tile of live rows: the active K-block mask of k_spconv_tc."""
    out = []
    for t in range(-(-live // SPT_M)):
        h = (nbr[t * SPT_M:min(live, t * SPT_M + SPT_M)] >= 0).any(0)
        m = 0
        for k in np.flatnonzero(h):
            m |= 1 << (int(k) // tpk)
        out.append(m)
    return out


def _tc_census(case, nbr=None):
    if nbr is None:
        nbr = _tc_inputs(case)[0]
    masks = _masks(nbr, case.live, case.tpk)
    grid = min(-(-case.cap // SPT_M), NUM_SMS)
    full, found = (1 << case.KB) - 1, set()
    S = _stages(case.cout)
    for t, m in enumerate(masks):
        bits = [b for b in range(case.KB) if (m >> b) & 1]
        if m == 0:
            found.add("empty_tile")
        elif len(bits) == 1 and bits[0] != 0:
            found.add("single_kblock_not_first")
        if bits and bits[-1] - bits[0] + 1 != len(bits):
            found.add("kblock_gap")
        if m == full:
            found.add("all_kblocks")
        if case.K % case.tpk and (m >> (case.KB - 1)) & 1:
            found.add("padding_offsets")
        if t + grid < len(masks) and max(len(bits), 1) % S:
            found.add("ring_offset")
        if t >= grid and bits and bits[0] != 0:
            found.add("late_first_kblock")
    if case.live % SPT_M:
        found.add("partial_last_tile")
    if case.live < case.cap:
        found.add("dead_tail")
    if case.live > 3 * NUM_SMS * SPT_M:
        found.add("three_tiles_per_cta")
    return found, dict(tiles=len(masks), grid=grid, stages=S)


@pytest.mark.parametrize("name", list(TCASE))
def test_tc_case_produces_its_situations(name):
    case = TCASE[name]
    found, stats = _tc_census(case)
    assert set(case.situations) <= set(TC_SITUATIONS)
    assert set(case.situations) <= found, f"{name}: {sorted(set(case.situations) - found)} do not occur ({stats})"


def test_tc_cases_cover_every_situation():
    found = set()
    for c in TCASES:
        found |= _tc_census(c)[0]
    assert found == set(TC_SITUATIONS), sorted(set(TC_SITUATIONS) - found)
    three = {_stages(c.cout) for c in TCASES if "three_tiles_per_cta" in _tc_census(c)[0]}
    assert three >= {2, 4}, "three tiles per CTA must run on a 2-stage and on a 4-stage instantiation"


def _split_np(x):
    """hi, lo of a float32 tensor as the kernels split it (round to nearest even)."""
    hi = x.to(torch.bfloat16)
    return hi, (x - hi.float()).to(torch.bfloat16)


def _gemm_ref(a, nbr, w, b, relu, rows, fault=None, tiles=None):
    """float64 (y after the activation, y before it, sum |a| |w|, hits per row) over rows [0, rows).  a (Min, Cin) and w
    (K, Cin, Cout) float64, b (Cout) float64 or None.  `fault` restates a plausible kernel bug (tiles = (tpk, grid) of the
    tensor-core tiling for the faults that depend on it)."""
    nbr = nbr[:rows].copy()
    K, cout = w.shape[0], w.shape[2]
    if fault == "flip":                                  # convolution instead of cross-correlation
        w = w[::-1]
    if fault == "tap_neighbour":                         # a tap read from the neighbouring offset (pairs k, k ^ 1)
        sw = [k ^ 1 if (k ^ 1) < K else k for k in range(K)]
        nbr = nbr[:, sw]
    if fault == "skip_last_kblock":
        tpk = tiles[0]
        for t in range(-(-rows // SPT_M)):
            blk = nbr[t * SPT_M:t * SPT_M + SPT_M]
            act = [k // tpk for k in np.flatnonzero((blk >= 0).any(0))]
            if act:
                last = max(act)
                blk[:, last * tpk:(last + 1) * tpk] = -1
    y = np.zeros((rows, cout))
    s = np.zeros((rows, cout))
    for k in range(K):
        idx = nbr[:, k]
        h = idx >= 0
        if h.any():
            y[h] += a[idx[h]] @ w[k]
            s[h] += np.abs(a[idx[h]]) @ np.abs(w[k])
    if fault == "stale_acc":                             # accumulators kept from the CTA's previous tile when the first active
        tpk, grid = tiles[:2]                            # K-block is not block 0
        acc = y.copy()
        for t in range(grid, -(-rows // SPT_M)):
            m = (nbr[t * SPT_M:t * SPT_M + SPT_M] >= 0).any(0)
            ks = np.flatnonzero(m)
            if ks.size and ks[0] // tpk != 0:
                r0, n = t * SPT_M, min(SPT_M, rows - t * SPT_M)
                p0 = (t - grid) * SPT_M
                y[r0:r0 + n] += acc[p0:p0 + n]
    if b is not None and fault != "no_bias":
        y = y + b * (2 if fault == "bias_twice" else 1)
    pre = y
    if fault == "row_shift":                             # row r written to r + 1 at a block / tile edge
        e = tiles[2] if tiles else SP_BLOCK
        pre = y.copy()
        for r in range(e - 1, rows - 1, e):
            pre[r + 1] = y[r]
    out = np.maximum(pre, 0) if relu and fault != "no_relu" else pre
    return out, y, s, (nbr >= 0).sum(1)


def _simt_bound(y_pre, s, hits, cin, b):
    babs = np.abs(b) if b is not None else 0.0
    return U * (hits[:, None] * cin + 1) * (s + babs)


def _tc_bound(y_pre, s):
    return ALPHA * s + REL * np.abs(y_pre)


def _report(what, got, y, bound):
    err = np.abs(got.astype(np.float64) - y)
    bad = ~(err <= bound)
    ratio = _ratio(err, bound)
    print(f"{what}: max err / bound {ratio:.4f} (max err {err.max(initial=0):.3e}, max |y| {np.abs(y).max(initial=0):.3f})")
    if bad.any():
        r, c = np.unravel_index(int(np.argmax(np.where(bad, err / np.maximum(bound, 1e-300), -1))), err.shape)
        pytest.fail(f"{what}: {int(bad.sum())} elements outside the bound, worst row {r} channel {c}: got {got[r, c]!r}, "
                    f"expected {y[r, c]!r}, bound {bound[r, c]:.3e}")



def _simt_case(cin, cout, K, rng):
    cap, live = 700, 650
    nbr = np.full((cap, K), -1, dtype=np.int32)
    for b0 in range(0, live, SP_BLOCK):              # per 32-row block a random subset of the offsets is active
        r1 = min(live, b0 + SP_BLOCK)
        if (b0 // SP_BLOCK) % 7 == 3:
            continue                                 # a block with no hit at all
        ks = np.flatnonzero(rng.random(K) < 0.6)
        hit = rng.random((r1 - b0, ks.size)) < 0.4
        nbr[b0:r1, ks] = np.where(hit, rng.integers(0, MIN_ROWS, (r1 - b0, ks.size)), -1)
    nbr[live:] = rng.integers(0, MIN_ROWS, (cap - live, K))
    x = rng.standard_normal((MIN_ROWS, cin)).astype(np.float32)
    w = (rng.standard_normal((K, cin, cout)) / math.sqrt(K * cin)).astype(np.float32)
    b = rng.standard_normal(cout).astype(np.float32)
    return nbr, x, w, b, live


@pytest.mark.gpu
@pytest.mark.parametrize("bias, relu", [(True, True), (True, False), (False, True), (False, False)])
@pytest.mark.parametrize("cin, cout, K", SIMT_KERNELS)
def test_gather_gemm_simt(cin, cout, K, bias, relu):
    from heal_b200 import ops
    rng = _rng(f"{cin}x{cout}", "simt")
    nbr, x, w, b, live = _simt_case(cin, cout, K, rng)
    cap = nbr.shape[0]
    out = _i32((cap, cout)).view(torch.float32)
    rows = torch.tensor([live], dtype=torch.int32, device="cuda")
    bt = torch.from_numpy(b).cuda() if bias else None
    xd, nd, wd = (torch.from_numpy(a).cuda() for a in (x, nbr, w))          # held: the call takes raw pointers
    ops._call("heal_spconv_gather_gemm", ops._p(xd), ops._p(nd), ops._p(rows), cap, K, ops._p(wd), ops._p(bt), cin, cout,
              1 if relu else 0, ops._p(out))
    got = out.cpu()
    y, pre, s, hits = _gemm_ref(x.astype(np.float64), nbr, w.astype(np.float64), b.astype(np.float64) if bias else None, relu, live)
    _report(f"heal_spconv_gather_gemm ({cin},{cout}) K {K} bias {int(bias)} relu {int(relu)}", got[:live].numpy(), y,
            _simt_bound(pre, s, hits, cin, b if bias else None))
    assert bool((got[live:].view(torch.int32) == SENT).all()), "rows beyond the live count were written"
    empty = hits == 0
    assert empty.any() and np.array_equal(got[:live].numpy()[empty], y[empty].astype(np.float32)), "an empty row is not act(bias)"


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(TCASE))
def test_gather_gemm_tc(name):
    from heal_b200 import ops
    case = TCASE[name]
    nbr, x, w, b = _tc_inputs(case)
    found, stats = _tc_census(case, nbr)
    cin, cout, cap, K = case.cin, case.cout, case.cap, case.K
    hi, lo = _split_np(x)
    fs = torch.cat([hi, lo], 1).contiguous().cuda()
    pk = ops.pack_spconv_tc(w.cuda())
    nb = torch.from_numpy(nbr).cuda()
    rows = torch.tensor([case.live], dtype=torch.int32, device="cuda")
    bt = b.cuda() if b is not None else None
    P = 80 if case.planar else 2 * cout
    c0 = 8 if case.planar else 0
    lo_off = cap * P if case.planar else cout

    def run(want_f32, want_split):
        f32 = _i32((cap, cout)).view(torch.float32) if want_f32 else None
        sp = torch.full((2, cap, P) if case.planar else (cap, P), SENT16, dtype=torch.int16, device="cuda").view(torch.bfloat16) \
            if want_split else None
        ptr = ops._vp(sp.data_ptr() + 2 * c0) if want_split else ops._vp(0)
        ops._call("heal_spconv_gather_gemm_tc", ops._p(fs), ops._p(nb), ops._p(rows), cap, K, ops._p(pk), ops._p(bt), cin, cout,
                  1 if case.relu else 0, ptr, ops._p(f32), 0, 0, P if case.planar else 0, lo_off if case.planar else 0)
        return f32, sp

    f32, sp = run(True, True)
    a64 = (hi.double() + lo.double()).numpy()
    y, pre, s, hits = _gemm_ref(a64, nbr, w.double().numpy(), b.double().numpy() if b is not None else None, case.relu, case.live)
    got = f32.cpu()
    _report(f"heal_spconv_gather_gemm_tc {name} ({stats['tiles']} tiles on {stats['grid']} CTAs, "
                    f"{stats['stages']} stages)", got[:case.live].numpy(), y, _tc_bound(pre, s))
    assert bool((got[case.live:].view(torch.int32) == SENT).all()), f"{name}: fp32 rows beyond the live count were written"
    empty = hits == 0
    if "empty_tile" in found:
        assert empty.any() and np.array_equal(got[:case.live].numpy()[empty], y[empty].astype(np.float32)), \
            f"{name}: an empty row is not act(bias)"
    # the split output of the same run: hi = bf16(v), lo = bf16(v - hi), in the view; everything else keeps its sentinel
    bits = sp.cpu().view(torch.int16)
    hp, lp = (bits[0], bits[1]) if case.planar else (bits[:, :cout], bits[:, cout:])
    want_hi, want_lo = (t.view(torch.int16) for t in _split_np(got[:case.live]))
    assert torch.equal(hp[:case.live, c0:c0 + cout], want_hi), f"{name}: split hi != bf16(fp32 output)"
    assert torch.equal(lp[:case.live, c0:c0 + cout], want_lo), f"{name}: split lo != bf16(fp32 output - hi)"
    untouched = torch.ones_like(bits, dtype=torch.bool)
    if case.planar:
        untouched[:, :case.live, c0:c0 + cout] = False
    else:
        untouched[:case.live] = False
    assert bool((bits[untouched] == SENT16).all()), f"{name}: split elements outside the written view changed"
    # the product asks for one output per call: the same bits as the run that wrote both
    assert torch.equal(run(True, False)[0].cpu().view(torch.int32), got.view(torch.int32)), f"{name}: an fp32-only run differs"
    assert torch.equal(run(False, True)[1].cpu().view(torch.int16), bits), f"{name}: a split-only run differs"

def test_pack_spconv_tc_layout():
    """pack_spconv_tc: [2 planes][KB Cout rows][64]; K-block kb holds offsets kb TPK .. kb TPK + TPK - 1 side by side, zero
    columns for padding offsets; hi + lo is the weight to 2^-16."""
    from heal_b200 import ops
    rng = np.random.default_rng(5)
    for cin, cout, K in [(16, 32, 27), (16, 16, 5), (32, 64, 3), (32, 32, 27), (64, 128, 3), (64, 64, 1)]:
        w = torch.from_numpy(rng.standard_normal((K, cin, cout)).astype(np.float32))
        pk = ops.pack_spconv_tc(w)
        tpk = 64 // cin
        KB = -(-K // tpk)
        assert pk.shape == (2, KB * cout, 64) and pk.dtype == torch.bfloat16
        full = pk.float().sum(0).reshape(KB, cout, 64)
        want = torch.zeros(KB, cout, 64)
        for k in range(K):
            want[k // tpk, :, (k % tpk) * cin:(k % tpk + 1) * cin] = w[k].t()
        assert bool(((full - want).abs() <= 2.0 ** -16 * want.abs()).all()), (cin, cout, K)
        assert bool((pk[1].float().reshape(KB, cout, 64)[want == 0] == 0).all())      # zero padding columns in both planes
        assert K % tpk == 0 or bool((want[-1, :, (K % tpk) * cin:] == 0).all())
        assert torch.equal(pk[0], want.reshape(KB * cout, 64).to(torch.bfloat16))


# ================================================================================================ helpers
def _bf16_bits(x32):
    """Round-to-nearest-even of float32 values to bf16 bit patterns (finite inputs)."""
    b = np.asarray(x32, dtype=np.float32).view(np.uint32).astype(np.uint64)
    return (((b + 0x7FFF + ((b >> 16) & 1)) >> 16) & 0xFFFF).astype(np.uint16)


def _bf16_value(bits):
    return (bits.astype(np.uint32) << 16).view(np.float32)


def _tricky_f32(rng, n):
    """Random values plus ties (lower 16 bits 0x8000 with even and odd kept parts), one ulp either side of a tie, +-0,
    subnormals and values near the largest finite bf16."""
    base = rng.integers(0x00800000, 0x7F000000, n, dtype=np.uint64).astype(np.uint32)
    kind = np.arange(n) % 6
    tie = (base & np.uint32(0xFFFF0000)) | np.uint32(0x8000)
    bits = np.select([kind == 1, kind == 2, kind == 3, kind == 4], [tie, tie + np.uint32(1), tie - np.uint32(1),
                     base & np.uint32(0x000FFFFF)], base).astype(np.uint32)
    bits[::7] |= np.uint32(0x80000000)
    bits[:4] = [0, 0x80000000, 0x7F7F0000, 0x00000001]
    return bits.view(np.float32)


@pytest.mark.gpu
def test_rows_to_split():
    from heal_b200 import ops
    rng = np.random.default_rng(3)
    cap, C, live = 999, 48, 917
    x = _tricky_f32(rng, cap * C).reshape(cap, C)
    out = _i32((cap, C)).view(torch.bfloat16)                                       # (cap, 2C) bf16
    rows = torch.tensor([live], dtype=torch.int32, device="cuda")
    xd = torch.from_numpy(x).cuda()
    ops._call("heal_rows_to_split", ops._p(xd), ops._p(rows), cap, C, ops._p(out))
    got = out.cpu().view(torch.int16).numpy().view(np.uint16)
    hi = _bf16_bits(x[:live])
    lo = _bf16_bits(x[:live] - _bf16_value(hi))
    assert np.array_equal(got[:live, :C], hi), "hi != bf16(x)"
    assert np.array_equal(got[:live, C:], lo), "lo != bf16(x - hi)"
    assert bool((got[live:] == SENT16).all()), "rows beyond the live count were written"
    assert np.array_equal(ops.rows_to_split(xd, None).cpu().view(torch.int16).numpy().view(np.uint16)[:live],
                          got[:live])


@pytest.mark.gpu
def test_sparse_to_bev():
    from heal_b200 import ops
    rng = np.random.default_rng(4)
    B, D, H, W, C = 2, 5, 12, 20, 16
    cells = B * D * H * W
    k = rng.choice(cells, 400, replace=False)
    live, n = _decode(k[:300], (D, H, W)), 300
    tail = np.r_[_decode(k[300:], (D, H, W)), live[:20]]                            # other sites, duplicates of live ones
    coords = np.ascontiguousarray(np.r_[live, tail].astype(np.int32))
    feats = rng.standard_normal((coords.shape[0], C)).astype(np.float32)
    st = ops.SparseTensor(torch.from_numpy(feats).cuda(), torch.from_numpy(coords).cuda(),
                          torch.tensor([n], dtype=torch.int32, device="cuda"), [D, H, W], B)
    got = ops.sparse_to_bev(st).t.cpu().numpy()
    want = np.zeros((B, H, W, C * D), dtype=np.float32)
    for i in range(n):
        b, z, y, x = live[i]
        want[b, y, x, np.arange(C) * D + z] = feats[i]
    assert got.shape == want.shape and np.array_equal(got.view(np.int32), want.view(np.int32))


@pytest.mark.gpu
@pytest.mark.parametrize("with_count", [True, False])
def test_pillar_idmap(with_count):
    from heal_b200 import ops
    rng = np.random.default_rng(6)
    B, ny, nx = 3, 10, 14
    k = rng.choice(B * ny * nx, 150, replace=False)
    n = 120 if with_count else 150
    c = _decode(k, (1, ny, nx))
    coords = np.ascontiguousarray(np.r_[c, c[:10]].astype(np.int32)) if with_count else np.ascontiguousarray(c)
    idmap = _i32((B, ny, nx))
    cnt = torch.tensor([n], dtype=torch.int32, device="cuda") if with_count else None
    cd = torch.from_numpy(coords).cuda()
    ops._call("heal_pillar_idmap", ops._p(cd), ops._p(cnt), coords.shape[0], B, ny, nx, ops._p(idmap))
    want = np.full((B, ny, nx), -1, dtype=np.int32)
    want[c[:n, 0], c[:n, 2], c[:n, 3]] = np.arange(n)
    assert np.array_equal(idmap.cpu().numpy(), want)


def stem_rulebook_ref(idmap, k, pad):
    B, ny, nx = idmap.shape
    Ho, Wo = ny // 2, nx // 2
    P = np.full((B, ny + 2 * pad + 2, nx + 2 * pad + 2), -1, dtype=np.int32)
    P[:, pad:pad + ny, pad:pad + nx] = idmap
    taps = [P[:, r:r + 2 * Ho:2, s:s + 2 * Wo:2] for r in range(k) for s in range(k)]
    return np.stack(taps, -1).reshape(B * Ho * Wo, k * k)


@pytest.mark.gpu
@pytest.mark.parametrize("k, pad", [(3, 1), (1, 0)])
def test_stem_rulebook(k, pad):
    from heal_b200 import ops
    rng = np.random.default_rng(7 + k)
    B, ny, nx = 3, 12, 18
    idmap = np.where(rng.random((B, ny, nx)) < 0.4, rng.integers(0, 5000, (B, ny, nx)), -1).astype(np.int32)
    idmap[:, [0, -1], :] = rng.integers(0, 5000, (B, 2, nx))                        # hits on every border row and column
    idmap[:, :, [0, -1]] = rng.integers(0, 5000, (B, ny, 2))
    nbr = _i32((B * (ny // 2) * (nx // 2), k * k))
    idd = torch.from_numpy(idmap).cuda()
    ops._call("heal_stem_rulebook", ops._p(idd), B, ny, nx, k, pad, ops._p(nbr))
    assert np.array_equal(nbr.cpu().numpy(), stem_rulebook_ref(idmap, k, pad))


# ================================================================================================ sparse stem
STEM_SITUATIONS = tuple(f"tap{t}_alone" for t in range(9)) + (
    "border_top", "border_left", "last_row", "last_col",   # hits on input row 0 / column 0 / the last row / the last column
    "centre_absent", "centre_present",                     # pixels with hits without and with the centre (downsample) tap
    "group_hi_only",                                       # a 16-pixel group of the mma.sync kernel whose hits are in pixels 8-15
    "all_empty",                                           # no pixel has a hit
    "batch3",                                              # three or more images
    "nx_not_32")                                           # nx even but not a multiple of 32 (the SIMT kernel only)


@dataclass(frozen=True)
class SCase:
    name: str
    B: int
    ny: int
    nx: int
    map: str
    situations: Tuple[str, ...]


SCASES = [
    SCase("taps", 1, 24, 32, "taps", tuple(f"tap{t}_alone" for t in range(9)) + ("centre_absent", "centre_present")),
    SCase("border_b3", 3, 14, 64, "border", ("border_top", "border_left", "last_row", "last_col", "batch3", "centre_absent")),
    SCase("hi_only", 2, 8, 64, "hi_only", ("group_hi_only", "centre_absent")),
    SCase("empty", 2, 6, 32, "empty", ("all_empty",)),
    SCase("random_nx44", 3, 10, 44, "random", ("nx_not_32", "batch3", "border_top", "last_col", "centre_present")),
]
SCASE = {c.name: c for c in SCASES}


def _stem_map(case):
    rng = _rng(case.name, "stem")
    B, ny, nx = case.B, case.ny, case.nx
    occ = np.zeros((B, ny, nx), dtype=bool)
    if case.map == "taps":                # isolated cells 6 apart, at every parity of row and column
        for a, iy in enumerate(range(2, ny - 2, 6)):
            for c, ix in enumerate(range(2, nx - 2, 6)):
                occ[0, iy + (a % 2), ix + (c % 2)] = True
    elif case.map == "border":
        occ = rng.random((B, ny, nx)) < 0.1
        occ[:, 0, ::3] = occ[:, ::4, 0] = occ[:, -1, 1::3] = occ[:, 2::3, -1] = True
    elif case.map == "hi_only":           # group 1 of row 2: cells in columns 48..62 only (pixels 24..31 = 8..15 of the group)
        occ[:, 4:7, 48:63] = rng.random((B, 3, 15)) < 0.5
        occ[:, 4, 50] = True
    elif case.map == "random":
        occ = rng.random((B, ny, nx)) < 0.35
        occ[:, 0, 3] = occ[:, 5, -1] = True
    idmap = np.full((B, ny, nx), -1, dtype=np.int32)
    n = int(occ.sum())
    idmap[occ] = rng.permutation(n) + 7                   # pillar rows in scrambled order, row 0..6 unused
    return idmap, n + 7


def _stem_taps(idmap):
    """(B, Ho, Wo, 9) pillar row of each tap of each output pixel, -1 for none."""
    B, ny, nx = idmap.shape
    return stem_rulebook_ref(idmap, 3, 1).reshape(B, ny // 2, nx // 2, 9)


def _stem_census(case):
    idmap, _ = _stem_map(case)
    taps = _stem_taps(idmap) >= 0
    found = set()
    cnt = taps.sum(-1)
    for t in range(9):
        if (taps[..., t] & (cnt == 1)).any():
            found.add(f"tap{t}_alone")
    occ = idmap >= 0
    for name, on in (("border_top", occ[:, 0].any()), ("border_left", occ[:, :, 0].any()), ("last_row", occ[:, -1].any()),
                     ("last_col", occ[:, :, -1].any()), ("centre_absent", ((cnt > 0) & ~taps[..., 4]).any()),
                     ("centre_present", taps[..., 4].any()), ("all_empty", not occ.any()), ("batch3", case.B >= 3),
                     ("nx_not_32", case.nx % 32 != 0)):
        if on:
            found.add(name)
    if case.nx % 32 == 0:
        g = (cnt > 0).reshape(case.B, case.ny // 2, case.nx // 32, 16)
        if (g[..., 8:].any(-1) & ~g[..., :8].any(-1)).any():
            found.add("group_hi_only")
    return found


@pytest.mark.parametrize("name", list(SCASE))
def test_stem_case_produces_its_situations(name):
    case = SCASE[name]
    found = _stem_census(case)
    assert set(case.situations) <= set(STEM_SITUATIONS)
    assert set(case.situations) <= found, f"{name}: {sorted(set(case.situations) - found)} do not occur"


def test_stem_cases_cover_every_situation():
    found = set()
    for c in SCASES:
        found |= _stem_census(c)
    assert found == set(STEM_SITUATIONS), sorted(set(STEM_SITUATIONS) - found)


def _stem_inputs(case):
    idmap, M = _stem_map(case)
    rng = _rng(case.name, "stem-weights")
    f = rng.standard_normal((M, 64)).astype(np.float32)
    w1 = (rng.standard_normal((9, 64, 64)) / 24).astype(np.float32)
    b1 = rng.standard_normal(64).astype(np.float32)
    w2 = (rng.standard_normal((64, 64)) / 8).astype(np.float32)
    b2 = rng.standard_normal(64).astype(np.float32)
    return idmap, f, w1, b1, w2, b2


def stem_ref(idmap, f, w1, b1, w2, b2, fault=None):
    """float64 (conv after ReLU, conv before it, sum |a w| of the conv, hits; downsample, its sum |a w|, centre hit)."""
    taps = _stem_taps(idmap)
    f, w1, w2 = f.astype(np.float64), w1.astype(np.float64), w2.astype(np.float64)
    shp = taps.shape[:3] + (64,)
    y1, s1 = np.zeros(shp), np.zeros(shp)
    for t in range(9):
        ids = taps[..., t]
        h = ids >= 0
        wt = w1[8 - t] if fault == "flip" else w1[t]
        y1[h] += f[ids[h]] @ wt
        s1[h] += np.abs(f[ids[h]]) @ np.abs(wt)
    c = taps[..., 0 if fault == "down_tap0" else 4]
    y2, s2 = np.zeros(shp), np.zeros(shp)
    y2[c >= 0] = f[c[c >= 0]] @ w2
    s2[c >= 0] = np.abs(f[c[c >= 0]]) @ np.abs(w2)
    if fault != "no_bias":
        y1, y2 = y1 + b1, y2 + b2
    conv = y1 if fault == "no_relu" else np.maximum(y1, 0)
    return conv, y1, s1, (taps >= 0).sum(-1), y2, s2, c >= 0


def _stem_bounds(kind, y1, s1, hits, y2, s2, cntr, b1, b2):
    if kind == "heal_sparse_stem":
        return (U * (hits[..., None] * 64 + 1) * (s1 + np.abs(b1)), U * (cntr[..., None] * 64 + 1) * (s2 + np.abs(b2)))
    return _tc_bound(y1, s1), _tc_bound(y2, s2)


STEM_CS, STEM_CO = 80, 8          # channel stride and (even) channel offset of the output views


def _stem_out(case, fmt):
    Ho, Wo = case.ny // 2, case.nx // 2
    planes = {"f32": 0, "bf16": 1, "split": 2}[fmt]
    if fmt == "f32":
        t = _i32((case.B, Ho, Wo, STEM_CS)).view(torch.float32)
    else:
        t = torch.full((planes, case.B, Ho, Wo, STEM_CS), SENT16, dtype=torch.int16, device="cuda").view(torch.bfloat16)
    return t


def _run_stem(kind, case, fmt, tensors):
    from heal_b200 import ops
    from heal_b200._lib import HealAct
    idmap, f, w1, b1, w2, b2 = tensors
    o1, o2 = _stem_out(case, fmt), _stem_out(case, fmt)
    plane = case.B * (case.ny // 2) * (case.nx // 2) * STEM_CS
    acts = [HealAct(o.data_ptr(), ops.FMT[fmt], STEM_CS, STEM_CO, plane if fmt != "f32" else 0) for o in (o1, o2)]
    ops._call(kind, ops._p(f), ops._p(idmap), case.B, case.ny, case.nx, ops._p(w1), ops._p(b1), ops._p(w2), ops._p(b2), 64,
              acts[0], acts[1])
    return o1.cpu(), o2.cpu()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["heal_sparse_stem", "heal_sparse_stem_tc"])
@pytest.mark.parametrize("name", list(SCASE))
def test_sparse_stem(kind, name):
    case = SCASE[name]
    if kind == "heal_sparse_stem_tc" and case.nx % 32:
        pytest.skip("heal_sparse_stem_tc takes nx in multiples of 32 (its refusal is test_refusals)")
    idmap, f, w1, b1, w2, b2 = _stem_inputs(case)
    dev = [torch.from_numpy(a).cuda() for a in (idmap, f, w1, b1, w2, b2)]
    conv, y1, s1, hits, y2, s2, cntr = stem_ref(idmap, f, w1, b1, w2, b2)
    bd1, bd2 = _stem_bounds(kind, y1, s1, hits, y2, s2, cntr, b1, b2)
    a1, a2 = _run_stem(kind, case, "f32", dev)
    sl = slice(STEM_CO, STEM_CO + 64)
    _report(f"{kind} {name} conv", a1[..., sl].reshape(-1, 64).numpy(), conv.reshape(-1, 64), bd1.reshape(-1, 64))
    _report(f"{kind} {name} down", a2[..., sl].reshape(-1, 64).numpy(), y2.reshape(-1, 64), bd2.reshape(-1, 64))
    g1, g2 = a1[..., sl].numpy(), a2[..., sl].numpy()
    assert np.array_equal(g2[~cntr], np.broadcast_to(b2, g2[~cntr].shape)), "downsample without a centre hit != its bias"
    assert np.array_equal(g1[hits == 0], np.broadcast_to(np.maximum(b1, 0), g1[hits == 0].shape)), "no hit != ReLU(bias)"
    outside = torch.ones(STEM_CS, dtype=torch.bool)
    outside[sl] = False
    for a in (a1, a2):
        assert bool((a.view(torch.int32)[..., outside] == SENT).all()), "channels outside the view changed"
    for fmt in ("bf16", "split"):
        for got, ref in zip(_run_stem(kind, case, fmt, dev), (a1, a2)):
            v = ref[..., sl]
            hi = v.to(torch.bfloat16)
            assert torch.equal(got[0][..., sl].view(torch.int16), hi.view(torch.int16)), f"{fmt}: hi != bf16(f32 output)"
            if fmt == "split":
                lo = (v - hi.float()).to(torch.bfloat16)
                assert torch.equal(got[1][..., sl].view(torch.int16), lo.view(torch.int16)), "split: lo != bf16(f32 - hi)"
            assert bool((got.view(torch.int16)[..., outside] == SENT16).all()), f"{fmt}: channels outside the view changed"



# ================================================================================================ refusals
REFUSALS = [
    ("gemm_16x64", "heal_spconv_gather_gemm", "HEAL_ERR_UNSUPPORTED"),
    ("gemm_4x32", "heal_spconv_gather_gemm", "HEAL_ERR_UNSUPPORTED"),
    ("tc_cin8", "heal_spconv_gather_gemm_tc", "HEAL_ERR_UNSUPPORTED"),
    ("tc_kvol0", "heal_spconv_gather_gemm_tc", "HEAL_ERR_UNSUPPORTED"),
    ("tc_kvol28", "heal_spconv_gather_gemm_tc", "HEAL_ERR_UNSUPPORTED"),
    ("tc_pitch12", "heal_spconv_gather_gemm_tc", "HEAL_ERR_UNSUPPORTED"),
    ("tc_no_output", "heal_spconv_gather_gemm_tc", "HEAL_ERR_ARG"),
    ("strided_in_capacity", "heal_spconv_strided_rulebook", "HEAL_ERR_ARG"),
    ("strided_workspace", "heal_spconv_strided_rulebook", "HEAL_ERR_WORKSPACE"),
    ("strided_cells", "heal_spconv_strided_rulebook", "HEAL_ERR_UNSUPPORTED"),
    ("table_cells", "heal_spconv_build_table", "HEAL_ERR_UNSUPPORTED"),
    ("stem_c32", "heal_sparse_stem", "HEAL_ERR_UNSUPPORTED"),
    ("stem_odd_ny", "heal_sparse_stem", "HEAL_ERR_UNSUPPORTED"),
    ("stem_odd_coffset", "heal_sparse_stem", "HEAL_ERR_UNSUPPORTED"),
    ("stem_tc_c32", "heal_sparse_stem_tc", "HEAL_ERR_UNSUPPORTED"),
    ("stem_tc_odd_ny", "heal_sparse_stem_tc", "HEAL_ERR_UNSUPPORTED"),
    ("stem_tc_nx48", "heal_sparse_stem_tc", "HEAL_ERR_UNSUPPORTED"),
    ("stem_tc_odd_coffset", "heal_sparse_stem_tc", "HEAL_ERR_UNSUPPORTED"),
    ("stem_rulebook_odd_nx", "heal_stem_rulebook", "HEAL_ERR_ARG"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("what, symbol, error", REFUSALS)
def test_refusals(what, symbol, error):
    """Each unsupported call is refused by name, and nothing is launched."""
    from heal_b200 import ops
    from heal_b200._lib import lib, HealAct
    buf = torch.zeros(1 << 16, dtype=torch.float32, device="cuda")
    p, n = ops._p(buf), ops._vp(0)
    h3 = ops._host_i32

    def call():
        if symbol == "heal_spconv_gather_gemm":
            ci, co = (16, 64) if what == "gemm_16x64" else (4, 32)
            ops._call(symbol, p, p, n, 64, 1, p, n, ci, co, 0, p)
        elif symbol == "heal_spconv_gather_gemm_tc":
            cin, K, pitch, out = 16, 27, 0, p
            cin = 8 if what == "tc_cin8" else cin
            K = {"tc_kvol0": 0, "tc_kvol28": 28}.get(what, K)
            pitch = 12 if what == "tc_pitch12" else 0
            out = n if what == "tc_no_output" else out
            ops._call(symbol, p, p, n, 64, K, p, n, cin, 16, 0, out, n, 0, 0, pitch, 0)
        elif symbol == "heal_spconv_strided_rulebook":
            cap = (1 << 20) + 1 if what == "strided_in_capacity" else 64
            osh = [2048, 2048, 1024] if what == "strided_cells" else [8, 8, 8]
            wsb = lib.heal_spconv_strided_workspace(64, 64, 27)
            ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
            ops._call(symbol, p, n, cap, h3(osh), 1, h3([3, 3, 3]), h3([2, 2, 2]), h3([1, 1, 1]), 64, p, p, p, p, p, ops._p(ws),
                      wsb - 1 if what == "strided_workspace" else wsb)
        elif symbol == "heal_spconv_build_table":
            ops._call(symbol, p, n, 64, h3([1024, 2048, 1024]), 2, p, p)
        elif symbol in ("heal_sparse_stem", "heal_sparse_stem_tc"):
            C = 32 if what.endswith("c32") else 64
            ny = 7 if what.endswith("odd_ny") else 8
            nx = 48 if what.endswith("nx48") else 32
            co = 1 if what.endswith("odd_coffset") else 0
            a = HealAct(buf.data_ptr(), 0, 64, co, 0)
            ops._call(symbol, p, p, 1, ny, nx, p, p, p, p, C, a, HealAct(buf.data_ptr(), 0, 64, 0, 0))
        else:
            ops._call(symbol, p, 1, 8, 9, 3, 1, p)

    torch.cuda.synchronize()
    before = lib.heal_launch_count()
    with pytest.raises(RuntimeError, match=f"{symbol} failed: {error}"):
        call()
    torch.cuda.synchronize()
    assert lib.heal_launch_count() == before


# ================================================================================================ coverage and sharpness (CPU)
def _instantiations(path, macro):
    return {tuple(int(v) for v in m) for m in re.findall(macro + r"\((\d+), (\d+)\);", (CSRC / path).read_text())}


def _exports(*paths):
    return {m for p in paths for m in re.findall(r'extern "C" \w+ (heal_\w+)\(', (CSRC / p).read_text())}


REACHED = {   # every C-ABI entry point of the three files -> the test that calls it
    "heal_spconv_table_size": "test_rulebook", "heal_spconv_build_table": "test_rulebook",
    "heal_spconv_subm_neighbors": "test_rulebook", "heal_spconv_strided_workspace": "test_rulebook",
    "heal_spconv_strided_rulebook": "test_rulebook", "heal_spconv_gather_gemm": "test_gather_gemm_simt",
    "heal_sparse_to_bev": "test_sparse_to_bev", "heal_stem_rulebook": "test_stem_rulebook",
    "heal_spconv_gather_gemm_tc": "test_gather_gemm_tc", "heal_rows_to_split": "test_rows_to_split",
    "heal_pillar_idmap": "test_pillar_idmap", "heal_sparse_stem": "test_sparse_stem", "heal_sparse_stem_tc": "test_sparse_stem",
}


def test_every_kernel_and_instantiation_is_reached():
    """7 SIMT and 6 tensor-core gather-GEMM instantiations (read from the sources), both stems on at least one case, and
    every entry point of the three files has its test."""
    simt = _instantiations("spconv.cu", "GG")
    tc = _instantiations("spconv_tc.cu", "SPT")
    assert len(simt) == 7 and len(tc) == 6
    assert {(ci, co) for ci, co, _ in SIMT_KERNELS} == simt
    assert {(c.cin, c.cout) for c in TCASES if c.K == 27} == tc
    assert {(c.cin, c.cout, c.K) for c in TCASES} >= {(64, 128, 3), (64, 64, 9), (64, 64, 1)}
    assert {c.K % c.tpk != 0 for c in TCASES if (c.cin, c.cout) in ((16, 32), (32, 64)) and c.K != 27} == {True}
    assert any(c.nx % 32 == 0 for c in SCASES) and any(c.nx % 32 for c in SCASES)
    assert set(REACHED) == _exports("spconv.cu", "spconv_tc.cu", "sparse_stem.cu")
    assert all(callable(globals()[t]) for t in REACHED.values())


FAULTS = ("flip", "skip_last_kblock", "tap_neighbour", "a_lo", "w_lo", "no_bias", "bias_twice", "no_relu", "row_shift",
          "stale_acc", "down_tap0")


def test_bound_rejects_plausible_kernel_bugs():
    """On a shrunken case of each GEMM kind, each plausible kernel bug restated on the float64 reference leaves the bound on
    some element: a flipped kernel offset, the last active K-block skipped, a 16-channel tap read from the neighbouring offset,
    the lo plane of the input or of the weights dropped, the bias missing or added twice, the ReLU missing, row r written to
    r + 1 at a block / tile edge, accumulators kept from the CTA's previous tile when a tile's first active K-block is not
    block 0, and the stem's downsample read from tap 0 instead of tap 4."""
    applied = set()

    def reject(kind, fault, got, y, bound):
        r = _ratio(np.abs(got - y), bound)
        assert r > 1, f"{kind}: the bound does not reject '{fault}' (max err / bound {r:.3f})"
        applied.add(fault)

    # SIMT gather-GEMM, (16, 16)
    rng = _rng("sharp", "simt")
    nbr, x, w, b, live = _simt_case(16, 16, 27, rng)
    x64, w64, b64 = x.astype(np.float64), w.astype(np.float64), b.astype(np.float64)
    y, pre, s, hits = _gemm_ref(x64, nbr, w64, b64, True, live)
    bound = _simt_bound(pre, s, hits, 16, b)
    for fault in ("flip", "no_bias", "bias_twice", "no_relu", "row_shift"):
        reject("simt", fault, _gemm_ref(x64, nbr, w64, b64, True, live, fault=fault)[0], y, bound)
    # tensor-core gather-GEMM: (16, 16) at K = 27 with two tiles on some CTAs
    case = TCase("sharp", 16, 16, 27, NUM_SMS * SPT_M + 700, NUM_SMS * SPT_M + 800, MIX)
    nbr, xt, wt, bt = _tc_inputs(case)
    assert "late_first_kblock" in _tc_census(case, nbr)[0]
    hi, lo = _split_np(xt)
    a64 = hi.double().numpy() + lo.double().numpy()
    w64, b64 = wt.double().numpy(), bt.double().numpy()
    tiles = (case.tpk, min(-(-case.cap // SPT_M), NUM_SMS), SPT_M)
    y, pre, s, _ = _gemm_ref(a64, nbr, w64, b64, True, case.live)
    bound = _tc_bound(pre, s)
    for fault in ("flip", "skip_last_kblock", "tap_neighbour", "no_bias", "bias_twice", "no_relu", "row_shift", "stale_acc"):
        reject("tc", fault, _gemm_ref(a64, nbr, w64, b64, True, case.live, fault=fault, tiles=tiles)[0], y, bound)
    reject("tc", "a_lo", _gemm_ref(hi.double().numpy(), nbr, w64, b64, True, case.live)[0], y, bound)
    reject("tc", "w_lo", _gemm_ref(a64, nbr, wt.to(torch.bfloat16).double().numpy(), b64, True, case.live)[0], y, bound)
    # the stem, both bounds
    idmap, f, w1, b1, w2, b2 = _stem_inputs(SCASE["taps"])
    conv, y1, s1, hits, y2, s2, cntr = stem_ref(idmap, f, w1, b1, w2, b2)
    for kind in ("heal_sparse_stem", "heal_sparse_stem_tc"):
        bd1, bd2 = _stem_bounds(kind, y1, s1, hits, y2, s2, cntr, b1, b2)
        for fault in ("flip", "no_bias", "no_relu", "down_tap0"):
            r = stem_ref(idmap, f, w1, b1, w2, b2, fault=fault)
            reject(kind, fault, np.r_[r[0].reshape(-1), r[4].reshape(-1)], np.r_[conv.reshape(-1), y2.reshape(-1)],
                   np.r_[bd1.reshape(-1), bd2.reshape(-1)])
    assert applied == set(FAULTS)
