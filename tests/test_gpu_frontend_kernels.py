"""The LiDAR front-end kernels of csrc/points.cu, csrc/voxelize.cu and csrc/pillar_vfe.cu against exact or float64 references,
on inputs built for the places they can go wrong.

heal_mask_points + heal_voxelize (exact).  The references are oracle/pcd.py (shuffle -> ego mask -> strict range mask per agent)
and oracle/voxelizer.c (the sequential voxel generator) + collate, per agent on the rows [off[a], off[a+1]).  Compared bit for
bit: features (as uint32), coords, point counts, num_voxels[0], every per-agent count, the filtered rows and the new offsets.
Rows before off[0] and from off[A] on belong to no agent; both kernels ignore them, so the filtered offsets start at 0.  Voxel
rows at or past the capacity are dropped while num_voxels keeps the true counts; the outputs carry sentinel guard rows past the
capacity and every row from min(M, capacity) on must keep its sentinel.  The bit-exact comparison also shows that no point of a
cell dropped by max_voxels lands in a kept voxel.
  The voxeliser's hash table is restated (slot = (key 2654435761 mod 2^32) >> (32 - lg), 2^lg >= 2 P, lg >= 10, key =
agent cells + cell) so that a case can aim cells at the last slot (a probe that wraps) and at a run of consecutive homes (a long
cluster); _vox_census names what each case contains (scan blocks of 1024 rows crossed, a max_voxels cut in another scan block
than the agent's first row, voxels of exactly 32 / 33 / more than 64 points, 64 agents with empty ones, ...).

heal_pillar_vfe_scatter (float64 with a first-order bound).  The reference is PillarVFE in float64 on the exact fp32 inputs the
kernel reads: voxels, coords, the fp32 folded W, b (ops.fold_linear_bn, itself checked to be the float64 fold rounded once),
the fp32 voxel size v and centre offset o.  Per output channel j of a pillar with n real points, u = 2^-24:
    |err_j| <= max over real points t of  u (11 sum_k |x_tk w_kj| + |b_j|)                    10-term FMA chain + bias add
                                          + sum_{k cluster} |w_kj| (e_mean_k + u |x_tk|)       mean, then the subtraction
                                          + sum_{k centre}  |w_kj| (u |c_k v_k| + u |c_k v_k + o_k| + u |x_tk|)
    e_mean_k = (5 u sum_t |p_tk| + u |sum_t p_tk|) / n     (5-level butterfly sum, one division)
ReLU and the max over the slots are 1-Lipschitz, and a padded slot contributes ReLU(b) exactly, so the largest per-point bound
bounds the output.  Exact relations on the same run: the f32 canvas cell is the pf row bit for bit; the bf16 canvas, the split
canvas and the split rows are hi = RNE-bf16(pf), lo = RNE-bf16(pf - hi); cells no live pillar hits, the channels beside a
channel view and every row past the live count keep their sentinel.  Pillars with n = 0 are out of scope: the voxeliser never
emits one, the reference yields NaN there and the kernel ReLU(b).

heal_pillar_scatter (exact): a copy or its RNE rounding at cell z + y nx + x of image b.  heal_mean_vfe (exact): a sequential
float32 sum over all T slots then an IEEE division by max(n, 1), restated in numpy; and within (T u sum|p| + u |mean|) of the
float64 mean, as the reference's torch expression also is.

test_bound_rejects_plausible_kernel_bugs (no GPU) restates plausible PillarVFE bugs on the float64 reference and shows that the
bound rejects each.  What the GPU tests printed on an H100 80GB HBM3 at a 700 W power limit is kept in MEASURED below."""
import functools
import re
import zlib
from dataclasses import dataclass, field
from pathlib import Path
from typing import Optional, Tuple

import numpy as np
import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]
CSRC = ROOT / "heal_b200" / "csrc"

U = 2.0 ** -24
SENT = 0x5A5A5A5A          # int32 / fp32 sentinel bits of outputs that must stay untouched (fp32: 1.5e16, finite)
SENT16 = 0x5A5A            # bf16 sentinel bits
GUARD = 64                 # sentinel rows behind every output the voxeliser writes
SCAN = 1024                # rows per block of the voxeliser's scans
PV_WARPS_TOTAL = 132 * 8 * 8   # warps of a full heal_pillar_vfe_scatter grid (132 SMs x 8 blocks x 8 warps)
PP_RANGE = [-102.4, -102.4, -3, 102.4, 102.4, 1]
PP_VOXEL = [0.4, 0.4, 4]
SECOND_VOXEL = [0.1, 0.1, 0.1]
EGO = (-1.95, 2.95, -1.1, 1.1)

# What the GPU tests print, on an H100 80GB HBM3 at a 700 W power limit (err / bound of 0 means an exact output).
MEASURED = """
heal_voxelize, 29 cases: exact; e.g. c2_pp 293051 points -> 52804 voxels, c2_second 221181 voxels (T 5), c5_pp 463511 points,
    c2_pp_capacity 52804 voxels on a capacity of 52027 (guard rows untouched), scan_3073_cap1500 2338 voxels, 1500 rows written
heal_mask_points (+ heal_voxelize on its output): exact; 4 option sets, off[0] = 500, 4262 / 4799 of 8460 rows kept;
    c2 full size permuted 291434 rows kept, 52804 voxels
heal_pillar_vfe_scatter, max err / bound: t1 0.643, t5_rounds 0.504, t20_dev_dead 0.390, t32 0.465, t32_dev_dead 0.451,
    t32_dev_zero 0 (nothing written), t32_dev_over 0.450, c2 full size (52804 pillars) 0.444; split rows and the f32 / bf16 /
    split canvas views exact
heal_pillar_scatter, C 4 / 64 / 96 / 128 x f32 / bf16 / split x plain / channel view: exact
heal_mean_vfe: bit-exact to the sequential order; err / bound T 1 0, T 5 0.365 and 0.501 (M 70001), T 32 0.085, M 0 nothing
    written; the torch expression 0 / 0.365 / 0.501 / 0.082
18 refusals, nothing launched or written
"""


def _rng(*what):
    return np.random.default_rng(zlib.crc32("/".join(map(str, what)).encode()))


def _ratio(err, bound):
    err, bound = np.asarray(err, dtype=np.float64), np.asarray(bound, dtype=np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(err == 0, 0.0, err / bound)
    return float(np.nanmax(np.where(np.isnan(r), np.inf, r))) if r.size else 0.0


def _grid(rng_, vs):
    g = (np.array(rng_[3:6]) - np.array(rng_[0:3])) / np.array(vs)
    return np.round(g).astype(np.int64)


def _f32(v):
    return np.float32(v)


def _ulp(v, k):
    """fp32 value k ulps from float32(v) (k < 0: towards -inf)."""
    x = np.float32(v)
    for _ in range(abs(k)):
        x = np.nextafter(x, np.float32(np.inf if k > 0 else -np.inf))
    return x


# ================================================================================================ voxeliser cases
def _cells_f32(pts, rng_, vs):
    """Cell index (z-major, then y, x) of each point as the kernel computes it (fp32 subtract, IEEE divide, floor), -1 outside."""
    g = _grid(rng_, vs)
    q = np.floor((pts[:, :3] - np.asarray(rng_[:3], np.float32)) / np.asarray(vs, np.float32)).astype(np.float64)
    ok = ((q >= 0) & (q < g)).all(1)
    q = np.where(ok[:, None], q, 0).astype(np.int64)
    return np.where(ok, (q[:, 2] * g[1] + q[:, 1]) * g[0] + q[:, 0], -1)


def _cell_points(cells, rng_, vs, rng, spread=0.8):
    """One point strictly inside each (linear) cell, intensity in (0.05, 1)."""
    g = _grid(rng_, vs)
    cells = np.asarray(cells, dtype=np.int64)
    x, y, z = cells % g[0], (cells // g[0]) % g[1], cells // (g[0] * g[1])
    frac = 0.5 + spread * (rng.random((cells.size, 3)) - 0.5)
    xyz = np.asarray(rng_[:3]) + (np.stack([x, y, z], 1) + frac) * np.asarray(vs)
    return np.concatenate([xyz, rng.uniform(0.05, 1, (cells.size, 1))], 1).astype(np.float32)


def _uniform(rng, n, lo=-100.0, hi=100.0, z=(-2.9, 0.9)):
    return np.concatenate([rng.uniform(lo, hi, (n, 2)), rng.uniform(z[0], z[1], (n, 1)), rng.uniform(0.05, 1, (n, 1))],
                          1).astype(np.float32)


def table_log2(n):
    lg = 10
    while (1 << lg) < 2 * n:
        lg += 1
    return lg


def vox_hash(keys, lg):
    return ((np.asarray(keys, dtype=np.uint64) * np.uint64(2654435761)) & np.uint64(0xFFFFFFFF)) >> np.uint64(32 - lg)


def _longest_run(keys, lg):
    """Longest circular run of occupied slots after inserting `keys` by linear probing."""
    T = 1 << lg
    occ = np.zeros(T, dtype=bool)
    for h in vox_hash(keys, lg).tolist():
        s = h
        while occ[s]:
            s = (s + 1) & (T - 1)
        occ[s] = True
    if occ.all():
        return T
    d = np.r_[occ, occ].astype(np.int8)
    edges = np.flatnonzero(np.diff(np.r_[0, d, 0]))
    return int(min((edges[1::2] - edges[0::2]).max(initial=0), T))


@dataclass(frozen=True)
class VCase:
    name: str
    build: str                       # builder name in _BUILDERS
    vs: Tuple[float, float, float]
    T: int
    maxv: int
    cap: object = None               # None: the wrapper's default; an int; 'M-k' / 'M+k' relative to the true voxel count
    arg: object = None               # builder argument
    situations: Tuple[str, ...] = field(default_factory=tuple)


VOX_SITUATIONS = (
    "full_size",          # a C2 / C5 scene of 64-line clouds
    "second_grid",        # the 2048 x 2048 x 40 SECOND grid
    "scan_minus1",        # P = 1024 k - 1, P = 1024 k, P = 1024 k + 1
    "scan_exact",
    "scan_plus1",
    "count_blocks",       # more than 1024 voxels: the count scan has several blocks
    "cut_other_block",    # a max_voxels cut whose first dropped cell appears in another scan block than the agent's first row
    "cut_one",            # max_voxels = 1 with an agent of more cells
    "select_32",          # voxels of exactly 32, 33 and more than 64 points
    "select_33",
    "select_over_64",
    "select_T_over_32",   # T > 32: two rounds of k_select's >= 33-point path
    "static_tail",        # in-range rows from off[A] to P
    "lead_rows",          # in-range rows before off[0]
    "probe_wrap",         # two or more keys whose home is the table's last slot
    "long_cluster",       # 32 or more consecutive occupied slots
    "agents_64",
    "empty_first", "empty_middle", "empty_last",
    "agent_all_out",      # an agent with points, none in range
    "one_point_agent",
    "no_points",          # P = 0
    "range_faces",        # points on a range face and one ulp either side, x, y and z
    "voxel_faces",        # points on voxel boundaries and one ulp either side
    "capacity_cut",       # more voxels than the capacity
)


def _b_scene(arg):
    from oracle import make_golden_fullsize as mgf
    from workloads import synth
    sc = mgf.c2_scene() if arg == "c2" else synth.scene(501, n_agents=8, max_cav=8, rings=64, azimuth=1024)
    return sc["points"], 0, 0


def _b_scan(total):
    rng = _rng("scan", total)
    a = [total // 3, total // 3]
    a.append(total - sum(a))
    clouds = []
    for n in a:
        p = _uniform(rng, n, -105, 105, (-3.2, 1.2))          # some out of range
        rep = rng.random(n) < 0.15
        p[rep] = p[rng.integers(0, n, rep.sum())]
        clouds.append(p)
    return clouds, 0, 0


def _cut_clouds():
    rng = _rng("cut")
    g = _grid(PP_RANGE, PP_VOXEL)
    cells = rng.choice(int(g.prod()), 2000, replace=False)
    a0 = _uniform(rng, 700)
    c1 = cells[:600]
    seq = np.empty(1500, dtype=np.int64)
    firsts = np.sort(rng.choice(np.arange(1, 1300), 598, replace=False))
    k = 1
    seq[0] = 0
    for r in range(1, 1300):
        if k < 599 and r == firsts[k - 1]:
            seq[r] = k
            k += 1
        else:
            seq[r] = rng.integers(0, k)
    seq[1300] = 599
    seq[1301:] = rng.integers(0, 600, 199)
    a1 = _cell_points(c1[seq], PP_RANGE, PP_VOXEL, rng)
    c2 = cells[600:1400]
    a2 = _cell_points(c2[np.r_[np.arange(800), rng.integers(0, 800, 100)]], PP_RANGE, PP_VOXEL, rng)
    return [a0, a1, a2]


def _b_cut(_):
    return _cut_clouds(), 0, 0


def _b_select(_):
    rng = _rng("select")
    g = _grid(PP_RANGE, PP_VOXEL)
    cells = rng.choice(int(g.prod()), 20, replace=False)
    clouds = []
    for counts, cs in (([1, 2, 31, 32, 33, 63, 64, 65, 100, 200], cells[:10]), ([33, 70, 5, 32, 129], cells[10:15])):
        p = _cell_points(np.repeat(cs, counts), PP_RANGE, PP_VOXEL, rng)
        clouds.append(p[rng.permutation(p.shape[0])])
    return clouds, 0, 0


def _b_static(lead):
    rng = _rng("static", lead)
    clouds = [_uniform(rng, 2000), _uniform(rng, 1500)]
    for c in clouds:
        c[rng.integers(0, c.shape[0], 300)] = c[rng.integers(0, c.shape[0], 300)]
    live = np.concatenate(clouds)
    extra = lambda n: np.concatenate([live[rng.integers(0, live.shape[0], n // 2)], _uniform(rng, n - n // 2)])
    return clouds, (extra(700) if lead else 0), extra(800)


def _b_hash(_):
    """Two agents of 1500 rows on the PointPillars grid: keys aimed at the last slot and at a run of 40 consecutive homes."""
    rng = _rng("hash")
    P = 3000
    lg = table_log2(P)
    T = 1 << lg
    cells = int(_grid(PP_RANGE, PP_VOXEL).prod())
    keys = np.arange(2 * cells, dtype=np.int64)
    home = vox_hash(keys, lg).astype(np.int64)
    chosen = list(rng.choice(keys[home == T - 1], 3, replace=False)) + list(rng.choice(keys[home == T - 2], 2, replace=False))
    s0 = T // 3
    for s in range(s0, s0 + 40):
        chosen += list(rng.choice(keys[home == s], 1 + (s % 3 == 0), replace=False))
    chosen = np.asarray(chosen)
    clouds = []
    for a in range(2):
        mine = chosen[chosen // cells == a] % cells
        p = _cell_points(np.repeat(mine, rng.integers(1, 4, mine.size)), PP_RANGE, PP_VOXEL, rng)
        p = np.concatenate([p, _uniform(rng, P // 2 - p.shape[0])])
        clouds.append(p[rng.permutation(p.shape[0])])
    return clouds, 0, 0


def _b_agents64(_):
    rng = _rng("agents64")
    clouds = []
    for a in range(64):
        if a in (0, 31, 63):
            n = 0
        elif a in (5, 40):
            n = 1
        else:
            n = int(rng.integers(2, 200))
        p = _uniform(rng, n)
        if a == 10:                                           # every point outside the range
            p[:, 0] = rng.uniform(102.5, 150, n)
        if n > 4:
            p[rng.integers(0, n, n // 4)] = p[rng.integers(0, n, n // 4)]
        clouds.append(p)
    return clouds, 0, 0


def _face_points(rng_, vs, rng):
    """Points on each range face and one ulp either side, and on voxel boundaries and one ulp either side."""
    g = _grid(rng_, vs)
    inner = np.array([rng_[j] + vs[j] * (g[j] // 2 + 0.5) for j in range(3)], np.float32)
    out = []
    for j in range(3):
        vals = [_ulp(rng_[j], k) for k in (-1, 0, 1)] + [_ulp(rng_[3 + j], k) for k in (-1, 0, 1)]
        for k in rng.choice(int(g[j]) + 1, min(40, int(g[j]) + 1), replace=False):
            vals += [_ulp(rng_[j] + k * vs[j], d) for d in (-2, -1, 0, 1, 2)]
            vals += [_ulp(np.float32(rng_[j]) + np.float32(k) * np.float32(vs[j]), d) for d in (-1, 0, 1)]
        for v in vals:
            p = np.r_[inner, np.float32(0.5)].astype(np.float32)
            p[j] = v
            out.append(p)
    out = np.asarray(out, np.float32)
    return out[rng.permutation(out.shape[0])]


def _b_faces(which):
    rng = _rng("faces", which)
    vs = PP_VOXEL if which == "pp" else SECOND_VOXEL
    f = _face_points(PP_RANGE, vs, rng)
    return [f[: f.shape[0] // 2], f[f.shape[0] // 2:]], 0, 0


def _b_empty(_):
    return [np.zeros((0, 4), np.float32)] * 3, 0, 0


_BUILDERS = {"scene": _b_scene, "scan": _b_scan, "cut": _b_cut, "select": _b_select, "static": _b_static, "hash": _b_hash,
             "agents64": _b_agents64, "faces": _b_faces, "empty": _b_empty}

_PP, _SC = tuple(PP_VOXEL), tuple(SECOND_VOXEL)
VCASES = [
    VCase("c2_pp", "scene", _PP, 32, 70000, arg="c2", situations=("full_size",)),
    VCase("c2_second", "scene", _SC, 5, 70000, arg="c2", situations=("full_size", "second_grid", "count_blocks")),
    VCase("c5_pp", "scene", _PP, 32, 70000, arg="c5", situations=("full_size", "count_blocks")),
    VCase("c2_pp_capacity", "scene", _PP, 32, 70000, cap="M-777", arg="c2", situations=("full_size", "capacity_cut")),
    VCase("scan_1023", "scan", _PP, 32, 70000, arg=1023, situations=("scan_minus1",)),
    VCase("scan_1024", "scan", _PP, 32, 70000, arg=1024, situations=("scan_exact",)),
    VCase("scan_1025", "scan", _PP, 32, 70000, arg=1025, situations=("scan_plus1",)),
    VCase("scan_3071", "scan", _PP, 32, 70000, arg=3071, situations=("scan_minus1", "count_blocks")),
    VCase("scan_3072", "scan", _PP, 32, 70000, arg=3072, situations=("scan_exact", "count_blocks")),
    VCase("scan_3073", "scan", _PP, 32, 70000, arg=3073, situations=("scan_plus1", "count_blocks")),
    VCase("scan_3073_cap1", "scan", _PP, 32, 70000, cap=1, arg=3073, situations=("capacity_cut",)),
    VCase("scan_3073_cap1500", "scan", _PP, 32, 70000, cap=1500, arg=3073, situations=("capacity_cut", "count_blocks")),
    VCase("scan_3073_cap_m1", "scan", _PP, 32, 70000, cap="M-1", arg=3073, situations=("capacity_cut", "count_blocks")),
    VCase("scan_3073_cap_exact", "scan", _PP, 32, 70000, cap="M+0", arg=3073, situations=("count_blocks",)),
    VCase("cut_1", "cut", _PP, 32, 1, situations=("cut_one",)),
    VCase("cut_na_m1", "cut", _PP, 32, 599, situations=("cut_other_block",)),
    VCase("cut_na", "cut", _PP, 32, 600),
    VCase("cut_na_p1", "cut", _PP, 32, 601),
    VCase("select_t5", "select", _PP, 5, 70000, situations=("select_32", "select_33", "select_over_64")),
    VCase("select_t32", "select", _PP, 32, 70000, situations=("select_32", "select_33", "select_over_64")),
    VCase("select_t33", "select", _PP, 33, 70000, situations=("select_33", "select_over_64", "select_T_over_32")),
    VCase("select_t64", "select", _PP, 64, 70000, situations=("select_over_64", "select_T_over_32")),
    VCase("static_tail", "static", _PP, 32, 70000, arg=False, situations=("static_tail",)),
    VCase("lead_rows", "static", _PP, 32, 70000, arg=True, situations=("static_tail", "lead_rows")),
    VCase("hash_wrap_cluster", "hash", _PP, 32, 70000, situations=("probe_wrap", "long_cluster")),
    VCase("agents_64", "agents64", _PP, 32, 70000, situations=("agents_64", "empty_first", "empty_middle", "empty_last",
                                                              "agent_all_out", "one_point_agent")),
    VCase("faces_pp", "faces", _PP, 32, 70000, arg="pp", situations=("range_faces", "voxel_faces")),
    VCase("faces_second", "faces", _SC, 5, 70000, arg="second", situations=("range_faces", "voxel_faces")),
    VCase("no_points", "empty", _PP, 32, 70000, situations=("no_points",)),
]
VCASE = {c.name: c for c in VCASES}


@functools.lru_cache(maxsize=None)
def _vox_inputs(name):
    """(buffer (P,4) f32, offsets (A+1) i32, the agents' clouds): rows [0, off[0]) and [off[A], P) belong to no agent."""
    case = VCASE[name]
    clouds, lead, tail = _BUILDERS[case.build](case.arg)
    clouds = [np.ascontiguousarray(c, dtype=np.float32).reshape(-1, 4) for c in clouds]
    lead = np.zeros((0, 4), np.float32) if isinstance(lead, int) else lead
    tail = np.zeros((0, 4), np.float32) if isinstance(tail, int) else tail
    offs = (lead.shape[0] + np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds])])).astype(np.int32)
    buf = np.concatenate([lead] + clouds + [tail]).astype(np.float32)
    return buf, offs, clouds


def _vox_ref(clouds, vs, T, maxv):
    from oracle import voxelizer
    per_agent = [voxelizer.points_to_voxel_c(c, list(vs), PP_RANGE, T, maxv) for c in clouds]
    return voxelizer.collate(per_agent), [a[0].shape[0] for a in per_agent]


def _capacity(spec, M, P, A, maxv):
    if spec is None:
        return max(1, min(P, A * maxv))
    if isinstance(spec, int):
        return spec
    return max(1, M + int(spec[1:]))


def _vox_census(case):
    """The situations a voxeliser case contains (numpy only)."""
    buf, offs, clouds = _vox_inputs(case.name)
    found = set()
    A, P = len(clouds), buf.shape[0]
    g = _grid(PP_RANGE, case.vs)
    cells_total = int(g.prod())
    per_agent_cells, total_vox = [], 0
    for a, c in enumerate(clouds):
        cl = _cells_f32(c, PP_RANGE, case.vs)
        u, first, cnt = np.unique(cl[cl >= 0], return_index=True, return_counts=True)
        per_agent_cells.append((cl, u, first, cnt))
        total_vox += min(u.size, case.maxv)
        if case.maxv < u.size:
            rows = np.sort(np.flatnonzero(cl >= 0)[first])
            if case.maxv == 1:
                found.add("cut_one")
            if (offs[a] + rows[case.maxv]) // SCAN != offs[a] // SCAN:
                found.add("cut_other_block")
        if (cnt == 32).any():
            found.add("select_32")
        if (cnt == 33).any():
            found.add("select_33")
        if (cnt > 64).any():
            found.add("select_over_64")
        if c.shape[0] and not (cl >= 0).any():
            found.add("agent_all_out")
        if c.shape[0] == 1:
            found.add("one_point_agent")
    if case.T > 32 and any((x[3] > 32).any() for x in per_agent_cells):
        found.add("select_T_over_32")
    if P > 0:
        k = P % SCAN
        found.add({SCAN - 1: "scan_minus1", 0: "scan_exact", 1: "scan_plus1"}.get(k, "scan_other"))
    if total_vox > SCAN:
        found.add("count_blocks")
    M = total_vox
    if case.cap is not None and _capacity(case.cap, M, P, A, case.maxv) < M:
        found.add("capacity_cut")
    if offs[0] > 0:
        found.add("lead_rows")
    if offs[-1] < P:
        found.add("static_tail")
    if P == 0:
        found.add("no_points")
    if A == 64:
        found.add("agents_64")
    sizes = [c.shape[0] for c in clouds]
    if A > 2 and sizes[0] == 0:
        found.add("empty_first")
    if A > 2 and sizes[-1] == 0:
        found.add("empty_last")
    if A > 2 and any(s == 0 for s in sizes[1:-1]):
        found.add("empty_middle")
    if max(g) >= 2048:
        found.add("second_grid")
    if A >= 5 and min(sizes) >= 50000:
        found.add("full_size")
    live = np.concatenate(clouds) if P else np.zeros((0, 4), np.float32)
    if live.shape[0]:
        lo = np.asarray(PP_RANGE[:3], np.float32)
        hi = np.asarray(PP_RANGE[3:], np.float32)
        xyz = live[:, :3]
        if ((xyz == lo) | (xyz == hi)).any(0).all() and (xyz == np.nextafter(lo, -np.inf)).any(0).all():
            found.add("range_faces")
        vsf = np.asarray(case.vs, np.float32)
        q = (xyz - lo) / vsf
        if ((q == np.floor(q)) & (q > 0) & (q < g)).any(0)[:2].all():
            found.add("voxel_faces")
        keys = np.unique(np.concatenate([a * cells_total + x[0][x[0] >= 0] for a, x in enumerate(per_agent_cells)]))
        lg = table_log2(P)
        if int((vox_hash(keys, lg) == (1 << lg) - 1).sum()) >= 2:
            found.add("probe_wrap")
        if _longest_run(keys, lg) >= 32:
            found.add("long_cluster")
    return found


@pytest.mark.parametrize("name", [c.name for c in VCASES if c.build != "scene"])
def test_vox_case_produces_its_situations(name):
    case = VCASE[name]
    found = _vox_census(case)
    assert set(case.situations) <= set(VOX_SITUATIONS)
    assert set(case.situations) <= found, f"{name}: {sorted(set(case.situations) - found)} do not occur"


def test_vox_cases_cover_every_situation():
    """Every situation is declared by some case; the full-size scenes' own census runs with the GPU test."""
    declared = set().union(*(c.situations for c in VCASES))
    assert declared == set(VOX_SITUATIONS), sorted(set(VOX_SITUATIONS) - declared)
    assert {c.T for c in VCASES if c.build == "select"} == {5, 32, 33, 64}
    cl = _cells_f32(_cut_clouds()[1], PP_RANGE, PP_VOXEL)
    n_a = np.unique(cl[cl >= 0]).size
    assert {c.maxv for c in VCASES if c.build == "cut"} == {1, n_a - 1, n_a, n_a + 1}


def test_hash_restatement_matches_the_kernel_source():
    """The restated table (multiplier, shift, size rule) is the one csrc/voxelize.cu uses."""
    src = (CSRC / "voxelize.cu").read_text()
    assert "(key * 2654435761u) >> c.tshift" in src
    assert "int lg = 10;" in src and "while ((1 << lg) < 2 * P) ++lg;" in src
    assert "constexpr int SCAN_BLOCK = 1024;" in src


# ------------------------------------------------------------------------------------------------ voxeliser (GPU)
def _i32(shape, fill=SENT):
    return torch.full(shape, fill, dtype=torch.int32, device="cuda")


def _f32s(shape):
    return _i32(shape).view(torch.float32)


def _vox_call(buf, offs, vs, T, maxv, cap, A=None, P=None, ws_short=0):
    """heal_voxelize into outputs with GUARD sentinel rows past `cap`; returns the device tensors."""
    from heal_b200 import ops
    from heal_b200._lib import lib
    A = len(offs) - 1 if A is None else A
    P = buf.shape[0] if P is None else P
    pts = torch.from_numpy(buf if buf.shape[0] else np.zeros((1, 4), np.float32)).cuda().contiguous()
    od = torch.from_numpy(np.asarray(offs, np.int32)).cuda()
    vox, crd, npt = _f32s((cap + GUARD, T, 4)), _i32((cap + GUARD, 4)), _i32((cap + GUARD,))
    nv = _i32((1 + max(A, 1) + GUARD,))
    wsb = lib.heal_voxelize_workspace(P, cap, max(A, 1))
    ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    ops._call("heal_voxelize", ops._p(pts), ops._p(od), A, P, ops._host_f32(PP_RANGE[0:3]), ops._host_f32(list(vs)),
              ops._host_i32(_grid(PP_RANGE, vs)), T, maxv, cap, ops._p(vox), ops._p(crd), ops._p(npt), ops._p(nv), ops._p(ws),
              wsb - ws_short)
    return vox, crd, npt, nv


def _check_vox(what, outs, ref, counts, cap):
    vox, crd, npt, nv = (t.cpu().numpy() for t in outs)
    A = len(counts)
    M = int(sum(counts))
    k = min(M, cap)
    assert int(nv[0]) == M, f"{what}: num_voxels[0] = {int(nv[0])}, expected {M}"
    assert nv[1:1 + A].tolist() == counts, f"{what}: per-agent counts differ"
    assert (nv[1 + A:] == SENT).all(), f"{what}: num_voxels written past 1 + A"
    assert np.array_equal(crd[:k], ref["voxel_coords"][:k]), f"{what}: coords differ"
    assert np.array_equal(npt[:k], ref["voxel_num_points"][:k]), f"{what}: point counts differ"
    assert np.array_equal(vox[:k].view(np.uint32), ref["voxel_features"][:k].view(np.uint32)), f"{what}: features differ"
    assert (crd[k:] == SENT).all() and (npt[k:] == SENT).all(), f"{what}: rows from min(M, capacity) on were written"
    assert (vox[k:].view(np.uint32) == SENT).all(), f"{what}: voxel rows from min(M, capacity) on were written"
    return M, k


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(VCASE))
def test_voxelize(name):
    case = VCASE[name]
    buf, offs, clouds = _vox_inputs(name)
    if case.build == "scene":
        found = _vox_census(case)
        assert set(case.situations) <= found, f"{name}: {sorted(set(case.situations) - found)} do not occur"
    ref, counts = _vox_ref(clouds, case.vs, case.T, case.maxv)
    M = int(sum(counts))
    cap = _capacity(case.cap, M, buf.shape[0], len(clouds), case.maxv)
    outs = _vox_call(buf, offs, case.vs, case.T, case.maxv, cap)
    torch.cuda.synchronize()
    M, k = _check_vox(name, outs, ref, counts, cap)
    print(f"voxelize {name}: P {buf.shape[0]} (live {offs[-1] - offs[0]}), A {len(clouds)}, T {case.T}, M {M}, capacity {cap}, "
          f"{k} rows written: exact")


def _mask_clouds():
    """Four agents behind 500 lead rows and before 300 tail rows: range faces and ego-box faces, an empty agent, an agent
    entirely inside the ego box, an agent of random points partly out of range."""
    rng = _rng("mask")
    lo, hi = PP_RANGE[:3], PP_RANGE[3:]
    faces = []
    for j in range(3):
        for v in [_ulp(lo[j], k) for k in (-1, 0, 1)] + [_ulp(hi[j], k) for k in (-1, 0, 1)]:
            p = np.array([10.0, -20.0, -1.0, 0.5], np.float32)
            p[j] = v
            faces.append(p)
    for x in [_ulp(EGO[0], k) for k in (-1, 0, 1)] + [_ulp(EGO[1], k) for k in (-1, 0, 1)]:
        for y in [_ulp(EGO[2], k) for k in (-1, 0, 1)] + [_ulp(EGO[3], k) for k in (-1, 0, 1)] + [np.float32(0.3)]:
            faces.append(np.array([x, y, -1.0, 0.5], np.float32))
    faces = np.asarray(faces, np.float32)
    a0 = np.concatenate([faces, _uniform(rng, 2000, -110, 110, (-3.5, 1.5))])
    a0 = a0[rng.permutation(a0.shape[0])]
    ego = np.concatenate([rng.uniform(-1.9, 2.9, (400, 1)), rng.uniform(-1.05, 1.05, (400, 1)), rng.uniform(-2, 0, (400, 1)),
                          rng.uniform(0, 1, (400, 1))], 1).astype(np.float32)
    a3 = _uniform(rng, 6000, -120, 120, (-4, 2))
    a3[:600, :2] = rng.uniform(-3, 3, (600, 2))
    clouds = [a0, np.zeros((0, 4), np.float32), ego, a3]
    live = np.concatenate(clouds)
    lead = np.concatenate([live[rng.integers(0, live.shape[0], 250)], _uniform(rng, 250)])
    tail = np.concatenate([live[rng.integers(0, live.shape[0], 150)], _uniform(rng, 150)])
    return clouds, lead, tail


def _mask_call(buf, offs, perms, remove_ego):
    """heal_mask_points into a sentinel-filled output; returns (rows, offsets) on the host."""
    from heal_b200 import ops
    from heal_b200._lib import lib
    P, A = buf.shape[0], len(offs) - 1
    gperm = None
    if perms is not None:
        gperm = np.arange(P, dtype=np.int32)
        for a, pm in enumerate(perms):
            gperm[offs[a]:offs[a + 1]] = offs[a] + pm
    pts = torch.from_numpy(buf).cuda()
    od = torch.from_numpy(offs).cuda()
    pm = torch.from_numpy(gperm).cuda() if gperm is not None else None
    out, o2 = _f32s((P + GUARD, 4)), _i32((A + 1 + GUARD,))
    wsb = lib.heal_mask_points_workspace(P)
    ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    ops._call("heal_mask_points", ops._p(pts), ops._p(pm), ops._p(od), A, P, ops._host_f32(PP_RANGE), 1 if remove_ego else 0,
              ops._p(out), ops._p(o2), ops._p(ws), wsb)
    torch.cuda.synchronize()
    return out, o2


def _mask_and_voxelize(what, clouds, lead, tail, perms, remove_ego):
    from oracle import pcd
    sizes = [c.shape[0] for c in clouds]
    offs = (lead.shape[0] + np.concatenate([[0], np.cumsum(sizes)])).astype(np.int32)
    buf = np.concatenate([lead] + list(clouds) + [tail]).astype(np.float32)
    ref = [pcd.filter_cloud(c, PP_RANGE, pm, remove_ego) for c, pm in zip(clouds, perms or [None] * len(clouds))]
    ref_offs = np.concatenate([[0], np.cumsum([r.shape[0] for r in ref])]).astype(np.int32)
    out, o2 = _mask_call(buf, offs, perms, remove_ego)
    A = len(clouds)
    got_o = o2.cpu().numpy()
    assert np.array_equal(got_o[:A + 1], ref_offs), f"{what}: offsets {got_o[:A + 1]} != {ref_offs}"
    assert (got_o[A + 1:] == SENT).all(), f"{what}: offsets written past A + 1"
    rows = out.cpu().numpy()
    n = int(ref_offs[-1])
    assert np.array_equal(rows[:n].view(np.uint32), np.concatenate(ref).view(np.uint32)), f"{what}: filtered rows differ"
    assert (rows[n:].view(np.uint32) == SENT).all(), f"{what}: rows past the kept count were written"
    # the voxeliser reads the filtered buffer as it stands: rows past the kept count are sentinels (in range: 1.5e16 is not)
    vref, counts = _vox_ref(ref, PP_VOXEL, 32, 70000)
    M = int(sum(counts))
    outs = _vox_call(rows[:buf.shape[0]], got_o[:A + 1], PP_VOXEL, 32, 70000, max(1, M))
    torch.cuda.synchronize()
    _check_vox(what + " voxelize", outs, vref, counts, max(1, M))
    return n, M


@pytest.mark.gpu
@pytest.mark.parametrize("use_perm", [False, True])
@pytest.mark.parametrize("remove_ego", [True, False])
def test_mask_points_then_voxelize(remove_ego, use_perm):
    """heal_mask_points == shuffle -> ego mask -> strict range mask per agent, on range and ego-box faces one ulp either side,
    with 500 rows before off[0] and 300 after off[A] that belong to no agent; then heal_voxelize on its output."""
    clouds, lead, tail = _mask_clouds()
    rng = _rng("mask_perm")
    perms = [rng.permutation(c.shape[0]).astype(np.int32) for c in clouds] if use_perm else None
    n, M = _mask_and_voxelize(f"mask ego={remove_ego} perm={use_perm}", clouds, lead, tail, perms, remove_ego)
    print(f"mask_points remove_ego={remove_ego} perm={use_perm}: {n} of {sum(c.shape[0] for c in clouds)} rows kept, "
          f"off[0] = {lead.shape[0]}, {M} voxels: exact")


@pytest.mark.gpu
def test_mask_points_then_voxelize_full_size():
    """The C2 scene's unfiltered clouds with a host-drawn permutation through mask_points into voxelize."""
    from oracle import make_golden_fullsize as mgf
    clouds = mgf.c2_scene()["points"]
    rng = _rng("mask_full")
    perms = [rng.permutation(c.shape[0]).astype(np.int32) for c in clouds]
    z = np.zeros((0, 4), np.float32)
    n, M = _mask_and_voxelize("mask c2", clouds, z, z, perms, True)
    print(f"mask_points c2 full size (5 x 65536, permuted): {n} rows kept, {M} voxels: exact")


# ================================================================================================ PillarVFE
def fold64(weight, bn_w, bn_b, bn_mean, bn_var, eps):
    """Linear (Cout, Cin) followed by eval BatchNorm1d, folded in float64: W' (Cin, Cout), b' (Cout)."""
    scale = bn_w.astype(np.float64) / np.sqrt(bn_var.astype(np.float64) + eps)
    shift = bn_b.astype(np.float64) - bn_mean.astype(np.float64) * scale
    return (weight.astype(np.float64) * scale[:, None]).T, shift


def _pv_params(seed):
    """Linear(10, 64) + BatchNorm1d(64) parameters.  Channels 0-15: the only weight is a negative one on the intensity and the
    folded bias is positive, so ReLU(b) lies above every real point's output (intensities are > 0).  Channels 16-31: a negative
    folded bias, so ReLU(b) = 0.  The rest are random."""
    rng = _rng("pv_params", seed)
    w = (rng.standard_normal((64, 10)) * 0.3).astype(np.float32)
    w[:16] = 0
    w[:16, 3] = -rng.uniform(0.5, 2, 16)
    bn_w = rng.uniform(0.5, 1.5, 64).astype(np.float32)
    bn_var = rng.uniform(0.5, 1.5, 64).astype(np.float32)
    bn_mean = (rng.standard_normal(64) * 0.1).astype(np.float32)
    scale = bn_w.astype(np.float64) / np.sqrt(bn_var.astype(np.float64) + 1e-3)
    shift = rng.standard_normal(64) * 0.5
    shift[:16] = rng.uniform(0.5, 2, 16)
    shift[16:32] = -rng.uniform(0.5, 2, 16)
    bn_b = (shift + bn_mean.astype(np.float64) * scale).astype(np.float32)
    return w, bn_w, bn_b, bn_mean, bn_var


def _pv_folded(seed):
    w, bn_w, bn_b, m, v = _pv_params(seed)
    W, b = fold64(w, bn_w, bn_b, m, v, 1e-3)
    return np.ascontiguousarray(W, dtype=np.float32), b.astype(np.float32)       # (Cin, Cout) row-major, as the kernel reads it


def pv_ref(vf, n, coords, W, b, vs, off, fault=None, chunk=2048):
    """PillarVFE in float64 on the fp32 inputs (and the bound of the module docstring).  `fault` restates a kernel bug."""
    M, T, _ = vf.shape
    W64, b64 = W.astype(np.float64), b.astype(np.float64)
    aW = np.abs(W64)
    vs64, off64 = vs.astype(np.float64), off.astype(np.float64)
    out, bound = np.empty((M, 64)), np.empty((M, 64))
    for s in range(0, M, chunk):
        p = vf[s:s + chunk].astype(np.float64)
        nn = n[s:s + chunk].astype(np.float64)
        cd = coords[s:s + chunk]
        m = np.arange(T)[None] < nn[:, None]
        S = p[:, :, :3].sum(1)
        mean = S / (float(T) if fault == "mean_over_T" else nn[:, None])
        cl = p[:, :, :3] - mean[:, None]
        c = cd[:, [2, 3, 1] if fault == "swap_xy" else [3, 2, 1]].astype(np.float64)
        prod = c * vs64
        ctr = prod + off64 + (vs64 / 2 if fault == "half_voxel" else 0)
        ce = p[:, :, :3] - ctr[:, None]
        x = np.concatenate([p, cl, ce], -1) * m[..., None]
        r = np.maximum(x @ W64 + b64, 0)                    # padded slots: x = 0 -> ReLU(b)
        if fault == "fold_skipped":
            r = np.where(m[..., None], r, 0)
        o = r.max(1)
        if fault == "fold_when_full":
            o = np.maximum(o, np.maximum(b64, 0))
        out[s:s + chunk] = o
        if fault is None:
            em = (5 * U * np.abs(p[:, :, :3]).sum(1) + U * np.abs(S)) / nn[:, None]
            ecl = em[:, None] + U * np.abs(cl)
            ece = U * (np.abs(prod) + np.abs(ctr))[:, None] + U * np.abs(ce)
            pb = U * (11 * (np.abs(x) @ aW) + np.abs(b64)) + ecl @ aW[4:7] + ece @ aW[7:10]
            bound[s:s + chunk] = np.where(m[..., None], pb, 0).max(1)
    return out, bound


@dataclass(frozen=True)
class PCase:
    name: str
    T: int
    M: int                   # rows passed as num_voxels
    live: Optional[int]      # num_voxels_dev[0], or None (not passed)
    extra: int = 0           # valid pillars at otherwise empty cells in rows [M, M + extra) (never to be read)
    B: int = 3
    ny: int = 144
    nx: int = 176


PCASES = [
    PCase("t1", 1, 3001, None),
    PCase("t5_rounds", 5, 4 * PV_WARPS_TOTAL + 1234, None),     # five rounds of the persistent warps
    PCase("t20_dev_dead", 20, 5000, 3999, extra=100),
    PCase("t32", 32, PV_WARPS_TOTAL + 553, None),
    PCase("t32_dev_dead", 32, 12000, 9001),
    PCase("t32_dev_zero", 32, 2000, 0),
    PCase("t32_dev_over", 32, 3000, 3500, extra=200),
]
PCASE = {c.name: c for c in PCASES}
VS32 = np.asarray(PP_VOXEL, np.float32)
OFF32 = np.asarray([PP_VOXEL[i] / 2 + PP_RANGE[i] for i in range(3)], np.float32)


@functools.lru_cache(maxsize=None)
def _pv_inputs(name):
    """(voxels (R,T,4), n (R,), coords (R,4) [b, 0, y, x]) with R = M + extra rows, each row at its own cell.  Point counts
    cycle through 1, 2, T - 1, T and random ones; the last agent's last row and column are used."""
    case = PCASE[name]
    rng = _rng("pv", name)
    R = case.M + case.extra
    cells = rng.choice(case.B * case.ny * case.nx, R, replace=False)
    last = (case.B - 1) * case.ny * case.nx
    corner = [last + case.ny * case.nx - 1, last + (case.ny - 1) * case.nx, last + case.nx - 1]
    for i, cc in enumerate(corner):
        j = np.flatnonzero(cells == cc)
        if j.size:
            cells[j[0]], cells[i] = cells[i], cells[j[0]]
        else:
            cells[i] = cc
    b, y, x = cells // (case.ny * case.nx), (cells // case.nx) % case.ny, cells % case.nx
    coords = np.stack([b, np.zeros_like(b), y, x], 1).astype(np.int32)
    T = case.T
    cyc = np.array([v for v in (1, 2, T - 1, T) if 1 <= v <= T])
    n = np.where(np.arange(R) % 2 == 0, cyc[np.arange(R) // 2 % cyc.size], rng.integers(1, T + 1, R)).astype(np.int32)
    vf = np.zeros((R, T, 4), np.float32)
    pos = np.stack([x, y], 1)[:, None, :] + rng.uniform(0.02, 0.98, (R, T, 2))
    vf[..., :2] = np.asarray(PP_RANGE[:2]) + pos * np.asarray(PP_VOXEL[:2])
    vf[..., 2] = rng.uniform(-2.9, 0.9, (R, T))
    vf[..., 3] = rng.uniform(0.05, 1, (R, T))
    vf[np.arange(T)[None] >= n[:, None]] = 0
    return vf, n, coords


def _split_np(t):
    hi = t.to(torch.bfloat16)
    return hi, (t - hi.float()).to(torch.bfloat16)


def _bf16s(shape):
    return torch.full(shape, SENT16, dtype=torch.int16, device="cuda").view(torch.bfloat16)


def _canvas(fmt, B, ny, nx, cs):
    if fmt == "f32":
        return _f32s((B, ny, nx, cs))
    return _bf16s((2 if fmt == "split" else 1, B, ny, nx, cs))


def _hact(buf, fmt, cs, co):
    from heal_b200._lib import HealAct
    from heal_b200 import ops
    return HealAct(buf.data_ptr(), ops.FMT[fmt], cs, co, buf[0].numel() if fmt != "f32" else 0)


def _expected_canvas(fmt, B, ny, nx, cs, co, cells, rows):
    """Sentinel canvas with `rows` (m, C) f32 stored at flat cells `cells` in channels [co, co + C)."""
    exp = _canvas(fmt, B, ny, nx, cs)
    C = rows.shape[1]
    if fmt == "f32":
        exp.view(-1, cs)[cells, co:co + C] = rows
    else:
        hi, lo = _split_np(rows)
        exp[0].view(-1, cs)[cells, co:co + C] = hi
        if fmt == "split":
            exp[1].view(-1, cs)[cells, co:co + C] = lo
    return exp


def _same_bits(a, b):
    if a.dtype == torch.float32:
        return torch.equal(a.view(torch.int32), b.view(torch.int32))
    return torch.equal(a.view(torch.int16), b.view(torch.int16))


def _pv_run(vf, n, coords, M, live, W, b, B, ny, nx, fmt, cs, co):
    """One heal_pillar_vfe_scatter call with pf rows, split rows and a canvas view, all sentinel-filled."""
    from heal_b200 import ops
    R, T = vf.shape[0], vf.shape[1]
    vd, nd, cd, wd, bd = (torch.from_numpy(a).cuda() for a in (vf, n, coords, W, b))      # held until the kernel has run
    nvd = torch.tensor([live], dtype=torch.int32, device="cuda") if live is not None else None
    pf, split = _f32s((R, 64)), _bf16s((R, 128))
    canvas = _canvas(fmt, B, ny, nx, cs)
    ops._call("heal_pillar_vfe_scatter", ops._p(vd), ops._p(nd), ops._p(cd), ops._p(nvd), M, T,
              ops._p(wd), ops._p(bd), 10, 64,
              ops._host_f32(list(VS32)), ops._host_f32(list(OFF32)), nx, ny, ops._p(pf), ops._p(split), _hact(canvas, fmt, cs, co))
    torch.cuda.synchronize()
    return pf, split, canvas


def _pv_check(what, vf, n, coords, M, live, W, b, B, ny, nx, views=(("f32", 192, 64), ("bf16", 192, 64), ("split", 192, 64))):
    k = M if live is None else max(0, min(M, live))
    ref, bound = pv_ref(vf[:k], n[:k], coords[:k], W, b, VS32, OFF32)
    cells = torch.from_numpy((coords[:k, 0].astype(np.int64) * ny + coords[:k, 2]) * nx + coords[:k, 3]).cuda()
    pf0 = None
    for fmt, cs, co in views:
        pf, split, canvas = _pv_run(vf, n, coords, M, live, W, b, B, ny, nx, fmt, cs, co)
        if pf0 is None:
            pf0 = pf
            got = pf[:k].cpu().numpy().astype(np.float64)
            r = _ratio(np.abs(got - ref), bound)
            assert r <= 1, f"{what}: max err / bound {r:.3f}"
        else:
            assert _same_bits(pf, pf0), f"{what} {fmt}: pf differs between runs"
        assert bool((pf[k:].view(torch.int32) == SENT).all()), f"{what}: pf rows past the live count were written"
        hi, lo = _split_np(pf[:k])
        assert _same_bits(split[:k, :64], hi) and _same_bits(split[:k, 64:], lo), f"{what}: split rows != RNE split of pf"
        assert bool((split[k:].view(torch.int16) == SENT16).all()), f"{what}: split rows past the live count were written"
        assert _same_bits(canvas, _expected_canvas(fmt, B, ny, nx, cs, co, cells, pf[:k])), \
            f"{what} {fmt} (cstride {cs}, coffset {co}): canvas differs (hit cells, untouched cells or neighbouring channels)"
    return r, k


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(PCASE))
def test_pillar_vfe_scatter(name):
    case = PCASE[name]
    vf, n, coords = _pv_inputs(name)
    W, b = _pv_folded(name)
    r, k = _pv_check(name, vf, n, coords, case.M, case.live, W, b, case.B, case.ny, case.nx)
    print(f"pillar_vfe_scatter {name}: T {case.T}, M {case.M}, live {k}, max err / bound {r:.3f}; split rows and f32 / bf16 / "
          f"split canvas views exact")


@pytest.mark.gpu
def test_pillar_vfe_scatter_full_size():
    """The voxeliser's output for the full-size C2 scene into a plain 64-channel canvas and a 192-channel view."""
    from heal_b200 import ops
    from oracle import make_golden_fullsize as mgf
    clouds = mgf.c2_scene()["points"]
    offs = np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds])]).astype(np.int32)
    buf = np.concatenate(clouds)
    vox, crd, npt, nv = ops.voxelize(torch.from_numpy(buf).cuda(), torch.from_numpy(offs).cuda(), PP_RANGE, PP_VOXEL, 32, 70000)
    M = int(nv[0].item())
    vf, n, coords = (t[:M].cpu().numpy() for t in (vox, npt, crd))
    W, b = _pv_folded("c2")
    r, k = _pv_check("c2", vf, n, coords, M, M, W, b, len(clouds), 512, 512,
                     views=(("f32", 64, 0), ("split", 192, 64)))
    print(f"pillar_vfe_scatter c2 full size: {M} pillars, max err / bound {r:.3f}; canvases exact")


def test_fold_linear_bn_is_the_float64_fold_rounded_once():
    from heal_b200 import ops
    w, bn_w, bn_b, m, v = _pv_params("fold")
    W64, b64 = fold64(w, bn_w, bn_b, m, v, 1e-3)
    W, b = ops.fold_linear_bn(*(torch.from_numpy(a) for a in (w, bn_w, bn_b, m, v)), 1e-3)
    assert W.dtype == torch.float32 and W.shape == (10, 64)
    assert np.array_equal(W.numpy().view(np.uint32), W64.astype(np.float32).view(np.uint32))
    assert np.array_equal(b.numpy().view(np.uint32), b64.astype(np.float32).view(np.uint32))


FAULTS = ("mean_over_T", "fold_skipped", "fold_when_full", "half_voxel", "swap_xy")


def test_bound_rejects_plausible_kernel_bugs():
    """On a shrunken T = 20 case, each plausible bug restated on the float64 reference leaves the bound on some element: the
    mean over T instead of n, the padded-slot ReLU(b) fold skipped or applied to a full pillar, a centre offset moved by half a
    voxel, x and y swapped in the centre."""
    vf, n, coords = (a[:600] for a in _pv_inputs("t20_dev_dead"))
    assert (n == 20).any() and (n < 20).any()
    W, b = _pv_folded("t20_dev_dead")
    ref, bound = pv_ref(vf, n, coords, W, b, VS32, OFF32)
    assert (bound > 0).all()
    for fault in FAULTS:
        got = pv_ref(vf, n, coords, W, b, VS32, OFF32, fault=fault)[0]
        r = _ratio(np.abs(got - ref), bound)
        assert r > 1, f"the bound does not reject '{fault}' (max err / bound {r:.3f})"


# ================================================================================================ PointPillarScatter
@pytest.mark.gpu
@pytest.mark.parametrize("C", [4, 64, 96, 128])
def test_pillar_scatter(C):
    """Rows -> cell z + y nx + x of image b, f32 / bf16 / split, into a channel view; rows past num_voxels_dev are dead and
    hold valid rows at otherwise empty cells."""
    from heal_b200 import ops
    rng = _rng("scatter", C)
    B, ny, nx, M, live = 3, 40, 56, 2500, 2100
    cells = rng.choice(B * ny * nx, M, replace=False)
    b, rest = cells // (ny * nx), cells % (ny * nx)
    y, x = rest // nx, rest % nx
    z = np.where(rng.random(M) < 0.3, np.minimum(x, rng.integers(1, 4, M)), 0)     # z != 0 moves x back by z
    coords = np.stack([b, z, y, x - z], 1).astype(np.int32)
    feats = (rng.standard_normal((M, C)) * 3).astype(np.float32)
    fd, cd = torch.from_numpy(feats).cuda(), torch.from_numpy(coords).cuda()
    nvd = torch.tensor([live], dtype=torch.int32, device="cuda")
    assert (z > 0).any()
    tcells = torch.from_numpy(cells[:live]).cuda()
    # the reference's own index z + y nx + x (point_pillar_scatter.py), via the oracle
    from oracle import nets
    ref = nets.scatter(torch.from_numpy(feats[:live]), torch.from_numpy(coords[:live]), nx, ny, B)
    for fmt in ("f32", "bf16", "split"):
        for cs, co in ((C, 0), (C + 64, 32)):
            canvas = _canvas(fmt, B, ny, nx, cs)
            ops._call("heal_pillar_scatter", ops._p(fd), ops._p(cd), ops._p(nvd), M, C, nx, ny, _hact(canvas, fmt, cs, co))
            torch.cuda.synchronize()
            assert _same_bits(canvas, _expected_canvas(fmt, B, ny, nx, cs, co, tcells, fd[:live])), f"C {C} {fmt} cs {cs}"
            if fmt == "f32" and co == 0:
                got = canvas.view(-1, cs)[:, :C].cpu().clone()
                got[got.view(torch.int32) == SENT] = 0
                assert torch.equal(got.view(B, ny, nx, C).permute(0, 3, 1, 2), ref)
    print(f"pillar_scatter C {C}: f32 / bf16 / split, plain and channel view, {live} live of {M}: exact")


# ================================================================================================ MeanVFE
def mean_f32(v, n):
    """heal_mean_vfe's documented order: a float32 sum over all T slots in order, then an IEEE division by max(n, 1)."""
    s = np.zeros((v.shape[0], 4), np.float32)
    for t in range(v.shape[1]):
        s = (s + v[:, t]).astype(np.float32)
    return s / np.maximum(n.astype(np.float32), np.float32(1))[:, None]


@pytest.mark.gpu
@pytest.mark.parametrize("T,M", [(1, 1153), (5, 1000), (5, 70001), (32, 4099), (32, 0)])
def test_mean_vfe(T, M):
    from heal_b200 import ops
    rng = _rng("mean", T, M)
    v = (rng.standard_normal((M, T, 4)) * rng.uniform(0.1, 100, (M, 1, 1))).astype(np.float32)
    n = rng.integers(0, T + 1, M).astype(np.int32)
    n[: min(M, 7)] = 0
    v[np.arange(T)[None] >= n[:, None]] = 0
    vd, nd = torch.from_numpy(v).cuda(), torch.from_numpy(n).cuda()
    out = _f32s((M + GUARD, 4))
    ops._call("heal_mean_vfe", ops._p(vd), ops._p(nd), M, T, ops._p(out))
    got = out.cpu().numpy()
    assert (got[M:].view(np.uint32) == SENT).all(), "rows past M were written"
    got = got[:M]
    assert np.array_equal(got.view(np.uint32), mean_f32(v, n).view(np.uint32)), "not the documented summation order"
    den = np.maximum(n, 1).astype(np.float64)[:, None]
    ref64 = v.astype(np.float64).sum(1) / den
    bound = T * U * np.abs(v.astype(np.float64)).sum(1) / den + U * np.abs(ref64)
    ref_t = (torch.from_numpy(v).sum(1) / torch.clamp_min(torch.from_numpy(n).view(-1, 1), 1.0).float()).numpy()
    r, rt = _ratio(np.abs(got - ref64), bound), _ratio(np.abs(ref_t - ref64), bound)
    assert r <= 1 and rt <= 1, (r, rt)
    print(f"mean_vfe T {T} M {M}: bit-exact to the sequential order; err / bound {r:.3f} (torch expression {rt:.3f})")


# ================================================================================================ refusals
REFUSALS = [
    ("vox_agents0", "heal_voxelize", "HEAL_ERR_ARG"),
    ("vox_agents65", "heal_voxelize", "HEAL_ERR_ARG"),
    ("vox_T0", "heal_voxelize", "HEAL_ERR_ARG"),
    ("vox_maxv0", "heal_voxelize", "HEAL_ERR_ARG"),
    ("vox_P_over", "heal_voxelize", "HEAL_ERR_ARG"),
    ("vox_cells", "heal_voxelize", "HEAL_ERR_ARG"),
    ("vox_workspace", "heal_voxelize", "HEAL_ERR_WORKSPACE"),
    ("mask_agents0", "heal_mask_points", "HEAL_ERR_ARG"),
    ("mask_agents65", "heal_mask_points", "HEAL_ERR_ARG"),
    ("mask_workspace", "heal_mask_points", "HEAL_ERR_WORKSPACE"),
    ("pv_cin9", "heal_pillar_vfe_scatter", "HEAL_ERR_UNSUPPORTED"),
    ("pv_cout32", "heal_pillar_vfe_scatter", "HEAL_ERR_UNSUPPORTED"),
    ("pv_T0", "heal_pillar_vfe_scatter", "HEAL_ERR_UNSUPPORTED"),
    ("pv_T33", "heal_pillar_vfe_scatter", "HEAL_ERR_UNSUPPORTED"),
    ("pv_odd_cstride", "heal_pillar_vfe_scatter", "HEAL_ERR_UNSUPPORTED"),
    ("pv_odd_coffset", "heal_pillar_vfe_scatter", "HEAL_ERR_UNSUPPORTED"),
    ("scatter_c0", "heal_pillar_scatter", "HEAL_ERR_ARG"),
    ("mean_T0", "heal_mean_vfe", "HEAL_ERR_ARG"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("what, symbol, error", REFUSALS)
def test_refusals(what, symbol, error):
    """Each unsupported call is refused by name, nothing is launched and every output keeps its sentinel."""
    from heal_b200 import ops
    from heal_b200._lib import lib
    pts = torch.zeros((64, 4), dtype=torch.float32, device="cuda")
    offs = torch.tensor([0] + [1] * 65, dtype=torch.int32, device="cuda")
    outs = [_i32((4096,)) for _ in range(4)]
    canvas = _f32s((1, 4, 4, 130))
    p = ops._p
    sent = [o.clone() for o in outs] + [canvas.clone()]

    def call():
        if symbol == "heal_voxelize":
            A = {"vox_agents0": 0, "vox_agents65": 65, "vox_cells": 26}.get(what, 2)
            vs = SECOND_VOXEL if what == "vox_cells" else PP_VOXEL
            P = (1 << 20) + 1 if what == "vox_P_over" else 64
            T = 0 if what == "vox_T0" else 4
            maxv = 0 if what == "vox_maxv0" else 16
            wsb = lib.heal_voxelize_workspace(P, 16, max(A, 1))
            ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
            ops._call(symbol, p(pts), p(offs), A, P, ops._host_f32(PP_RANGE[:3]), ops._host_f32(vs),
                      ops._host_i32(_grid(PP_RANGE, vs)), T, maxv, 16, p(outs[0]), p(outs[1]), p(outs[2]), p(outs[3]), p(ws),
                      wsb - 1 if what == "vox_workspace" else wsb)
        elif symbol == "heal_mask_points":
            A = {"mask_agents0": 0, "mask_agents65": 65}.get(what, 2)
            wsb = lib.heal_mask_points_workspace(64)
            ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
            ops._call(symbol, p(pts), ops._vp(0), p(offs), A, 64, ops._host_f32(PP_RANGE), 1, p(outs[0]), p(outs[1]), p(ws),
                      wsb - 1 if what == "mask_workspace" else wsb)
        elif symbol == "heal_pillar_vfe_scatter":
            cin, cout = (9 if what == "pv_cin9" else 10), (32 if what == "pv_cout32" else 64)
            T = {"pv_T0": 0, "pv_T33": 33}.get(what, 4)
            cs = 129 if what == "pv_odd_cstride" else 130
            co = 1 if what == "pv_odd_coffset" else 0
            ops._call(symbol, p(outs[0]), p(outs[1]), p(outs[2]), ops._vp(0), 1, T, p(outs[3]), p(outs[3]), cin, cout,
                      ops._host_f32(PP_VOXEL), ops._host_f32([0.2, 0.2, 0.2]), 4, 4, p(outs[0]), p(outs[1]),
                      _hact(canvas, "f32", cs, co))
        elif symbol == "heal_pillar_scatter":
            ops._call(symbol, p(outs[0]), p(outs[1]), ops._vp(0), 1, 0, 4, 4, _hact(canvas, "f32", 130, 0))
        else:
            ops._call(symbol, p(outs[0]), p(outs[1]), 1, 0, p(outs[2]))

    torch.cuda.synchronize()
    before = lib.heal_launch_count()
    with pytest.raises(RuntimeError, match=f"{symbol} failed: {error}"):
        call()
    torch.cuda.synchronize()
    assert lib.heal_launch_count() == before
    assert all(_same_bits(a, b) for a, b in zip(outs + [canvas], sent)), "an output was written"


# ================================================================================================ coverage (CPU)
def _exports(*paths):
    return {m for p in paths for m in re.findall(r'extern "C" \w+ (heal_\w+)\(', (CSRC / p).read_text())}


REACHED = {
    "heal_mask_points_workspace": "test_mask_points_then_voxelize", "heal_mask_points": "test_mask_points_then_voxelize",
    "heal_voxelize_workspace": "test_voxelize", "heal_voxelize": "test_voxelize", "heal_mean_vfe": "test_mean_vfe",
    "heal_pillar_vfe_scatter": "test_pillar_vfe_scatter", "heal_pillar_scatter": "test_pillar_scatter",
}


def test_every_entry_point_is_reached():
    assert set(REACHED) == _exports("points.cu", "voxelize.cu", "pillar_vfe.cu")
    assert all(callable(globals()[t]) for t in REACHED.values())
    assert any(c.M > PV_WARPS_TOTAL for c in PCASES) and any(c.M > 3 * PV_WARPS_TOTAL for c in PCASES)
    assert {c.T for c in PCASES} == {1, 5, 20, 32}
    lives = [(c.M, c.live) for c in PCASES if c.live is not None]
    assert any(l == 0 for _, l in lives) and any(0 < l < M for M, l in lives) and any(l > M for M, l in lives)
