"""The post-processing kernels of csrc/postprocess.cu against a float64 (or exact) reference restated in this file.

The kernels (k_decode, the cub sort, k_gather_top, k_iou_mask, k_nms_finish, k_emit) sit behind three C entry points; every case
drives them through ops.box_decode_nms, ops.box_decode_nms_multi or ops.box_decode_nms_late and isolates a stage with the call's
own parameters.  u = 2^-24 is the fp32 unit roundoff.

Decode, score threshold, size / z filters (k_decode).  nms_threshold = 2.0 (an IoU is never above it), `top` >= the candidate
count, no gt_range: the output is every surviving candidate in sort order.  The reference is a float64 restatement of
delta_to_boxes3d -> direction-bin fix (limit_period twice) -> boxes_to_corners_3d -> project_box3d on the fp32 inputs the kernel
reads.  Each output box is identified with its candidate by its centre (cases keep centres >= MIN_SEP apart); the set and the
order must match exactly and `stats` must equal the exact counts after the threshold and after the filters.
  Corners: a first-order bound per coordinate, built from the kernel's operation sequence: sqrtf (3u relative on the anchor
  diagonal), expf (2 ulp = 4u, plus the product: 5u on each size), the direction fix (one rounding per operation on |v|,
  |k| period, |rot|, |offset|, |y2| and the final 2 pi wrap, plus the fp32 rounding of 2 pi / bins and 2 pi), sinf / cosf
  (2 ulp = 4u |cos|, plus the yaw error), two roundings per term of the rotated corner and four in the 4x4 projection.
  corner_bound() spells it out; no blanket tolerance.
  Scores: SCORE_REL = 8u relative for the sigmoid (expf 2 ulp, the add, the division); SCORE_REL_IOU = 40u with the IoU factor
  ((clamp(sigmoid(q), 0, 1) + 1) / 2)^4 (the same sigmoid error on q, four times over through powf's 4 ulp).
  Generated candidates keep every decision outside MARGIN times its bound: logit vs logit(thr), x / y length vs 6, z vs -3 / 1,
  the first limit_period's floor; adjacent scores of different candidates are separated by more than MARGIN times the sum of
  their bounds.  _decode_census asserts all of it.  The edge cases are exact instead (zero deltas, yaw 0, dyadic sizes,
  identity transform): there both sides decide identically at exactly 6 m, exactly -3, exactly 1 and y_len == 0, and the
  kernel's corners must equal the float64 ones.
  Non-finite inputs: NaN / -inf logits fail the threshold, +inf passes with score 1; inf / NaN deltas give inf or NaN corners
  that fail the filters (a NaN corner drops the box, as the reference's NaN lengths do).  Where the kernel and torch differ by
  design, the kernel's rule is the specification here: a NaN direction logit never wins the argmax scan (a NaN in bin 0 keeps
  bin 0), and a NaN IoU logit counts as sigmoid 0, so the score is multiplied by 1/16.

Sort and top cut (cub + k_gather_top).  Order: descending score, then ascending candidate slot
slot = cav * H*W*A + (h*W + w)*A + a.  Ties come from identical logits (also across cavs) or from sigmoids that round to 1.0f.
Candidate counts top - 1, top and top + 1 for top in 1, 63, 64, 65, 128, 1000, 1320, tie groups straddling the cut, and
high-scored candidates that the size filter drops (the cut comes after the filters).  The expected list is the first `top`.
These boxes are exact (dyadic anchors, zero deltas), so corners must match bit for bit.

Rotated NMS (k_iou_mask + k_nms_finish).  A decode-only run gives the kernel's own fp32 corners and order; ref_nms runs the
reference's greedy NMS on exactly those corners in float64 (Sutherland-Hodgman clipping of the counter-clockwise quads, IoU
cast to fp32 and compared with the fp32 threshold with `>`).  The pick list must match index for index, boxes and scores bit
for bit.  Every generated pair that is clipped has |IoU - thr| > NEAR_THR (the GPU's FMA-contracted float64 may round
differently closer than that); only the built exact cases come closer.

Range mask.  The output with gt_range must equal the output without it, filtered by the float64 test lo <= c <= hi on the
kernel's own corners: the reference's mask_boxes_outside_range_numpy compares fp32 corners with a float64 slice of the range.

Entry points.  single, multi (1, 2 and 16 cavs) and late give bit-identical outputs on the same cavs, and every run repeats
bit for bit.

test_bound_rejects_plausible_kernel_bugs (no GPU) restates nine plausible bugs on the reference and shows that the comparisons
above reject each.  What the GPU tests printed on an H100 is kept in MEASURED below."""
import math
import os
from dataclasses import dataclass
from typing import List, Optional, Tuple

import numpy as np
import pytest
import torch

U = 2.0 ** -24
TWO_PI = 2.0 * math.pi
SCORE_REL = 8 * U
SCORE_REL_IOU = 40 * U
MARGIN = 2.0               # generated decisions stay MARGIN x their bound away from the edge
MIN_SEP = 0.05             # least distance between the centres of two surviving candidates (m)
NEAR_THR = 1e-9            # least |IoU - thr| of a generated clipped pair
THR = 0.2                  # score threshold of every case
THR32 = float(np.float32(THR))   # the kernel compares the fp32 sigmoid with the fp32 threshold
LOGIT_THR = math.log(THR / (1.0 - THR))
DIR_OFFSET = float(np.float32(0.7853))

MEASURED = """
H100 80GB HBM3, 700 W power limit; the whole file ran in 17 s (pytest -m gpu -s prints these lines).
decode   largest err / bound, corners and scores:
  hwl_bins2_A2 0.311 / 0.291, lhw_bins4_A3_argmax_ties 0.273 / 0.224, hwl_bins1_A1_offset0 0.307 / 0.226,
  nodir_A2_views_saturated 0.232 / 0.268, multi2_iou_views 0.250 / 0.149, late3_views_ties 0.298 / 0.216,
  multi1_iou_nonfinite 0.268 / 0.116, late2_bins4_nonfinite 0.254 / 0.202
  exact edges, sort and top cut: bit-exact corners (err 0)
nms      boxes, pairs clipped, pairs above the threshold, picks, least |IoU - thr| of a clipped pair:
  n63 63 38 26 38 0.00214, n64 64 41 33 34 0.0264, n65_chain 65 41 35 31 0.00827, n127 127 79 69 60 0.00186,
  n128 128 92 73 62 0.0064, n129_chain 129 91 78 55 0.00273, n1320_chains 1320 875 716 647 0.000514,
  n300_clockwise 300 198 157 153 0.000647, exact_pairs 16 8 2 14 0.0875, exact_thr_0.5 4 2 1 3 0 (built),
  exact_thr_0.25 4 2 1 3 0 (built), identical_1320 1320 1319 1319 1 0.85, disjoint_1320 1320 0 0 1320 -
"""


# ---------------------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------------------
@dataclass
class Cav:
    cls: np.ndarray                       # (H, W, A) fp32 logits
    reg: np.ndarray                       # (H, W, 7A) fp32 deltas
    dir: Optional[np.ndarray]             # (H, W, A*bins) fp32 or None
    iou: Optional[np.ndarray]             # (H, W, A) fp32 or None
    T: np.ndarray                         # (4, 4) fp32 cav -> ego


@dataclass
class Inputs:
    anchors: np.ndarray                   # (H, W, A, 7) fp32, shared by every cav
    cavs: List[Cav]
    bins: int = 0                         # 0: no direction head
    order: str = "hwl"
    dir_offset: float = DIR_OFFSET
    special: Optional[np.ndarray] = None  # (N,) planted on purpose (ties, saturation, non-finite): not moved by the margin fixes
    exact: Optional[np.ndarray] = None    # (N,) built with exact arithmetic: no margin needed, corners must be exact

    @property
    def shape(self):
        return self.anchors.shape[:3]

    @property
    def n1(self):
        H, W, A = self.shape
        return H * W * A

    @property
    def N(self):
        return self.n1 * len(self.cavs)


def _rz(theta, tx=0.0, ty=0.0, tz=0.0, tilt=0.0):
    c, s = math.cos(theta), math.sin(theta)
    R = np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]], dtype=np.float64)
    if tilt:
        ct, st = math.cos(tilt), math.sin(tilt)
        R = R @ np.array([[1, 0, 0], [0, ct, -st], [0, st, ct]])
    T = np.eye(4)
    T[:3, :3] = R
    T[:3, 3] = (tx, ty, tz)
    return T.astype(np.float32)


# ---------------------------------------------------------------------------------------------------------------------------
# float64 reference of the decode
# ---------------------------------------------------------------------------------------------------------------------------
SX = np.array([1, 1, -1, -1, 1, 1, -1, -1], dtype=np.float64)
SY = np.array([-1, 1, 1, -1, -1, 1, 1, -1], dtype=np.float64)
SZ = np.array([-1, -1, -1, -1, 1, 1, 1, 1], dtype=np.float64)


def _sigmoid(x):
    with np.errstate(over="ignore", invalid="ignore"):
        return 1.0 / (1.0 + np.exp(-x))


@dataclass
class Ref:
    slot: np.ndarray
    logit: np.ndarray
    iou_logit: Optional[np.ndarray]
    prob: np.ndarray
    passed: np.ndarray
    keep: np.ndarray
    score: np.ndarray
    score_bound: np.ndarray
    corners: np.ndarray                   # (N, 8, 3) float64
    bound: np.ndarray                     # (N, 8, 3)
    margins: dict                         # name -> (N,) margin / bound (inf where not applicable)
    wrapped: np.ndarray                   # the final limit_period moved the yaw by 2 pi
    lab: np.ndarray
    finite: np.ndarray
    x_len: np.ndarray
    y_len: np.ndarray
    z_min: np.ndarray
    z_max: np.ndarray

    @property
    def centre(self):
        return self.corners.mean(axis=1)


def ref_decode(inp: Inputs, bug=()) -> Ref:
    """k_decode's specification in float64.  bug: restated kernel bugs (test_bound_rejects_plausible_kernel_bugs)."""
    H, W, A = inp.shape
    n1 = inp.n1
    an = inp.anchors.reshape(-1, 7).astype(np.float64)
    acc = {k: [] for k in ("slot", "logit", "iou", "prob", "passed", "keep", "score", "sb", "corners", "bound", "wrapped",
                           "lab", "finite", "xl", "yl", "zmin", "zmax", "m_thr", "m_x", "m_y", "m_zmin", "m_zmax", "m_floor")}
    for c, cav in enumerate(inp.cavs):
        x = cav.cls.reshape(-1).astype(np.float64)
        d = cav.reg.reshape(-1, 7).astype(np.float64)
        prob = _sigmoid(x)
        passed = prob > THR32
        with np.errstate(over="ignore", invalid="ignore"):
            ad = np.sqrt(an[:, 4] ** 2 + an[:, 5] ** 2)
            b = np.empty_like(d)
            b[:, 0] = d[:, 0] * ad + an[:, 0]
            b[:, 1] = d[:, 1] * ad + an[:, 1]
            b[:, 2] = d[:, 2] * an[:, 3] + an[:, 2]
            b[:, 3:6] = np.exp(d[:, 3:6]) * an[:, 3:6]
            b[:, 6] = d[:, 6] + an[:, 6]
            eb0 = 4 * U * np.abs(d[:, 0] * ad) + U * np.abs(b[:, 0])
            eb1 = 4 * U * np.abs(d[:, 1] * ad) + U * np.abs(b[:, 1])
            eb2 = 2 * U * np.abs(d[:, 2] * an[:, 3]) + U * np.abs(b[:, 2])
            edim = 5 * U * np.abs(b[:, 3:6])
            yaw = b[:, 6].copy()
            eyaw = U * np.abs(b[:, 6])
            lab = np.zeros(n1, dtype=np.int64)
            wrapped = np.zeros(n1, dtype=bool)
            m_floor = np.full(n1, np.inf)
            if inp.bins:
                bins = inp.bins
                dl = cav.dir.reshape(-1, bins).astype(np.float64)
                best = dl[:, 0].copy()
                for q in range(1, bins):            # first largest bin wins; a NaN never replaces the running best
                    m = dl[:, q] > best
                    lab[m] = q
                    best = np.where(m, dl[:, q], best)
                off = 0.0 if "dir_offset_dropped" in bug else float(inp.dir_offset)
                period = TWO_PI / bins
                v = b[:, 6] - off
                k = np.floor(v / period)
                rot = v - k * period
                lab_used = lab + 1 if "period_off_by_one_bin" in bug else lab
                y2 = rot + off + period * lab_used
                m2 = np.floor(y2 / TWO_PI + 0.5)
                yaw = y2 - m2 * TWO_PI
                wrapped = m2 != 0
                eyaw = U * (2 * np.abs(b[:, 6]) + 2 * np.abs(v) + 3 * np.abs(k) * period + 2 * np.abs(rot) + 2 * abs(off)
                            + 3 * period * lab + 2 * np.abs(y2) + 3 * TWO_PI * np.abs(m2) + np.abs(yaw))
                frac = v / period - k
                m_floor = np.minimum(frac, 1.0 - frac) / (8 * U * (np.abs(v) / period + 1.0))
            if inp.order == "hwl":
                dx, dy, dz, edx, edy, edz = b[:, 5], b[:, 4], b[:, 3], edim[:, 2], edim[:, 1], edim[:, 0]
            else:
                dx, dy, dz, edx, edy, edz = b[:, 3], b[:, 4], b[:, 5], edim[:, 0], edim[:, 1], edim[:, 2]
            if "l_w_swapped" in bug:
                dx, dy, edx, edy = dy, dx, edy, edx
            ca, sa = np.cos(yaw)[:, None], np.sin(yaw)[:, None]
            eca = eyaw[:, None] + 4 * U * np.abs(ca)
            esa = eyaw[:, None] + 4 * U * np.abs(sa)
            lx, ly, lz = dx[:, None] * SX * 0.5, dy[:, None] * SY * 0.5, dz[:, None] * SZ * 0.5
            elx, ely, elz = 0.5 * edx[:, None], 0.5 * edy[:, None], 0.5 * edz[:, None]
            xx = lx * ca - ly * sa + b[:, 0:1]
            yy = lx * sa + ly * ca + b[:, 1:2]
            zz = lz + b[:, 2:3]
            ex = (np.abs(lx) * eca + np.abs(ly) * esa + elx * np.abs(ca) + ely * np.abs(sa) + eb0[:, None]
                  + 2 * U * (np.abs(lx * ca) + np.abs(ly * sa) + np.abs(b[:, 0:1])))
            ey = (np.abs(lx) * esa + np.abs(ly) * eca + elx * np.abs(sa) + ely * np.abs(ca) + eb1[:, None]
                  + 2 * U * (np.abs(lx * sa) + np.abs(ly * ca) + np.abs(b[:, 1:2])))
            ez = elz + eb2[:, None] + U * (np.abs(lz) + np.abs(b[:, 2:3]))
            T = cav.T.astype(np.float64)
            P = [xx, yy, zz]
            E = [ex, ey, ez]
            corners = np.stack([T[r, 0] * xx + T[r, 1] * yy + T[r, 2] * zz + T[r, 3] for r in range(3)], axis=-1)
            bound = np.stack([sum(abs(T[r, i]) * E[i] for i in range(3))
                              + 4 * U * (sum(np.abs(T[r, i] * P[i]) for i in range(3)) + abs(T[r, 3])) for r in range(3)], axis=-1)
            xl = corners[:, :, 0].max(1) - corners[:, :, 0].min(1)
            yl = corners[:, :, 1].max(1) - corners[:, :, 1].min(1)
            zmin, zmax = corners[:, :, 2].min(1), corners[:, :, 2].max(1)
            keep = passed & (xl <= 6) & (yl <= 6) & (yl != 0) & (zmin >= -3) & (zmax <= 1)
            score = prob.copy()
            srel = np.full(n1, SCORE_REL)
            iou_l = None
            if cav.iou is not None:
                iou_l = cav.iou.reshape(-1).astype(np.float64)
                q = np.fmin(np.fmax(_sigmoid(iou_l), 0.0), 1.0)     # fmaxf(NaN, 0) = 0: a NaN IoU logit counts as 0
                score = prob * ((q + 1.0) * 0.5) ** 4
                srel[:] = SCORE_REL_IOU
            finite = np.isfinite(corners).all(axis=(1, 2))
            bx = 2 * bound[:, :, 0].max(1)
            by = 2 * bound[:, :, 1].max(1)
            bz = bound[:, :, 2].max(1)
            acc["m_thr"].append(np.abs(prob - THR32) / (SCORE_REL * prob + 1e-300))
            acc["m_x"].append(np.abs(xl - 6) / bx)
            acc["m_y"].append(np.minimum(np.abs(yl - 6), np.abs(yl)) / by)
            acc["m_zmin"].append(np.abs(zmin + 3) / bz)
            acc["m_zmax"].append(np.abs(zmax - 1) / bz)
        acc["m_floor"].append(m_floor)
        acc["slot"].append(c * n1 + np.arange(n1))
        acc["logit"].append(x)
        acc["iou"].append(iou_l if iou_l is not None else np.full(n1, np.nan))
        acc["prob"].append(prob)
        acc["passed"].append(passed)
        acc["keep"].append(keep)
        acc["score"].append(score)
        acc["sb"].append(srel * score)
        acc["corners"].append(corners)
        acc["bound"].append(bound)
        acc["wrapped"].append(wrapped)
        acc["lab"].append(lab)
        acc["finite"].append(finite)
        acc["xl"].append(xl)
        acc["yl"].append(yl)
        acc["zmin"].append(zmin)
        acc["zmax"].append(zmax)
    cat = {k: np.concatenate(v) for k, v in acc.items()}
    has_iou = inp.cavs[0].iou is not None
    return Ref(slot=cat["slot"], logit=cat["logit"], iou_logit=cat["iou"] if has_iou else None, prob=cat["prob"],
               passed=cat["passed"], keep=cat["keep"], score=cat["score"], score_bound=cat["sb"], corners=cat["corners"],
               bound=cat["bound"], margins={k[2:]: cat[k] for k in cat if k.startswith("m_")}, wrapped=cat["wrapped"],
               lab=cat["lab"], finite=cat["finite"], x_len=cat["xl"], y_len=cat["yl"], z_min=cat["zmin"], z_max=cat["zmax"])


def _kernel_key(R: Ref, idx):
    """the fp32 score the kernel sorts by, where it is decided exactly: the fp32 rounding of the float64 score, except that the
    kernel's 1 / (1 + expf(-x)) is exactly 1.0f for x >= 17 (1 + expf(-x) rounds to 1), where the rounding of the true
    sigmoid would still give the fp32 value below 1 up to x = 17.3"""
    key = R.score[idx].astype(np.float32).astype(np.float64)
    if R.iou_logit is None:
        key[R.logit[idx] >= 17] = 1.0
    return key


def expected_order(R: Ref, top: int, bug=()) -> np.ndarray:
    """Candidates the kernel emits after the filters, in its pinned order: descending score, then ascending slot.  Equal keys
    are identical logits or sigmoids that round to 1.0f (_decode_census checks that no other pair comes close)."""
    cand = R.keep if "top_cut_before_filter" not in bug else R.passed
    idx = np.flatnonzero(cand)
    key = _kernel_key(R, idx)
    slot = -R.slot[idx] if "ties_reversed" in bug else R.slot[idx]
    o = idx[np.lexsort((slot, -key))][:top]
    if "top_cut_before_filter" in bug:
        o = o[R.keep[o]]
    return o


# ---------------------------------------------------------------------------------------------------------------------------
# float64 reference of the rotated NMS and of the range mask
# ---------------------------------------------------------------------------------------------------------------------------
def _area2(q):
    return sum(q[k][0] * q[(k + 1) % len(q)][1] - q[k][1] * q[(k + 1) % len(q)][0] for k in range(len(q)))


def _clip_area(P, Q):
    """Sutherland-Hodgman: the part of quad P on the left of each directed edge of quad Q (both counter-clockwise)."""
    poly = P
    for e in range(4):
        qx, qy = Q[e]
        ex, ey = Q[(e + 1) % 4][0] - qx, Q[(e + 1) % 4][1] - qy
        out = []
        n = len(poly)
        for k in range(n):
            ax, ay = poly[k]
            bx, by = poly[(k + 1) % n]
            sp = ex * (ay - qy) - ey * (ax - qx)
            sq = ex * (by - qy) - ey * (bx - qx)
            if sp >= 0.0:
                out.append((ax, ay))
            if (sp > 0.0 and sq < 0.0) or (sp < 0.0 and sq > 0.0):
                t = sp / (sp - sq)
                out.append((ax + t * (bx - ax), ay + t * (by - ay)))
        poly = out
        if len(poly) < 3:
            return 0.0
    return abs(0.5 * _area2(poly))


@dataclass
class NmsRun:
    pick: np.ndarray
    clipped: int                          # pairs that passed the bounding-box test and were clipped
    suppressed: int                       # pairs with IoU above the threshold
    nearest: float                        # least |IoU - thr| over the clipped pairs
    word_crossing_chains: int             # picks i that survive only because their suppressor j was itself removed, with
                                          # i and j (or j and its own suppressor) in different 64-bit words
    clockwise: int                        # quads that needed the reversal


def ref_nms(corners: np.ndarray, thr: float, bug=()) -> NmsRun:
    """nms_rotated (box_utils.py:693-738) on the corners in the given (score) order: greedy, IoU of the float64 polygons cast to
    fp32, suppressed when > fp32(thr).  A zero-area union gives NaN, which never suppresses."""
    c = np.asarray(corners, dtype=np.float64)
    n = len(c)
    thr32 = np.float32(thr)
    quads, areas = [], np.empty(n)
    cw = 0
    for i in range(n):
        q = [(c[i, k, 0], c[i, k, 1]) for k in range(4)]
        a2 = _area2(q)
        if a2 < 0:
            cw += 1
            if "no_ccw_reversal" not in bug:
                q = q[::-1]
        quads.append(q)
        areas[i] = abs(0.5 * a2)
    lo = c[:, :4, :2].min(axis=1)
    hi = c[:, :4, :2].max(axis=1)
    removed = np.zeros(n, dtype=bool)
    by = np.full(n, -1)
    pick, clipped, suppressed, nearest = [], 0, 0, math.inf
    for i in range(n):
        if removed[i] and "suppressor_state_ignored" not in bug:
            continue
        if not removed[i]:
            pick.append(i)
        js = np.arange(i + 1, n)
        js = js[~((hi[i, 0] < lo[js, 0]) | (hi[js, 0] < lo[i, 0]) | (hi[i, 1] < lo[js, 1]) | (hi[js, 1] < lo[i, 1]))]
        for j in js:
            inter = _clip_area(quads[i], quads[j])
            uni = areas[i] + areas[j] - inter
            iou = inter / uni if uni != 0.0 else math.nan
            clipped += 1
            if not math.isnan(iou):
                nearest = min(nearest, abs(iou - thr))
            iou32 = np.float32(iou)
            if (iou32 >= thr32) if "iou_ge" in bug else (iou32 > thr32):
                suppressed += 1
                if not removed[j]:
                    removed[j] = True
                    by[j] = i
    pick = np.array(pick, dtype=np.int64)
    chains = 0
    for i in pick:          # i overlaps a higher box j above the threshold, but j was removed by k first
        for j in range(i):
            if by[j] >= 0 and (j // 64 != i // 64 or by[j] // 64 != j // 64) and _iou32(quads, areas, j, i) > thr32:
                chains += 1
                break
    return NmsRun(pick, clipped, suppressed, nearest, chains, cw)


def _iou32(quads, areas, i, j):
    inter = _clip_area(quads[i], quads[j])
    uni = areas[i] + areas[j] - inter
    return np.float32(inter / uni if uni != 0.0 else math.nan)


def range_keep(corners: np.ndarray, gt_range, bug=()) -> np.ndarray:
    """mask_boxes_outside_range_numpy: fp32 corners against the float64 range (box_utils.py:415-416)."""
    lim = np.array(gt_range, dtype=np.float32 if "f32_range_limits" in bug else np.float64)
    c = np.asarray(corners)
    return ((c >= lim[0:3]) & (c <= lim[3:6])).all(axis=2).sum(axis=1) >= 8


# ---------------------------------------------------------------------------------------------------------------------------
# cases: generated decode maps
# ---------------------------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class DCase:
    name: str
    H: int
    W: int
    A: int
    bins: int = 2
    order: str = "hwl"
    dir_offset: float = DIR_OFFSET
    n_cav: int = 1
    path: str = "single"                  # single | multi | late
    iou: bool = False
    views: bool = False                   # heads as channel views of one fused cls|reg|dir(|iou) buffer
    ties: bool = False                    # tie groups of identical logits (across cavs where there are several)
    saturated: bool = False               # logits >= 17 and +inf: sigmoids equal to 1.0f
    argmax_ties: bool = False             # equal direction logits
    nonfinite: bool = False
    tilt: bool = False                    # a transform with roll
    seed: int = 0


DCASE_LIST = [
    DCase("hwl_bins2_A2", 13, 17, 2, seed=1, tilt=True),
    DCase("lhw_bins4_A3_argmax_ties", 9, 11, 3, bins=4, order="lhw", argmax_ties=True, seed=2),
    DCase("hwl_bins1_A1_offset0", 20, 30, 1, bins=1, dir_offset=0.0, seed=3),
    DCase("nodir_A2_views_saturated", 11, 23, 2, bins=0, views=True, saturated=True, seed=4),
    DCase("multi2_iou_views", 10, 13, 2, n_cav=2, path="multi", iou=True, views=True, ties=True, seed=5),
    DCase("late3_views_ties", 7, 19, 3, n_cav=3, path="late", views=True, ties=True, saturated=True, seed=6),
    DCase("multi1_iou_nonfinite", 12, 12, 2, path="multi", iou=True, nonfinite=True, seed=7),
    DCase("late2_bins4_nonfinite", 8, 11, 2, bins=4, n_cav=2, path="late", nonfinite=True, seed=8),
]
DCASES = {c.name: c for c in DCASE_LIST}


def _grid_anchors(H, W, A, order):
    ys, xs = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    an = np.zeros((H, W, A, 7))
    an[..., 0] = ((xs - W / 2) * 0.8)[..., None]
    an[..., 1] = ((ys - H / 2) * 0.8)[..., None]
    an[..., 2] = -1.0
    an[..., 3:6] = (1.56, 1.6, 3.9) if order == "hwl" else (3.9, 1.56, 1.6)
    an[..., 6] = np.arange(A) * (math.pi / A)
    return an.astype(np.float32)


def _decode_inputs(case: DCase) -> Inputs:
    rng = np.random.default_rng(case.seed)
    H, W, A = case.H, case.W, case.A
    n1 = H * W * A
    N = n1 * case.n_cav
    an = _grid_anchors(H, W, A, case.order)
    a64 = an.reshape(-1, 7).astype(np.float64)
    ad = np.sqrt(a64[:, 4] ** 2 + a64[:, 5] ** 2)
    z_dim = a64[:, 3]                                          # delta 2 scales with anchor column 3
    # logits: a shuffled lattice on [logit(thr) - 2, logit(thr) + 6], every point half a step away from logit(thr)
    step = 8.0 / N
    lat = LOGIT_THR + (np.arange(N) - N // 4 + 0.5) * step
    logits = rng.permutation(lat)
    cavs = []
    for c in range(case.n_cav):
        a_idx = np.arange(n1) % A
        d = np.zeros((n1, 7))
        d[:, 0] = ((a_idx - (A - 1) / 2) * 0.2 + rng.uniform(-0.03, 0.03, n1)) / ad
        d[:, 1] = rng.uniform(-0.03, 0.03, n1) / ad
        d[:, 2] = rng.uniform(-1.6, 1.2, n1) * 1.56 / z_dim
        d[:, 3:6] = rng.uniform(-0.4, 0.55, (n1, 3))
        d[:, 6] = rng.uniform(-math.pi, math.pi, n1)
        dirl = rng.normal(0, 1.5, (n1, case.bins)) if case.bins else None
        if dirl is not None and case.argmax_ties:
            t = rng.choice(n1, n1 // 4, replace=False)
            src = rng.integers(0, case.bins, len(t))
            dst = (src + rng.integers(1, case.bins, len(t))) % case.bins
            m = dirl[t].max(axis=1) + 0.5
            dirl[t, src] = m
            dirl[t, dst] = m
        iou = rng.normal(0, 2, n1) if case.iou else None
        T = _rz(0.3 + 1.1 * c, 60.0 * c + 3.3, 7.0 * c - 2.1, 0.05, tilt=0.01 if (case.tilt and c == 0) else 0.0)
        cavs.append(Cav(cls=logits[c * n1:(c + 1) * n1].reshape(H, W, A).astype(np.float32),
                        reg=d.reshape(H, W, 7 * A).astype(np.float32),
                        dir=None if dirl is None else dirl.reshape(H, W, A * case.bins).astype(np.float32),
                        iou=None if iou is None else iou.reshape(H, W, A).astype(np.float32), T=T))
    inp = Inputs(anchors=an, cavs=cavs, bins=case.bins, order=case.order, dir_offset=float(np.float32(case.dir_offset)),
                 special=np.zeros(N, dtype=bool), exact=np.zeros(N, dtype=bool))
    _fix_margins(inp)
    _plant(case, inp, rng)
    _fix_margins(inp)
    return inp


def _set(inp: Inputs, name: str, slot: int, k, value):
    """inp.cavs[cav].<name> at global slot, channel k of the anchor (reg: delta k, dir: bin k)."""
    c, i = divmod(int(slot), inp.n1)
    arr = getattr(inp.cavs[c], name)
    per = arr.shape[-1] // inp.shape[2]
    flat = arr.reshape(-1, per)
    flat[i, k] = value


def _get(inp: Inputs, name: str, slot: int, k=0):
    c, i = divmod(int(slot), inp.n1)
    arr = getattr(inp.cavs[c], name)
    return arr.reshape(-1, arr.shape[-1] // inp.shape[2])[i, k]


def _plant(case: DCase, inp: Inputs, rng):
    R = ref_decode(inp)
    kept = np.flatnonzero(R.keep)
    rng.shuffle(kept)
    pos = 0

    def take(k):
        nonlocal pos
        out = kept[pos:pos + k]
        pos += k
        return out

    if case.ties:                                   # groups of identical (cls, iou) logits; with several cavs, across cavs
        for g in range(6):
            members = take(3)
            if len(inp.cavs) > 1:
                members = np.array([m % inp.n1 + (q % len(inp.cavs)) * inp.n1 for q, m in enumerate(members)])
                members = np.array([m for m in members if R.keep[m]], dtype=np.int64)
            for m in members[1:]:
                _set(inp, "cls", m, 0, _get(inp, "cls", members[0]))
                if inp.cavs[0].iou is not None:
                    _set(inp, "iou", m, 0, _get(inp, "iou", members[0]))
            inp.special[members] = True
    if case.saturated:                              # sigmoid rounds to 1.0f: a tie whatever the logit
        for m, v in zip(take(5), (17.0, 19.5, 24.0, 88.0, np.inf)):
            _set(inp, "cls", m, 0, v)
            inp.special[m] = True
    if case.nonfinite:
        for m, v in zip(take(3), (np.nan, -np.inf, np.inf)):
            _set(inp, "cls", m, 0, v)
            inp.special[m] = True
        for k in range(7):                          # a NaN in each delta, an inf and a -inf in some
            for v in (np.nan, np.inf, -np.inf) if k in (0, 3, 5, 6) else (np.nan,):
                m = take(1)[0]
                _set(inp, "reg", m, k, v)
                inp.special[m] = True
        if inp.bins:
            for q in (0, 1):
                m = take(1)[0]
                _set(inp, "dir", m, q, np.nan)
                inp.special[m] = True
        if inp.cavs[0].iou is not None:
            for v in (np.nan, np.inf, -np.inf):
                m = take(1)[0]
                _set(inp, "iou", m, 0, v)
                inp.special[m] = True


def _fix_margins(inp: Inputs, rounds: int = 60):
    """Move generated candidates (not the planted ones) until every decision is MARGIN x its bound from its edge and adjacent
    scores of different candidates are MARGIN x the sum of their bounds apart."""
    for _ in range(rounds):
        R = ref_decode(inp)
        bad = _margin_violations(inp, R)
        near = _near_scores(inp, R)
        if not len(bad) and not len(near):
            return
        for s, what in bad:
            if what == "thr":
                _set(inp, "cls", s, 0, np.float32(_get(inp, "cls", s) + 0.05 * np.sign(_get(inp, "cls", s) - LOGIT_THR)))
            elif what in ("x", "y"):
                for k in (3, 4, 5):
                    _set(inp, "reg", s, k, np.float32(_get(inp, "reg", s, k) - 0.01))
            elif what in ("zmin", "zmax"):
                _set(inp, "reg", s, 2, np.float32(_get(inp, "reg", s, 2) + (0.01 if what == "zmin" else -0.01)))
            elif what == "floor":
                _set(inp, "reg", s, 6, np.float32(_get(inp, "reg", s, 6) + 0.003))
        for s in near:
            _set(inp, "cls", s, 0, np.float32(_get(inp, "cls", s) + 1e-3))
    raise AssertionError("margins could not be established")


def _margin_violations(inp: Inputs, R: Ref):
    out = []
    gen = ~inp.special & ~inp.exact
    for s in np.flatnonzero(gen):
        if R.margins["thr"][s] <= MARGIN:
            out.append((s, "thr"))
        elif R.passed[s]:
            for what in ("x", "y", "zmin", "zmax", "floor"):
                if R.margins[what][s] <= MARGIN:
                    out.append((s, what))
                    break
    return out


def _equal_by_design(inp: Inputs, R: Ref, i, j):
    same_iou = R.iou_logit is None or (R.iou_logit[i] == R.iou_logit[j])
    return (R.logit[i] == R.logit[j] and same_iou) or (R.iou_logit is None and R.logit[i] >= 17 and R.logit[j] >= 17)


def _near_scores(inp: Inputs, R: Ref):
    """lower member of each adjacent pair of surviving candidates whose scores are too close for their bounds, unless the
    two are equal by design; the generated member is the one moved."""
    idx = np.flatnonzero(R.keep)
    o = idx[np.argsort(-R.score[idx], kind="stable")]
    out = []
    for i, j in zip(o[:-1], o[1:]):
        if _equal_by_design(inp, R, i, j):
            continue
        if abs(R.score[i] - R.score[j]) <= MARGIN * (R.score_bound[i] + R.score_bound[j]):
            if not inp.special[j]:
                out.append(j)
            elif not inp.special[i]:
                out.append(i)
            else:
                raise AssertionError(f"planted candidates {i} and {j} have near scores")
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# cases: boxes given directly (anchors = boxes, zero deltas, no direction head)
# ---------------------------------------------------------------------------------------------------------------------------
def _box_inputs(boxes, logits, Ts, W: int = 64, exact: bool = True, rng=None) -> Tuple[Inputs, np.ndarray]:
    """boxes (n1, 7) [x y z h w l yaw] shared by every cav (anchor i of cav c is boxes[i] moved by Ts[c]); logits (n_cav, n1).
    The anchors are laid out on an H x W x 1 grid, padded with candidates below the threshold.  Returns the inputs and the
    slot of each box (the boxes go to shuffled slots when `rng` is given)."""
    boxes = np.asarray(boxes, dtype=np.float64)
    logits = np.atleast_2d(np.asarray(logits, dtype=np.float64))
    n = len(boxes)
    H = max(1, -(-n // W))
    n1 = H * W
    at = np.arange(n) if rng is None else rng.permutation(n1)[:n]
    an = np.zeros((n1, 7))
    an[:, 0] = 5000.0 + np.arange(n1)                   # padding: far away, never above the threshold
    an[:, 2:6] = (-1.0, 1.0, 1.0, 1.0)
    an[at] = boxes
    an32 = an.astype(np.float32)
    if exact:
        assert np.array_equal(an32.astype(np.float64), an), "box values must be fp32-exact"
    cavs = []
    for c, T in enumerate(Ts):
        lg = np.full(n1, -30.0)
        lg[at] = logits[c]
        cavs.append(Cav(cls=lg.reshape(H, W, 1).astype(np.float32), reg=np.zeros((H, W, 7), np.float32), dir=None, iou=None,
                        T=np.asarray(T, dtype=np.float32)))
    N = n1 * len(Ts)
    inp = Inputs(anchors=an32.reshape(H, W, 1, 7), cavs=cavs, special=np.zeros(N, bool), exact=np.full(N, exact))
    return inp, at


def _box(x, y, l=2.0, w=1.5, yaw=0.0, z=-1.0, h=1.5):
    return (x, y, z, h, w, l, yaw)


def _rank_logits(n):
    """distinct logits, highest first, all above the threshold and below saturation"""
    return np.linspace(6.0, -1.0, n) if n > 1 else np.array([3.0])


# exact edge cases of the size / z filters
EDGE_BOXES = [
    # (box, kept?)
    (_box(0.5, 0.0, l=6.0, w=2.0), True),                          # x_len exactly 6
    (_box(0.5, 4.0, l=6.0 + 2 ** -20, w=2.0), False),              # one step above 6
    (_box(0.5, 8.0, l=2.0, w=6.0), True),                          # y_len exactly 6
    (_box(40.0, 0.5, l=2.0, w=6.0 + 2 ** -20), False),
    (_box(0.5, 24.0, l=2.0, w=0.0), False),                        # y_len == 0
    (_box(0.5, 28.0, l=0.0, w=2.0), True),                         # x_len == 0: zero area, kept
    (_box(0.5, 32.0, z=-2.0, h=2.0), True),                        # z_min exactly -3
    (_box(0.5, 36.0, z=-2.0 - 2 ** -20, h=2.0), False),
    (_box(0.5, 40.0, z=0.0, h=2.0), True),                         # z_max exactly 1
    (_box(0.5, 44.0, z=2 ** -20, h=2.0), False),
    (_box(0.5, 48.0, l=2.0, w=2.0), True),
]


def _edge_inputs():
    boxes = [b for b, _ in EDGE_BOXES]
    return _box_inputs(boxes, [_rank_logits(len(boxes))], [np.eye(4)], W=5, rng=np.random.default_rng(11))


# sort / top cut
SORT_TOPS = [1, 63, 64, 65, 128, 1000, 1320]


def _sort_inputs(top: int, delta: int, n_cav: int = 1):
    """top + delta candidates that pass the filters (over n_cav cavs), a tie group of 4 straddling the cut when there are
    enough, 9 high-scored candidates the size filter drops, and padding below the threshold."""
    rng = np.random.default_rng(1000 + 7 * top + delta + 31 * n_cav)
    n_pass = top + delta
    n_drop = 9
    per = -(-n_pass // n_cav)
    boxes = [_box(8.0 * (i % 48), 8.0 * (i // 48), l=8.0 if i >= per else 2.0, w=1.5) for i in range(per + n_drop)]
    pass_pairs = [(c, i) for i in range(per) for c in range(n_cav)]
    rng.shuffle(pass_pairs)
    pass_pairs = pass_pairs[:n_pass]
    drop_pairs = [(k % n_cav, per + k) for k in range(n_drop)]          # x_len 8 > 6: dropped by the size filter
    drop_ranks = set(rng.choice(n_pass + n_drop, n_drop, replace=False).tolist())
    lg = _rank_logits(n_pass + n_drop)
    logits = np.full((n_cav, per + n_drop), -30.0)
    tie_at = [r for r in range(top - 2, top + 2) if 0 <= r < n_pass] if n_pass > top else []
    tie_logit = None
    r_pass = r_drop = 0
    for r in range(n_pass + n_drop):
        if r in drop_ranks:
            c, i = drop_pairs[r_drop]
            r_drop += 1
            logits[c, i] = lg[r]
            continue
        c, i = pass_pairs[r_pass]
        logits[c, i] = lg[r]
        if r_pass in tie_at:                                             # a tie group across the cut
            tie_logit = lg[r] if tie_logit is None else tie_logit
            logits[c, i] = tie_logit
        r_pass += 1
    Ts = [np.array([[1, 0, 0, 2048.0 * c], [0, 1, 0, 0], [0, 0, 1, 0], [0, 0, 0, 1]]) for c in range(n_cav)]
    inp, _ = _box_inputs(boxes, logits, Ts, W=48)
    return inp, len(tie_at)


SORT_CASES = ([("single", t, d) for t in SORT_TOPS for d in (-1, 0, 1)]
              + [("multi", 64, 1), ("multi", 1000, 0), ("late", 65, 1), ("late", 1320, -1)])


# NMS
@dataclass(frozen=True)
class NCase:
    name: str
    n: int
    thr: float = 0.15
    kind: str = "clusters"                # clusters | exact | identical | disjoint
    T: str = "rot"                        # rot | identity | reflect
    chain_ranks: Tuple[int, ...] = ()
    seed: int = 0


NCASE_LIST = [
    NCase("n63", 63, seed=1),
    NCase("n64", 64, seed=2),
    NCase("n65_chain", 65, chain_ranks=(62, 63, 64), seed=3),
    NCase("n127", 127, seed=4),
    NCase("n128", 128, seed=5),
    NCase("n129_chain", 129, chain_ranks=(63, 64, 128), seed=6),
    NCase("n1320_chains", 1320, chain_ranks=(60, 70, 130, 700, 704, 1280), seed=7),
    NCase("n300_clockwise", 300, T="reflect", seed=8),
    NCase("exact_pairs", 0, kind="exact", T="identity"),
    NCase("exact_thr_0.5", 0, thr=0.5, kind="exact", T="identity"),
    NCase("exact_thr_0.25", 0, thr=0.25, kind="exact", T="identity"),
    NCase("identical_1320", 1320, kind="identical", T="identity"),
    NCase("disjoint_1320", 1320, kind="disjoint", T="identity"),
]
NCASES = {c.name: c for c in NCASE_LIST}


def _exact_pairs(thr):
    """dyadic boxes in rank order; every group 16 m from the next"""
    out = []
    def at(k, b):
        return (b[0] + 16.0 * k,) + tuple(b[1:])
    if thr == 0.15:
        groups = [
            [_box(1, 1, 2, 2), _box(1, 1, 2, 2)],                              # identical: IoU 1
            [_box(1, 1, 2, 2), _box(1, 0.5, 1, 1)],                            # nested, IoU 1/4: suppressed
            [_box(1, 1, 4, 4), _box(1, 1, 1, 1)],                              # nested, IoU 1/16: kept
            [_box(1, 1, 2, 2), _box(3, 1, 2, 2)],                              # shared edge: IoU 0
            [_box(1, 1, 2, 2), _box(3, 3, 2, 2)],                              # shared vertex: IoU 0
            [_box(1, 1, 0, 2), _box(1, 1.5, 0, 2)],                            # two collinear zero-area boxes: NaN
            [_box(1, 1, 2, 2), _box(1, 1, 0, 1)],                              # a zero-area box inside a box: IoU 0
            [_box(1, 1, 0, 2), _box(1, 1, 2, 2)],                              # the same, zero-area box first
        ]
    else:
        e = 2.0 ** -23
        if thr == 0.5:
            groups = [[_box(1, 1, 2, 2), _box(1, 0.5, 2, 1)],                  # IoU exactly 0.5: kept
                      [_box(1, 1, 2, 2), _box(1, 0.5 + e / 2, 2, 1 + e)]]      # one fp32 ulp above: suppressed
        else:
            groups = [[_box(1, 1, 2, 2), _box(1, 1, 1, 1)],                    # IoU exactly 0.25
                      [_box(1, 1, 2, 2), _box(1, 0.5 + e / 2, 1, 1 + e)]]      # 0.25 + one ulp
    for k, g in enumerate(groups):
        out += [at(k, b) for b in g]
    return out


def _chain(x0, y0):
    """A > B > C along x: IoU(A, B) = IoU(B, C) = 1/3, IoU(A, C) = 0 -- C survives because B was removed"""
    return [_box(x0, y0, 4, 2), _box(x0 + 2, y0, 4, 2), _box(x0 + 4, y0, 4, 2)]


def _nms_inputs(case: NCase):
    rng = np.random.default_rng(case.seed)
    if case.kind == "exact":
        boxes = _exact_pairs(case.thr)
    elif case.kind == "identical":
        boxes = [_box(3.0, 2.0, 4.0, 2.0, 0.5)] * case.n
    elif case.kind == "disjoint":
        boxes = [_box(8.0 * (i % 40), 8.0 * (i // 40), 4.0, 2.0, 0.25 * (i % 7)) for i in range(case.n)]
    else:
        boxes = [None] * case.n
        spots = [(12.0 * (s % 40), 12.0 * (s // 40)) for s in range(case.n + 8)]
        spots = [spots[i] for i in rng.permutation(len(spots))]
        ranks = list(range(case.n))
        for k in range(0, len(case.chain_ranks), 3):            # each chain on a spot of its own
            x0, y0 = spots.pop()
            for r, b in zip(case.chain_ranks[k:k + 3], _chain(x0, y0)):
                boxes[r] = b
                ranks.remove(r)
        rng.shuffle(ranks)
        while ranks:                                           # clusters of 1 to 4 boxes around a spot
            x0, y0 = spots.pop()
            m = min(len(ranks), int(rng.integers(1, 5)))
            for _ in range(m):
                r = ranks.pop()
                boxes[r] = _box(x0 + rng.uniform(-1.2, 1.2), y0 + rng.uniform(-1.2, 1.2), rng.uniform(3.0, 5.0),
                                rng.uniform(1.5, 2.2), rng.uniform(-math.pi, math.pi))
    T = {"identity": np.eye(4), "rot": _rz(0.7, 3.0, -4.0), "reflect": np.diag([1.0, -1.0, 1.0, 1.0]) @ _rz(0.4, 1.0, 2.0)}[case.T]
    exact = case.kind != "clusters"
    if not exact:
        boxes = [tuple(float(np.float32(v)) for v in b) for b in boxes]
    inp, _ = _box_inputs(boxes, [_rank_logits(len(boxes))], [T], W=64, exact=True, rng=rng)
    return inp


# range mask
RANGES = {"r25.6": [-25.6, -25.6, -3.0, 25.6, 25.6, 1.0], "r102.4": [-102.4, -102.4, -3.0, 102.4, 102.4, 1.0],
          "r140.8": [-140.8, -40.0, -3.0, 140.8, 40.0, 1.0]}


def _neighbours(v):
    f = np.float32(v)
    return [np.nextafter(f, np.float32(-np.inf)), f, np.nextafter(f, np.float32(np.inf))]


def _range_inputs(name):
    """boxes with one corner coordinate at fp32(limit) and at its two fp32 neighbours, for each of the six limits; interior
    boxes; and an out-of-range box that suppresses an in-range one (NMS runs before the mask)."""
    lim = RANGES[name]
    boxes = []
    hx = 1.0                                                    # half size of every box on every axis
    for k in range(6):
        axis, upper = k % 3, k >= 3
        for j, t in enumerate(_neighbours(lim[k])):
            t = float(t)
            centre = t - hx if upper else t + hx
            if axis == 0:
                b = _box(centre, -12.0 + 3.0 * j + 9.0 * upper, l=2.0, w=2.0)
            elif axis == 1:
                b = _box(-12.0 + 3.0 * j + 9.0 * upper, centre, l=2.0, w=2.0)
            else:
                b = _box(-12.0 + 3.0 * j + 9.0 * upper, 3.0 * k - 12.0, z=centre, h=2.0)
            edge = (b[axis] + (hx if upper else -hx)) if axis < 2 else (b[2] + (1.0 if upper else -1.0))
            assert edge == t and np.float32(b[axis if axis < 2 else 2]) == b[axis if axis < 2 else 2], (name, k, j)
            boxes.append(b)
    boxes += [_box(-4.0 + 3.0 * i, 15.0, l=2.0, w=2.0) for i in range(4)]
    x_hi = float(np.float32(lim[3]))
    boxes.insert(0, _box(x_hi - 0.5, 20.0, l=2.0, w=2.0))         # pokes 0.5 m out of range, highest score
    boxes.insert(1, _box(x_hi - 1.5, 20.0, l=2.0, w=2.0))         # inside, IoU 1/3 with it: suppressed
    inp, _ = _box_inputs(boxes, [_rank_logits(len(boxes))], [np.eye(4)], W=16, rng=np.random.default_rng(5))
    return inp


# ---------------------------------------------------------------------------------------------------------------------------
# GPU runner
# ---------------------------------------------------------------------------------------------------------------------------
def _gpu(inp: Inputs, path: str, nms: float, top: int, gt_range=None, views: bool = False):
    """Run one entry point; returns (boxes (K, 8, 3), scores (K,), stats (2,)) as numpy."""
    from heal_b200 import ops
    dev = torch.device("cuda")
    H, W, A = inp.shape
    n = len(inp.cavs)
    bins = inp.bins
    has_iou = inp.cavs[0].iou is not None
    parts = [("cls", A), ("reg", 7 * A)] + ([("dir", A * bins)] if bins else []) + ([("iou", A)] if has_iou else [])
    anchors = torch.from_numpy(np.ascontiguousarray(inp.anchors)).to(dev)
    offs, chs = {}, dict(parts)
    if views:
        off = 1                                             # channel 0 and the last two are padding, NaN-poisoned
        for name, ch in parts:
            offs[name] = off
            off += ch
        buf = np.full((n, H, W, off + 2), np.nan, dtype=np.float32)
        for name, ch in parts:
            buf[..., offs[name]:offs[name] + ch] = np.stack([getattr(c, name) for c in inp.cavs])
        tb = torch.from_numpy(buf).to(dev)
        heads = {name: [ops.Act(tb[c:c + 1, :, :, offs[name]:offs[name] + ch], "f32") for c in range(n)] for name, ch in parts}
    else:
        tb = None
        batched = {name: torch.from_numpy(np.ascontiguousarray(np.stack([getattr(c, name) for c in inp.cavs]))).to(dev)
                   for name, _ in parts}
        heads = {name: [ops.Act(t[c:c + 1], "f32") for c in range(n)] for name, t in batched.items()}
    kw = dict(dir_offset=inp.dir_offset, num_bins=bins or 2, order=inp.order, gt_range=gt_range, top=top)
    if path == "single":
        assert n == 1 and not has_iou
        out = ops.box_decode_nms(heads["cls"][0], heads["reg"][0], heads["dir"][0] if bins else None, anchors, inp.cavs[0].T,
                                 THR, nms, **kw)
    elif path == "multi":
        cavs = [{"cls": heads["cls"][c], "reg": heads["reg"][c], "dir": heads["dir"][c] if bins else None,
                 "iou": heads["iou"][c] if has_iou else None, "anchors": anchors, "transform": inp.cavs[c].T} for c in range(n)]
        out = ops.box_decode_nms_multi(cavs, THR, nms, **kw)
    else:
        assert not has_iou
        Td = torch.from_numpy(np.stack([c.T for c in inp.cavs]).astype(np.float32)).to(dev)
        if views:
            a = ops.Act(tb, "f32")
            out = ops.box_decode_nms_late(a, a, a if bins else None, anchors, Td, THR, nms,
                                          coffsets=(offs["cls"], offs["reg"], offs.get("dir", 0)), **kw)
        else:
            out = ops.box_decode_nms_late(ops.Act(batched["cls"], "f32"), ops.Act(batched["reg"], "f32"),
                                          ops.Act(batched["dir"], "f32") if bins else None, anchors, Td, THR, nms, **kw)
    torch.cuda.synchronize()
    k = int(out.count.item())
    return out.boxes[:k].cpu().numpy().copy(), out.scores[:k].cpu().numpy().copy(), out.stats.cpu().numpy().copy()


def _gpu_twice(*args, **kwargs):
    a = _gpu(*args, **kwargs)
    b = _gpu(*args, **kwargs)
    for x, y in zip(a, b):
        assert x.tobytes() == y.tobytes(), "a repeated run gave other bits"
    return a


# ---------------------------------------------------------------------------------------------------------------------------
# comparisons (shared by the GPU tests and the bound check)
# ---------------------------------------------------------------------------------------------------------------------------
def _identify(R: Ref, exp: np.ndarray, boxes: np.ndarray) -> np.ndarray:
    """for each output box, the index into `exp` of the candidate with the nearest centre (within MIN_SEP / 4)"""
    from scipy.spatial import cKDTree
    if len(boxes) == 0:
        return np.zeros(0, dtype=np.int64)
    d, j = cKDTree(R.centre[exp]).query(boxes.astype(np.float64).mean(axis=1))
    assert d.max() < MIN_SEP / 4, f"an output box is {d.max():.3g} m from every expected candidate"
    return j


def check_decode(R: Ref, exp: np.ndarray, boxes: np.ndarray, scores: np.ndarray, exact=None):
    """set and order exact; corners and scores within their bounds (exactly equal for exact candidates).  Returns the largest
    err / bound of the corners and of the scores."""
    assert len(boxes) == len(exp), f"{len(boxes)} boxes, expected {len(exp)}"
    j = _identify(R, exp, boxes)
    assert np.array_equal(j, np.arange(len(exp))), f"set / order differs: first mismatch at {np.flatnonzero(j != np.arange(len(exp)))[:5]}"
    err = np.abs(boxes.astype(np.float64) - R.corners[exp])
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = float(np.where(err == 0, 0.0, err / R.bound[exp]).max()) if len(exp) else 0.0
    serr = np.abs(scores.astype(np.float64) - R.score[exp])
    sratio = float((serr / R.score_bound[exp]).max()) if len(exp) else 0.0
    assert ratio <= 1.0, f"corner err / bound {ratio:.3f}"
    assert sratio <= 1.0, f"score err / bound {sratio:.3f}"
    if exact is not None and exact[exp].any():
        ex = exact[exp]
        assert np.array_equal(boxes[ex].astype(np.float64), R.corners[exp][ex]), "exact candidates moved"
    return ratio, sratio


# ---------------------------------------------------------------------------------------------------------------------------
# census: every situation the file claims to reach
# ---------------------------------------------------------------------------------------------------------------------------
def _decode_census(case: DCase, inp: Inputs, R: Ref):
    assert not _margin_violations(inp, R) and not _near_scores(inp, R)
    kept = np.flatnonzero(R.keep)
    assert 0 < len(kept) <= 1320
    from scipy.spatial import cKDTree
    pairs = cKDTree(R.centre[kept][:, :2]).query_pairs(MIN_SEP)
    assert not pairs, f"{len(pairs)} pairs of surviving centres closer than {MIN_SEP} m"
    exp = expected_order(R, 1320)
    key = _kernel_key(R, exp)
    for k in range(len(exp) - 1):                          # equal keys only by design
        if key[k] == key[k + 1]:
            assert _equal_by_design(inp, R, exp[k], exp[k + 1]), (exp[k], exp[k + 1])
    H, W, A = inp.shape
    f = {f"order_{case.order}", f"A{A}", case.path, f"n_cav{len(inp.cavs)}", f"bins{case.bins}" if case.bins else "no_dir"}
    if (H * W * A) % 256:
        f.add("hwa_not_multiple_of_256")
    if case.views:
        f.add("channel_views")
    if case.views and case.path == "late":
        f.add("nonzero_coffset")
    if case.bins and case.dir_offset:
        f.add("dir_offset")
    if R.wrapped[kept].any():
        f.add("yaw_wraps_at_pi")
    if case.iou:
        f.add("iou_rescoring")
    f |= _decision_situations(R)
    if any(key[k] == key[k + 1] for k in range(len(key) - 1)):
        f.add("score_ties")
        slots = R.slot[exp]
        if any(key[k] == key[k + 1] and slots[k] // inp.n1 != slots[k + 1] // inp.n1 for k in range(len(key) - 1)):
            f.add("score_ties_across_cavs")
    if (key == 1.0).sum() > 1:
        f.add("saturated_sigmoid_ties")
    if case.bins:
        for c, cav in enumerate(inp.cavs):
            dl = cav.dir.reshape(-1, case.bins)
            sl = c * inp.n1 + np.arange(inp.n1)
            mx = np.nanmax(np.where(np.isnan(dl), -np.inf, dl), axis=1)
            if ((dl == mx[:, None]).sum(axis=1)[R.keep[sl]] > 1).any():
                f.add("dir_argmax_tie")
            if np.isnan(dl[R.passed[sl], 0]).any():
                f.add("nan_dir_logit_bin0")
            if np.isnan(dl[R.passed[sl], 1:]).any():
                f.add("nan_dir_logit_later_bin")
    lg = R.logit
    for name, m in (("nan_logit", np.isnan(lg)), ("neg_inf_logit", lg == -np.inf), ("pos_inf_logit", lg == np.inf)):
        if m.any():
            f.add(name)
    regs = np.concatenate([c.reg.reshape(-1, 7) for c in inp.cavs])
    for k in range(7):
        if np.isnan(regs[R.passed, k]).any():
            f.add(f"nan_delta{k}")
    if np.isinf(regs[R.passed]).any():
        f.add("inf_delta")
    if R.iou_logit is not None:
        if np.isnan(R.iou_logit[R.keep]).any():
            f.add("nan_iou_logit")
        if np.isinf(R.iou_logit[R.keep]).any():
            f.add("inf_iou_logit")
    return f


def _decision_situations(R: Ref):
    f = set()
    p = R.passed
    if (p & ~R.keep & ((R.x_len > 6) | (R.y_len > 6))).any():
        f.add("dropped_by_size")
    if (p & ~R.keep & ((R.z_min < -3) | (R.z_max > 1))).any():
        f.add("dropped_by_z")
    if (p & ~R.finite & ~R.keep).any():
        f.add("dropped_nonfinite")
    if (p & np.isnan(R.corners).any(axis=(1, 2))).any():
        f.add("nan_corner")
    if (p & (R.y_len == 0)).any():
        f.add("y_len_zero")
    if (R.keep & (R.x_len == 6)).any():
        f.add("x_len_exactly_6")
    if (R.keep & (R.y_len == 6)).any():
        f.add("y_len_exactly_6")
    if (R.keep & (R.z_min == -3)).any():
        f.add("z_min_exactly_-3")
    if (R.keep & (R.z_max == 1)).any():
        f.add("z_max_exactly_1")
    if (R.keep & (R.x_len == 0)).any():
        f.add("zero_area_kept")
    return f


DECODE_SITUATIONS = {
    "order_hwl", "order_lhw", "A1", "A2", "A3", "single", "multi", "late", "n_cav1", "n_cav2", "n_cav3", "bins1", "bins2",
    "bins4", "no_dir", "hwa_not_multiple_of_256", "channel_views", "nonzero_coffset", "dir_offset", "yaw_wraps_at_pi",
    "iou_rescoring", "dropped_by_size", "dropped_by_z", "dropped_nonfinite", "nan_corner", "score_ties", "score_ties_across_cavs",
    "saturated_sigmoid_ties", "dir_argmax_tie", "nan_dir_logit_bin0", "nan_dir_logit_later_bin", "nan_logit", "neg_inf_logit",
    "pos_inf_logit", "inf_delta", "nan_iou_logit", "inf_iou_logit",
} | {f"nan_delta{k}" for k in range(7)}
EDGE_SITUATIONS = {"y_len_zero", "x_len_exactly_6", "y_len_exactly_6", "z_min_exactly_-3", "z_max_exactly_1", "zero_area_kept",
                   "dropped_by_size", "dropped_by_z"}


@pytest.fixture(scope="module")
def decode_inputs():
    return {name: _decode_inputs(c) for name, c in DCASES.items()}


def test_decode_cases_cover_every_situation(decode_inputs):
    found = set()
    for name, case in DCASES.items():
        inp = decode_inputs[name]
        f = _decode_census(case, inp, ref_decode(inp))
        print(f"{name}: {sorted(f)}")
        found |= f
    missing = DECODE_SITUATIONS - found
    assert not missing, missing
    inp, _ = _edge_inputs()
    R = ref_decode(inp)
    c = R.corners[R.passed]
    assert np.array_equal(c.astype(np.float32).astype(np.float64), c), "edge corners must be fp32-exact"
    f = _decision_situations(R)
    assert EDGE_SITUATIONS <= f, EDGE_SITUATIONS - f
    assert [bool(R.keep[s]) for s in _edge_slots()] == [k for _, k in EDGE_BOXES]


def _edge_slots():
    return np.random.default_rng(11).permutation(5 * -(-len(EDGE_BOXES) // 5))[:len(EDGE_BOXES)]


def test_sort_cases_cover_every_situation():
    found = set()
    for path, top, delta in SORT_CASES:
        inp, ties = _sort_inputs(top, delta, 1 if path == "single" else (2 if path == "multi" else 3))
        R = ref_decode(inp)
        n_keep = int(R.keep.sum())
        assert n_keep == top + delta, (path, top, delta, n_keep)
        found.add(f"top{top}_count{['-1', '=', '+1'][delta + 1]}")
        exp = expected_order(R, top)
        key = _kernel_key(R, expected_order(R, 1320))
        if ties and len(key) > top and key[top - 1] == key[top]:
            found.add("tie_straddles_cut")
            sl = R.slot[expected_order(R, 1320)][top - 2:top + 2]
            if len(set((sl // inp.n1).tolist())) > 1:
                found.add(f"tie_across_cavs_{path}")
        drop = np.flatnonzero(R.passed & ~R.keep)
        assert len(drop) == 9
        if (R.score[drop].max() > R.score[exp].min()) if len(exp) else True:
            found.add("dropped_candidate_above_cut")
    want = {f"top{t}_count{d}" for t in SORT_TOPS for d in ("-1", "=", "+1")} | {
        "tie_straddles_cut", "tie_across_cavs_multi", "tie_across_cavs_late", "dropped_candidate_above_cut"}
    assert want <= found, want - found


def _nms_census(case: NCase, run: NmsRun, corners, inp: Inputs):
    f = {f"n{len(corners)}"}
    n = len(corners)
    if n % 64:
        f.add("partial_tile")
    if n > 64:
        f.add("diagonal_and_off_diagonal_tiles")
    if n > 1280:
        f.add("21_words")
    if run.word_crossing_chains:
        f.add("chain_across_word")
    if run.clockwise:
        f.add("clockwise_reversed")
    if case.kind == "identical" and len(run.pick) == 1:
        f.add("all_identical_one_survivor")
    if case.kind == "disjoint" and len(run.pick) == n == 1320:
        f.add("all_disjoint_all_survive")
    if case.kind == "exact":
        f.add(f"exact_thr_{case.thr}")
    if case.kind == "clusters":
        assert run.nearest > NEAR_THR, f"{case.name}: a generated pair has |IoU - thr| = {run.nearest:.3g}"
    return f


NMS_SITUATIONS = {"n63", "n64", "n65", "n127", "n128", "n129", "n1320", "partial_tile", "diagonal_and_off_diagonal_tiles",
                  "21_words", "chain_across_word", "clockwise_reversed", "all_identical_one_survivor", "all_disjoint_all_survive",
                  "exact_thr_0.15", "exact_thr_0.5", "exact_thr_0.25"}


def _ref_nms_case(case: NCase):
    """CPU stand-in for the kernel's decode-only output: the float64 corners rounded to fp32, in the pinned order."""
    inp = _nms_inputs(case)
    R = ref_decode(inp)
    exp = expected_order(R, 1320)
    corners = R.corners[exp].astype(np.float32)
    return inp, R, exp, corners


def test_nms_cases_cover_every_situation():
    found = set()
    for name, case in NCASES.items():
        inp, R, exp, corners = _ref_nms_case(case)
        assert len(exp) == int(R.keep.sum()) == (case.n or len(_exact_pairs(case.thr)))
        if case.kind == "exact":
            assert np.array_equal(corners.astype(np.float64), R.corners[exp]), "built corners must be fp32-exact"
        run = ref_nms(corners, case.thr)
        found |= _nms_census(case, run, corners, inp)
        print(f"{name}: {len(corners)} boxes, {run.clipped} pairs clipped, {run.suppressed} above the threshold, "
              f"{len(run.pick)} picks, nearest |IoU - thr| {run.nearest:.3g}")
    assert NMS_SITUATIONS <= found, NMS_SITUATIONS - found


def test_exact_nms_pairs_decide_as_built():
    """the exact groups: which member survives, stated by hand"""
    for thr in (0.15, 0.5, 0.25):
        case = NCase("x", 0, thr=thr, kind="exact", T="identity")
        _, _, _, corners = _ref_nms_case(case)
        pick = set(ref_nms(corners, thr).pick.tolist())
        if thr == 0.15:
            # groups: identical, nested 1/4, nested 1/16, edge, vertex, zero-area pair, zero-area inside, zero-area first
            want = [0, 0, 1, 1, 1, 1, 1, 1]
            assert [int((2 * g + 1) in pick) for g in range(8)] == want
        else:
            # IoU exactly the threshold is kept, one ulp above is suppressed
            assert [int((2 * g + 1) in pick) for g in range(2)] == [1, 0]


def _range_census(name, inp, R):
    f = set()
    exp = expected_order(R, 1320)
    corners = R.corners[exp].astype(np.float32)
    lim = RANGES[name]
    for k in range(6):
        if float(np.float32(lim[k])) != lim[k]:
            f.add("inexact_limit")
            break
    if (range_keep(corners, lim) != range_keep(corners, lim, ("f32_range_limits",))).any():
        f.add("f32_limit_disagrees")
    if any(float(v) == lim[k] for k in range(6) for v in [np.float32(lim[k])]):
        f.add("exact_limit")
    run = ref_nms(corners, 0.15)
    in_r = range_keep(corners, lim)
    if (~in_r[run.pick]).any() and any(in_r[j] and j not in set(run.pick.tolist()) for j in range(len(corners))):
        f.add("out_of_range_box_suppresses_in_range_box")
    return f


def test_range_cases_cover_every_situation():
    found = set()
    for name in RANGES:
        inp = _range_inputs(name)
        found |= _range_census(name, inp, ref_decode(inp))
    assert {"inexact_limit", "f32_limit_disagrees", "exact_limit", "out_of_range_box_suppresses_in_range_box"} <= found, found


# ---------------------------------------------------------------------------------------------------------------------------
# GPU tests
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(DCASES))
def test_decode(name, decode_inputs):
    case = DCASES[name]
    inp = decode_inputs[name]
    R = ref_decode(inp)
    top = int(R.keep.sum())
    boxes, scores, stats = _gpu_twice(inp, case.path, 2.0, top, views=case.views)
    assert stats.tolist() == [int(R.passed.sum()), int(R.keep.sum())]
    ratio, sratio = check_decode(R, expected_order(R, top), boxes, scores)
    print(f"MEASURED decode {name}: corners err/bound {ratio:.3f}, scores err/bound {sratio:.3f}, {top} boxes")


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["single", "multi", "late"])
def test_decode_exact_edges(path):
    inp, _ = _edge_inputs()
    R = ref_decode(inp)
    boxes, scores, stats = _gpu_twice(inp, path, 2.0, 64)
    assert stats.tolist() == [int(R.passed.sum()), int(R.keep.sum())]
    check_decode(R, expected_order(R, 64), boxes, scores, exact=inp.exact)


@pytest.mark.gpu
@pytest.mark.parametrize("path, top, delta", SORT_CASES)
def test_sort_and_top_cut(path, top, delta):
    inp, _ = _sort_inputs(top, delta, 1 if path == "single" else (2 if path == "multi" else 3))
    R = ref_decode(inp)
    boxes, scores, stats = _gpu(inp, path, 2.0, top)
    exp = expected_order(R, top)
    assert stats.tolist() == [int(R.passed.sum()), int(R.keep.sum())]
    assert len(boxes) == len(exp) == min(top, top + delta)
    assert np.array_equal(boxes.astype(np.float64), R.corners[exp]), "order or corners differ"
    assert (np.abs(scores - R.score[exp]) <= R.score_bound[exp]).all()


_NMS_MEASURED = {}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(NCASES))
def test_rotated_nms(name):
    case = NCASES[name]
    inp = _nms_inputs(case)
    n = int(ref_decode(inp).keep.sum())
    top = max(n, 1)
    d_boxes, d_scores, _ = _gpu_twice(inp, "single", 2.0, top)
    assert len(d_boxes) == n
    run = ref_nms(d_boxes, case.thr)
    _nms_census(case, run, d_boxes, inp)
    boxes, scores, _ = _gpu_twice(inp, "single", case.thr, top)
    assert len(boxes) == len(run.pick), f"{len(boxes)} picks, expected {len(run.pick)}"
    assert boxes.tobytes() == d_boxes[run.pick].tobytes(), "pick list differs"
    assert scores.tobytes() == d_scores[run.pick].tobytes()
    print(f"MEASURED nms {name}: {n} boxes, {run.clipped} pairs clipped, {run.suppressed} above the threshold, "
          f"{len(run.pick)} picks, nearest |IoU - thr| {run.nearest:.3g}")


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["single", "late"])
@pytest.mark.parametrize("name", list(RANGES))
def test_range_mask(name, path):
    inp = _range_inputs(name)
    lim = RANGES[name]
    top = int(ref_decode(inp).keep.sum())
    b0, s0, _ = _gpu(inp, path, 0.15, top)
    b1, s1, _ = _gpu(inp, path, 0.15, top, gt_range=lim)
    m = range_keep(b0, lim)
    assert 0 < m.sum() < len(b0)
    assert b1.tobytes() == b0[m].tobytes(), (f"{len(b1)} boxes kept, the float64 range test keeps {int(m.sum())}: "
                                             f"{_range_diff(b0, b1, m)}")
    assert s1.tobytes() == s0[m].tobytes()


def _range_diff(b0, b1, m):
    got = {bytes(b.tobytes()) for b in b1}
    extra = [b0[k].min(axis=0).tolist() + b0[k].max(axis=0).tolist() for k in range(len(b0)) if not m[k] and b0[k].tobytes() in got]
    return f"kept although outside (min xyz, max xyz): {extra[:3]}"


@pytest.mark.gpu
def test_entry_points_agree():
    """single == multi(1) == late(1); multi(n) == late(n) for n = 2 and 16; every run repeats bit for bit"""
    case = DCase("entry", 6, 7, 2, n_cav=16, path="multi", seed=21)
    inp = _decode_inputs(case)
    rng_ = RANGES["r140.8"]
    def sub(k):
        return Inputs(anchors=inp.anchors, cavs=inp.cavs[:k], bins=inp.bins, order=inp.order, dir_offset=inp.dir_offset)
    one = [_gpu_twice(sub(1), p, 0.15, 1000, gt_range=rng_, views=v) for p in ("single", "multi", "late") for v in (False, True)]
    for o in one[1:]:
        for x, y in zip(one[0], o):
            assert x.tobytes() == y.tobytes()
    for k in (2, 16):
        a = _gpu_twice(sub(k), "multi", 0.15, 1000, gt_range=rng_)
        b = _gpu_twice(sub(k), "late", 0.15, 1000, gt_range=rng_, views=True)
        for x, y in zip(a, b):
            assert x.tobytes() == y.tobytes()
        assert len(a[0]) > 0


# ---------------------------------------------------------------------------------------------------------------------------
# CPU tests: goldens, the range helper, the bound check
# ---------------------------------------------------------------------------------------------------------------------------
def _golden_filtered_scores(cavs, anchors, params):
    """the reference's scores after the threshold and the filters (oracle/postprocess.py's steps), all cavs together"""
    from oracle import postprocess as opp
    out = []
    for cav in cavs:
        prob = torch.sigmoid(cav["cls"].permute(0, 2, 3, 1)).reshape(1, -1)
        boxes3d = opp.delta_to_boxes3d(cav["reg"], anchors)
        mask = torch.gt(prob, params["target_args"]["score_threshold"]).view(1, -1)
        b = boxes3d[0][mask[0]]
        s = prob[0][mask[0]]
        if "iou" in cav:
            q = torch.sigmoid(cav["iou"].permute(0, 2, 3, 1)).reshape(1, -1)[0][mask[0]]
            s = s * torch.pow((torch.clamp(q, 0, 1) + 1) / 2, 4)
        nb, off = params["dir_args"]["num_bins"], params["dir_args"]["dir_offset"]
        dcls = cav["dir"].permute(0, 2, 3, 1).contiguous().reshape(1, -1, nb)[mask]
        lab = torch.max(dcls, dim=-1)[1]
        period = 2 * np.pi / nb
        b[..., 6] = opp.limit_period(b[..., 6] - off, 0, period) + off + period * lab.to(dcls.dtype)
        b[..., 6] = opp.limit_period(b[..., 6], 0.5, 2 * np.pi)
        c = opp.project_box3d(opp.boxes_to_corners_3d(b, params["order"]), cav["T"])
        xl = c[:, :, 0].max(1)[0] - c[:, :, 0].min(1)[0]
        yl = c[:, :, 1].max(1)[0] - c[:, :, 1].min(1)[0]
        keep = (xl <= 6) & (yl <= 6) & (yl != 0) & (c[:, :, 2].min(1)[0] >= -3) & (c[:, :, 2].max(1)[0] <= 1)
        out.append(s[keep])
    return torch.cat(out)


def test_golden_candidates_have_no_tied_scores(golden_dir):
    """tests/golden/postprocess.pt pins the reference only where its argsort order is defined: no two candidates left after
    the filters share a score, so numpy's tie order never enters the golden comparison."""
    from oracle import golden
    g = golden.load(os.path.join(golden_dir, "postprocess.pt"))
    sets = {f"cases/{k}": [g["cases"][k]] for k in ("dense", "sparse")}
    sets.update({f"multi/{k}": v["cavs"] for k, v in g["multi"].items()})
    for name, cavs in sets.items():
        s = _golden_filtered_scores(cavs, g["anchors"], g["params"]).numpy()
        assert len(s) > 0, name
        assert len(np.unique(s)) == len(s), f"{name}: {len(s) - len(np.unique(s))} tied scores"


CONFIGURED_RANGES = list(RANGES.values()) + [[-51.2, -51.2, -3, 51.2, 51.2, 1], [-100.8, -40, -3.5, 100.8, 40, 1.5]]


def test_box_range_limits_reproduce_the_float64_test():
    from heal_b200 import ops
    for lim in CONFIGURED_RANGES:
        f = list(ops._box_range_f32(lim))
        for k in range(6):
            c0 = np.float32(lim[k])
            cs = [c0]
            for _ in range(4):
                cs = [np.nextafter(cs[0], np.float32(-np.inf))] + cs + [np.nextafter(cs[-1], np.float32(np.inf))]
            for c in cs:
                got = (c >= np.float32(f[k])) if k < 3 else (c <= np.float32(f[k]))
                want = (float(c) >= lim[k]) if k < 3 else (float(c) <= lim[k])
                assert got == want, (lim, k, float(c))


def test_bound_rejects_plausible_kernel_bugs():
    """each bug restated on the float64 reference fails the comparison the GPU tests make"""
    # corners: l / w swapped, dir_offset dropped, a period off by one bin
    inp = _decode_inputs(DCASES["hwl_bins2_A2"])
    R = ref_decode(inp)
    exp = expected_order(R, 1320)
    for bug in ("l_w_swapped", "dir_offset_dropped", "period_off_by_one_bin"):
        B = ref_decode(inp, (bug,))
        eb = expected_order(B, 1320)
        with pytest.raises(AssertionError):
            check_decode(R, exp, B.corners[eb].astype(np.float32), B.score[eb].astype(np.float32))
    # the kernel's own result passes
    check_decode(R, exp, R.corners[exp].astype(np.float32), R.score[exp].astype(np.float32))
    # ties in reversed order
    inp = _decode_inputs(DCASES["late3_views_ties"])
    R = ref_decode(inp)
    assert not np.array_equal(expected_order(R, 1320, ("ties_reversed",)), expected_order(R, 1320))
    # the top cut before the size filter
    inp, _ = _sort_inputs(64, 1)
    R = ref_decode(inp)
    assert not np.array_equal(expected_order(R, 64, ("top_cut_before_filter",)), expected_order(R, 64))
    # NMS: `>=`, a removed box still suppressing, no clockwise reversal
    for name, bug in (("exact_thr_0.5", "iou_ge"), ("exact_thr_0.25", "iou_ge"), ("n129_chain", "suppressor_state_ignored"),
                      ("n300_clockwise", "no_ccw_reversal")):
        _, _, _, corners = _ref_nms_case(NCASES[name])
        good, bad = ref_nms(corners, NCASES[name].thr).pick, ref_nms(corners, NCASES[name].thr, (bug,)).pick
        assert not np.array_equal(good, bad), (name, bug)
    # range limits rounded to the nearest fp32
    for name, lim in RANGES.items():
        inp = _range_inputs(name)
        R = ref_decode(inp)
        c = R.corners[expected_order(R, 1320)].astype(np.float32)
        assert (range_keep(c, lim) != range_keep(c, lim, ("f32_range_limits",))).any(), name
