"""Golden vectors of the per-frame detection evaluation (TEST INFRASTRUCTURE ONLY): the UNMODIFIED reference's
eval_utils.caluclate_tp_fp at IoU 0.3, 0.5 and 0.7 over seeded frames, then its calculate_ap, with oracle.postprocess.QuadPolygon
installed as shapely.geometry.Polygon (shapely is not installed here; the same stand-in pins the NMS goldens).

    python oracle/make_golden_eval.py        (needs the reference package: oracle/_ref or HEAL_REFERENCE_ROOT)

Writes tests/golden/eval_tp_fp.pt: per frame the inputs (det (K, 8, 3) fp32 or None, score (K,) fp32 or None, gt (G, 8, 3) fp32)
and the reference's per-frame result_stat; the three accumulated result_stat dicts; AP30 / AP50 / AP70.

Frames:
  - OPV2V-like: GTs are mostly 4.5 x 2 m vehicles on a grid (some rotated, some other sizes), corners from boxes_to_corners_3d in
    'hwl' or 'lhw' order, half of the frames mirrored in y so that both corner orientations occur.  Dets are jittered GTs plus
    false positives, with some GTs missed; K from 0 to the 1000 cap, G from 0 to 300.  Every IoU the reference compares with a
    threshold lies at least MARGIN_ULPS float32 ulps away from it, and every TP's IoU at least MARGIN_ULPS above the runner-up: the
    fp64 area sums of the GPU and of np.dot round differently, so only constructed frames may sit on a boundary.
  - constructed: two dets competing for one GT; a det that loses its best GT and matches its second best; equal IoUs to two GTs
    (the lowest GT index wins), in both index orders; G = 0; an empty det tensor; det_boxes None.
  - exact thresholds: axis-aligned rectangles whose coordinates are exact in fp32 and whose clip and areas are exact in fp64, so
    the IoU is a known rational: IoU exactly 0.5; IoUs below 0.3 or 0.7 in fp64 that round to float32(thr) (TPs under NumPy 2);
    IoUs one float32 ulp below each threshold (FPs).
All det scores are distinct across frames, so neither the reference's unstable argsort nor calculate_ap's sort depends on ties."""
import os
import sys
import types
from fractions import Fraction

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import eval as oev                 # noqa: E402
from oracle import postprocess as opp          # noqa: E402
from oracle import ref_shim                    # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "eval_tp_fp.pt")
THRESHOLDS = (0.3, 0.5, 0.7)
MARGIN_ULPS = 4

# (name, seed, K, G, order, mirrored)
RANDOM_FRAMES = (
    ("k1_g1", 11, 1, 1, "hwl", False),
    ("k7_g5", 12, 7, 5, "lhw", True),
    ("k60_g40", 13, 60, 40, "hwl", True),
    ("k150_g100", 14, 150, 100, "lhw", False),
    ("k300_g150", 15, 300, 150, "hwl", False),
    ("k250_g120_mirrored", 16, 250, 120, "lhw", True),
    ("k1000_g300", 17, 1000, 300, "hwl", False),
    ("k40_g0", 18, 40, 0, "hwl", False),
    ("k0_g30", 19, 0, 30, "lhw", True),
)


# ---- box construction ------------------------------------------------------------------------------------------------
def corners_of(boxes7: np.ndarray, order: str, mirrored: bool) -> np.ndarray:
    """(N, 7) boxes in `order` -> (N, 8, 3) fp32 corners (box_utils.boxes_to_corners_3d), y mirrored on request"""
    if len(boxes7) == 0:
        return np.zeros((0, 8, 3), np.float32)
    c = opp.boxes_to_corners_3d(torch.from_numpy(np.asarray(boxes7, np.float32)), order).numpy().astype(np.float32)
    if mirrored:
        c[..., 1] = -c[..., 1]
    return c


def rect(x0, x1, y0, y1, ccw=True) -> np.ndarray:
    """(8, 3) fp32 corners of an axis-aligned box [x0, x1] x [y0, y1] x [-1, 1]"""
    q = [(x0, y0), (x1, y0), (x1, y1), (x0, y1)]
    if not ccw:
        q = q[::-1]
    return np.array([(x, y, z) for z in (-1.0, 1.0) for x, y in q], dtype=np.float32)


def _boxes7(xyz, lwh, yaw, order):
    x, y, z = xyz.T
    l, w, h = lwh.T
    cols = (x, y, z, h, w, l, yaw) if order == "hwl" else (x, y, z, l, w, h, yaw)
    return np.stack(cols, axis=1)


def random_frame(seed, K, G, order, mirrored):
    rng = np.random.default_rng(seed)
    cells = rng.choice(20 * 20, size=G, replace=False)
    xyz = np.stack([(cells % 20) * 8.0 - 80 + rng.uniform(-1, 1, G), (cells // 20) * 7.0 - 70 + rng.uniform(-0.5, 0.5, G),
                    np.full(G, -1.0)], axis=1)
    lwh = np.tile([4.5, 2.0, 1.5], (G, 1))
    other = rng.random(G) < 0.2
    lwh[other] = np.stack([rng.uniform(3.5, 5.5, other.sum()), rng.uniform(1.7, 2.3, other.sum()),
                           rng.uniform(1.4, 2.0, other.sum())], axis=1)
    yaw = rng.choice([0.0, np.pi / 2, np.pi, -np.pi / 2], G) + rng.normal(0, 0.05, G)
    rot = rng.random(G) < 0.25
    yaw[rot] = rng.uniform(-np.pi, np.pi, rot.sum())
    gt = _boxes7(xyz, lwh, yaw, order)
    hit = np.flatnonzero(rng.random(G) < 0.85)
    hit = hit[:K]
    n_fp = K - len(hit)
    dxyz = xyz[hit] + np.concatenate([rng.normal(0, 0.3, (len(hit), 2)), rng.normal(0, 0.1, (len(hit), 1))], axis=1)
    dlwh = lwh[hit] * (1 + rng.normal(0, 0.05, (len(hit), 3)))
    dyaw = yaw[hit] + rng.normal(0, 0.08, len(hit))
    fxyz = np.stack([rng.uniform(-90, 90, n_fp), rng.uniform(-80, 80, n_fp), np.full(n_fp, -1.0)], axis=1)
    flwh = np.stack([rng.uniform(3, 6, n_fp), rng.uniform(1.5, 2.5, n_fp), rng.uniform(1.4, 2.0, n_fp)], axis=1)
    fyaw = rng.uniform(-np.pi, np.pi, n_fp)
    det = _boxes7(np.concatenate([dxyz, fxyz]), np.concatenate([dlwh, flwh]), np.concatenate([dyaw, fyaw]), order)
    perm = rng.permutation(K)
    det = det[perm]
    score = np.concatenate([rng.uniform(0.3, 1.0, len(hit)), rng.uniform(0.1, 0.8, n_fp)])[perm].astype(np.float32)
    return corners_of(det, order, mirrored), score, corners_of(gt, order, mirrored)


def _ulps(a: np.float32, b: np.float32) -> int:
    ia, ib = np.array([a, b], np.float32).view(np.int32)
    return abs(int(ia) - int(ib))


def check_margins(det, score, gt):
    """every compared max IoU >= MARGIN_ULPS from each threshold; every TP's IoU >= MARGIN_ULPS above the runner-up"""
    if det is None or len(det) == 0 or len(gt) == 0:
        return True
    ious = oev.iou_matrix(det[oev.stable_order(score)], gt)
    for thr in THRESHOLDS:
        t32, left = np.float32(thr), np.ones(len(gt), bool)
        for r in range(len(det)):
            idx = np.flatnonzero(left)
            if idx.size == 0:
                break
            row = np.sort(ious[r, idx])[::-1]
            if _ulps(row[0], t32) < MARGIN_ULPS:
                return False
            if row[0] >= t32:
                if row.size > 1 and _ulps(row[0], row[1]) < MARGIN_ULPS:
                    return False
                left[idx[np.argmax(ious[r, idx])]] = False
    return True


def nested_pair(lo: Fraction, hi: Fraction = None, ccw=True):
    """det [0, w] x [0, h] inside gt [0, 16] x [0, 16] (units 2^-13 m, w, h integers <= 2^17): IoU = w h / 2^34 exactly, with
    lo < IoU < hi, or IoU == lo when hi is None"""
    S = 1 << 34
    for w in range(1 << 17, 0, -1):
        if hi is None:
            if (lo * S).denominator == 1 and int(lo * S) % w == 0 and int(lo * S) // w <= (1 << 17):
                h = int(lo * S) // w
                break
        else:
            h = int(lo * S / w) + 1
            if h <= (1 << 17) and Fraction(w * h, S) < hi:
                break
    else:
        raise RuntimeError("no rectangle pair")
    u = 2.0 ** -13
    iou = Fraction(w * h, S)
    assert (hi is None and iou == lo) or lo < iou < hi
    return rect(0, w * u, 0, h * u, ccw), rect(0, 16.0, 0, 16.0, not ccw), iou


def constructed_frames():
    f32 = lambda v: Fraction(float(np.float32(v)))            # noqa: E731
    ulp = {0.3: Fraction(1, 1 << 25), 0.5: Fraction(1, 1 << 25), 0.7: Fraction(1, 1 << 24)}    # float32 ulp just below thr
    fr = []
    # two dets for one GT: the higher score takes it
    fr.append(("two_dets_one_gt", np.stack([rect(0.5, 4.5, 0, 2), rect(1, 5, 0, 2)]), [0.93, 0.91], np.stack([rect(0, 4, 0, 2)])))
    # the second det's best GT (index 0) went to the first det; it matches its second best (IoU 1/3) at 0.3 only
    fr.append(("loses_best_gt", np.stack([rect(1, 5, 0, 2), rect(0, 4, 0, 2, False)]), [0.83, 0.87],
               np.stack([rect(0, 4, 0, 2), rect(3, 7, 0, 2)])))
    # equal IoU 1/3 to two GTs: the lowest GT index wins, and decides whether the second det finds a GT
    fr.append(("equal_iou_lowest_index", np.stack([rect(2, 6, 0, 2), rect(4.5, 8.5, 0, 2)]), [0.77, 0.75],
               np.stack([rect(0, 4, 0, 2), rect(4, 8, 0, 2)])))
    fr.append(("equal_iou_lowest_index_swapped", np.stack([rect(2, 6, 0, 2), rect(4.5, 8.5, 0, 2)]), [0.73, 0.71],
               np.stack([rect(4, 8, 0, 2), rect(0, 4, 0, 2)])))
    fr.append(("g0", np.stack([rect(0, 4, 0, 2), rect(10, 14, 0, 2)]), [0.67, 0.65], np.zeros((0, 8, 3), np.float32)))
    fr.append(("empty_det", np.zeros((0, 8, 3), np.float32), [], np.stack([rect(0, 4, 0, 2)])))
    fr.append(("det_none", None, None, np.stack([rect(0, 4, 0, 2), rect(5, 9, 0, 2)])))
    # exact thresholds
    fr.append(("iou_exactly_0.5", np.stack([rect(0, 3, 0, 1)]), [0.61], np.stack([rect(1, 4, 0, 1)])))
    exact = [
        ("iou_eq_f32(0.7)_below_0.7", f32(0.7), None),
        ("iou_between_f32(0.7)_and_0.7", f32(0.7), Fraction(7, 10)),
        ("iou_below_f32(0.7)_rounds_up", f32(0.7) - ulp[0.7] / 2, f32(0.7)),
        ("iou_one_ulp_below_f32(0.7)", f32(0.7) - ulp[0.7], None),
        ("iou_below_0.3_rounds_to_f32(0.3)", f32(0.3) - ulp[0.3] / 2, Fraction(3, 10)),
        ("iou_one_ulp_below_f32(0.3)", f32(0.3) - ulp[0.3], None),
        ("iou_one_ulp_below_0.5", Fraction(1, 2) - ulp[0.5], None),
    ]
    for k, (name, lo, hi) in enumerate(exact):
        d, g, _ = nested_pair(lo, hi, ccw=bool(k % 2))
        fr.append((name, d[None], [0.59 - 0.01 * k], g[None]))
    return [(n, d, None if s is None else np.asarray(s, np.float32), g) for n, d, s, g in fr]


def frames():
    out = []
    for name, seed, K, G, order, mirrored in RANDOM_FRAMES:
        for attempt in range(100):
            det, score, gt = random_frame(seed + 1000 * attempt, K, G, order, mirrored)
            if check_margins(det, score, gt):
                break
        else:
            raise RuntimeError(f"{name}: no seed within the margins")
        out.append((name, det, score, gt))
    out += constructed_frames()
    scores = np.concatenate([s for _, _, s, _ in out if s is not None])
    assert len(np.unique(scores)) == len(scores), "det scores must be distinct across frames"
    return out


def install_reference():
    """the unmodified reference with QuadPolygon as shapely.geometry.Polygon"""
    from unittest.mock import MagicMock
    sg = types.ModuleType("shapely.geometry")
    sg.Polygon = opp.QuadPolygon
    sg.Point, sg.MultiPoint = MagicMock(), MagicMock()
    sh = types.ModuleType("shapely")
    sh.geometry = sg
    sys.modules["shapely"], sys.modules["shapely.geometry"] = sh, sg
    ref_shim.install()
    import opencood.utils.eval_utils as eu
    return eu


def main():
    eu = install_reference()
    total = oev.new_result_stat(THRESHOLDS)
    rec = []
    orientations = set()
    for name, det, score, gt in frames():
        per = oev.new_result_stat(THRESHOLDS)
        t = lambda a: None if a is None else torch.from_numpy(a)          # noqa: E731
        for thr in THRESHOLDS:
            eu.caluclate_tp_fp(t(det), t(score), t(gt), per, thr)
            eu.caluclate_tp_fp(t(det), t(score), t(gt), total, thr)
        for boxes in (det, gt):
            if boxes is not None:
                orientations.update(np.sign(_signed_area(b)) for b in boxes)
        rec.append({"name": name, "det": t(det), "score": t(score), "gt": t(gt), "result_stat": per})
        print(f"{name:36s} K={0 if det is None else len(det):5d} G={len(gt):4d} " +
              " ".join(f"tp@{thr}={sum(per[thr]['tp'])}" for thr in THRESHOLDS))
    assert orientations >= {-1.0, 1.0}, "both corner orientations must occur"
    ap = {thr: eu.calculate_ap(total, thr)[0] for thr in THRESHOLDS}
    print("AP30 / AP50 / AP70:", [ap[t] for t in THRESHOLDS])
    torch.save({"thresholds": THRESHOLDS, "frames": rec, "result_stat": total, "ap": ap}, OUT)
    print(f"wrote {OUT} ({os.path.getsize(OUT)} bytes)")


def _signed_area(box) -> float:
    x, y = box[:4, 0].astype(np.float64), box[:4, 1].astype(np.float64)
    return float(np.dot(x, np.roll(y, -1)) - np.dot(y, np.roll(x, -1)))


if __name__ == "__main__":
    sys.exit(main())
