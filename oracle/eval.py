"""CPU restatement of the reference's per-frame detection evaluation (opencood/utils/eval_utils.py:40-92 caluclate_tp_fp,
:14-37 voc_ap, :95-137 calculate_ap; common_utils.py:230-270 compute_iou / convert_format) on QuadPolygon, the shapely stand-in
of oracle/postprocess.py.

TEST INFRASTRUCTURE ONLY (tests/, oracle/make_golden_eval.py, profiles/) -- never imported by heal_b200/.

Pinned to the unmodified reference by tests/golden/eval_tp_fp.pt (oracle/make_golden_eval.py).  Differences of form, not of
result: each (det, GT) IoU is computed once into a float32 matrix (the reference recomputes the row of every unmatched GT per
detection, with the same operations), pairs whose bounding boxes do not touch get 0 without building the clip (as
quad_intersection_area does), and the greedy pass runs for several thresholds.  Two rules are made explicit:
  - detections are ordered by a STABLE descending sort (ties by ascending index); the reference's np.argsort(-score) leaves ties in
    an unspecified order;
  - the threshold is compared in float32 (`max_iou < np.float32(thr)`), which is what NumPy 2 does with `np.max(ious) < iou_thresh`
    (NEP 50: the Python float takes the array's dtype); NumPy 1 compared in float64.
"""
from __future__ import annotations

import numpy as np

from oracle.postprocess import QuadPolygon, quad_intersection_area


def polygons(boxes) -> list:
    """convert_format: a polygon of corners 0..3, (x, y), per (8, 3) or (4, 2) box"""
    return [QuadPolygon([(b[i, 0], b[i, 1]) for i in range(4)]) for b in np.asarray(boxes)]


def iou_matrix(det, gt) -> np.ndarray:
    """(K, G) float32: compute_iou of every det against every GT, `intersection.area / union.area` in float64 rounded once.
    A union of area 0 raises ZeroDivisionError, as the reference's float division does."""
    det, gt = np.asarray(det), np.asarray(gt)
    P, Q = polygons(det), polygons(gt)
    out = np.zeros((len(P), len(Q)), dtype=np.float32)
    if not P or not Q:
        return out
    dmin, dmax = det[:, :4, :2].min(1).astype(np.float64), det[:, :4, :2].max(1).astype(np.float64)
    gmin, gmax = gt[:, :4, :2].min(1).astype(np.float64), gt[:, :4, :2].max(1).astype(np.float64)
    touch = ((dmax[:, None, 0] >= gmin[None, :, 0]) & (gmax[None, :, 0] >= dmin[:, None, 0]) &
             (dmax[:, None, 1] >= gmin[None, :, 1]) & (gmax[None, :, 1] >= dmin[:, None, 1]))
    for i, p in enumerate(P):
        for j, q in enumerate(Q):
            inter = quad_intersection_area(p.pts, q.pts) if touch[i, j] else 0.0
            out[i, j] = inter / (p.area + q.area - inter)
    return out


def stable_order(scores) -> np.ndarray:
    """descending score, ties by ascending index (NaN last, as np.argsort(-score) puts them)"""
    return np.argsort(-np.asarray(scores, dtype=np.float32), kind="stable")


def tp_fp(det, scores, gt, thresholds):
    """One frame at several thresholds -> (sorted scores (K,) float32, tp (n_thr, K) uint8), in stable descending score order."""
    scores = np.asarray(scores, dtype=np.float32)
    order = stable_order(scores)
    ious = iou_matrix(np.asarray(det)[order], gt)
    K, G = ious.shape
    tp = np.zeros((len(thresholds), K), dtype=np.uint8)
    for t, thr in enumerate(thresholds):
        left = np.ones(G, dtype=bool)
        for r in range(K):
            idx = np.flatnonzero(left)
            if idx.size == 0:
                continue
            row = ious[r, idx]
            if row.max() < np.float32(thr):
                continue
            tp[t, r] = 1
            left[idx[np.argmax(row)]] = False
    return scores[order], tp


def caluclate_tp_fp(det_boxes, det_score, gt_boxes, result_stat, iou_thresh):
    """the reference's effect on result_stat[iou_thresh] (numpy / torch CPU inputs)"""
    stat = result_stat[iou_thresh]
    if det_boxes is not None:
        s, tp = tp_fp(np.asarray(det_boxes), np.asarray(det_score), np.asarray(gt_boxes), [iou_thresh])
        stat["score"] += s.tolist()
        stat["tp"] += tp[0].tolist()
        stat["fp"] += (1 - tp[0]).tolist()
    stat["gt"] += int(gt_boxes.shape[0])


def calculate_ap(result_stat, iou):
    """AP of the accumulated lists: sort by score, cumulative TP / FP, recall and precision, then the VOC 2010 area under the
    monotone precision envelope, summed in the reference's order."""
    st = result_stat[iou]
    fp, tp, score = np.array(st["fp"]), np.array(st["tp"]), np.array(st["score"])
    assert len(fp) == len(tp) == len(score)
    order = np.argsort(-score)
    ctp, cfp = np.cumsum(tp[order]).tolist(), np.cumsum(fp[order]).tolist()
    rec = [0.0] + [float(v) / st["gt"] for v in ctp] + [1.0]
    prec = [0.0] + [float(a) / (b + a) for a, b in zip(ctp, cfp)] + [0.0]
    for i in range(len(prec) - 2, -1, -1):
        prec[i] = max(prec[i], prec[i + 1])
    ap = 0.0
    for i in range(1, len(rec)):
        if rec[i] != rec[i - 1]:
            ap += (rec[i] - rec[i - 1]) * prec[i]
    return ap


def new_result_stat(thresholds=(0.3, 0.5, 0.7)):
    return {t: {"tp": [], "fp": [], "gt": 0, "score": []} for t in thresholds}
