"""oracle/eval.py (the numpy restatement of the reference's per-frame evaluation) against tests/golden/eval_tp_fp.pt, which the
unmodified reference's caluclate_tp_fp and calculate_ap wrote (oracle/make_golden_eval.py); and the rules the restatement makes
explicit: the NumPy 2 threshold test, ZeroDivisionError on a zero-area union, the stable order of tied scores."""
import os

import numpy as np
import pytest
import torch

from oracle import eval as oev
from oracle.make_golden_eval import rect


@pytest.fixture(scope="module")
def golden(golden_dir):
    return torch.load(os.path.join(golden_dir, "eval_tp_fp.pt"), weights_only=False)


def _np(t):
    return None if t is None else t.numpy()


def test_restatement_reproduces_the_golden_lists_and_ap(golden):
    thr = golden["thresholds"]
    total = oev.new_result_stat(thr)
    for f in golden["frames"]:
        per = oev.new_result_stat(thr)
        for t in thr:
            oev.caluclate_tp_fp(_np(f["det"]), _np(f["score"]), f["gt"], per, t)
            oev.caluclate_tp_fp(_np(f["det"]), _np(f["score"]), f["gt"], total, t)
        assert per == f["result_stat"], f["name"]
    assert total == golden["result_stat"]
    for t in thr:
        assert oev.calculate_ap(total, t) == golden["ap"][t]
    assert [golden["ap"][t] for t in thr] == sorted((golden["ap"][t] for t in thr), reverse=True)


def test_golden_covers_the_cases_it_is_made_for(golden):
    names = {f["name"]: f for f in golden["frames"]}
    rs = lambda n, t: names[n]["result_stat"][t]["tp"]            # noqa: E731
    assert rs("iou_eq_f32(0.7)_below_0.7", 0.7) == [1] and rs("iou_one_ulp_below_f32(0.7)", 0.7) == [0]
    assert rs("iou_below_0.3_rounds_to_f32(0.3)", 0.3) == [1] and rs("iou_one_ulp_below_f32(0.3)", 0.3) == [0]
    assert rs("iou_exactly_0.5", 0.5) == [1] and rs("iou_one_ulp_below_0.5", 0.5) == [0]
    assert rs("equal_iou_lowest_index", 0.3) == [1, 1] and rs("equal_iou_lowest_index_swapped", 0.3) == [1, 0]
    assert rs("loses_best_gt", 0.3) == [1, 1] and rs("loses_best_gt", 0.5) == [1, 0]
    assert names["det_none"]["det"] is None and names["det_none"]["result_stat"][0.5] == {"tp": [], "fp": [], "gt": 2, "score": []}
    ks = [0 if f["det"] is None else f["det"].shape[0] for f in golden["frames"]]
    gs = [f["gt"].shape[0] for f in golden["frames"]]
    assert max(ks) == 1000 and 0 in ks and 1 in ks and max(gs) == 300 and 0 in gs


def test_threshold_is_compared_in_float32():
    """an IoU equal to float32(0.7), which is below 0.7, is a TP; one float32 ulp less is an FP"""
    f = np.float32(0.7)
    assert float(f) < 0.7
    if int(np.__version__.split(".")[0]) >= 2:
        assert not (np.max(np.array([f], dtype=np.float32)) < 0.7)        # what the reference's test does under NumPy 2
    below = np.nextafter(f, np.float32(0))
    gt = rect(0, 16.0, 0, 16.0)[None]
    for iou, want in ((f, 1), (below, 0)):
        w = float(iou) * 16.0                        # det [0, w] x [0, 16] inside the GT: IoU = w / 16 exactly
        det = rect(0, w, 0, 16.0)[None]
        assert oev.iou_matrix(det, gt)[0, 0] == iou
        assert oev.tp_fp(det, [0.5], gt, [0.7])[1].tolist() == [[want]]


def test_zero_area_union_raises():
    point = np.zeros((1, 8, 3), np.float32)
    segment = rect(0, 4, 0, 0)[None]
    with pytest.raises(ZeroDivisionError):
        oev.tp_fp(point, [0.5], segment, [0.5])
    # a degenerate det against a real GT is an FP, not an error
    assert oev.tp_fp(point, [0.5], rect(0, 1, 0, 1)[None], [0.5])[1].tolist() == [[0]]


def test_tied_scores_go_by_ascending_index():
    rng = np.random.default_rng(3)
    scores = rng.choice(np.float32([0.9, 0.5, 0.25, np.nan]), 64).astype(np.float32)
    order = oev.stable_order(scores)
    key = [(1, 0.0, i) if np.isnan(s) else (0, -float(s), i) for i, s in enumerate(scores)]
    assert order.tolist() == sorted(range(64), key=lambda i: key[i])
