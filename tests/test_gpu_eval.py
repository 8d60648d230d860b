"""heal_eval_tp_fp on the GPU (csrc/eval.cu through ops.eval_tp_fp and the eval_utils drop-in): flags and sorted scores bit-equal
to the reference's golden (tests/golden/eval_tp_fp.pt, oracle/make_golden_eval.py) and to the oracle restatement at three and at
eight thresholds, the stable tie rule, the zero-union status, empty inputs and the size limits; and the reference's own
opencood.utils.eval_utils driven over the golden frames with install_gpu_eval() applied."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import eval as oev
from oracle import ref_shim
from oracle.make_golden_eval import random_frame, rect

pytestmark = pytest.mark.gpu

THR8 = (0.3, 0.5, 0.7, 0.1, 0.25, 0.45, 0.6, 0.85)


@pytest.fixture(scope="module")
def golden(golden_dir):
    return torch.load(os.path.join(golden_dir, "eval_tp_fp.pt"), weights_only=False)


def _cuda(a):
    return torch.as_tensor(np.asarray(a, dtype=np.float32)).cuda()


def _run(det, score, gt, thresholds):
    from heal_b200 import ops
    buf = ops.eval_tp_fp(_cuda(det).reshape(-1, 8, 3), _cuda(score).reshape(-1), _cuda(gt).reshape(-1, 8, 3), thresholds)
    status, s, tp = ops.EvalBuffers.unpack(buf.packed.cpu(), len(score), len(thresholds))
    return status, s.numpy(), tp.numpy()


def _bits(a):
    return np.asarray(a, dtype=np.float32).view(np.int32).tolist()


@pytest.mark.parametrize("thresholds", [(0.3, 0.5, 0.7), THR8], ids=["3thr", "8thr"])
def test_flags_and_scores_equal_the_golden_and_the_oracle(golden, thresholds):
    n = 0
    for f in golden["frames"]:
        if f["det"] is None:
            continue
        det, score, gt = f["det"].numpy(), f["score"].numpy(), f["gt"].numpy()
        status, s, tp = _run(det, score, gt, thresholds)
        assert status == 0, f["name"]
        os_, otp = oev.tp_fp(det, score, gt, thresholds)
        assert _bits(s) == _bits(os_), f["name"]
        assert np.array_equal(tp, otp), (f["name"], np.flatnonzero((tp != otp).any(0))[:10])
        for t, thr in enumerate(thresholds):
            if thr in f["result_stat"]:
                st = f["result_stat"][thr]
                assert tp[t].tolist() == st["tp"] and (1 - tp[t]).tolist() == st["fp"], (f["name"], thr)
                assert _bits(s) == _bits(st["score"]), f["name"]
        n += 1
    assert n >= 20


def test_tied_scores_go_by_ascending_index():
    det, score, gt = random_frame(5, 300, 150, "hwl", False)
    score = np.float32([0.9, 0.6, 0.3])[np.arange(300) % 3]
    score[::37] = np.nan
    status, s, tp = _run(det, score, gt, THR8)
    os_, otp = oev.tp_fp(det, score, gt, THR8)
    assert status == 0 and _bits(s) == _bits(os_) and np.array_equal(tp, otp)
    # the frame tells the orders apart: with the ties taken in the other direction the flags differ
    _, rtp = oev.tp_fp(det[::-1].copy(), score[::-1].copy(), gt, THR8)
    assert not np.array_equal(rtp, otp)


def test_zero_area_union_sets_the_status_and_the_drop_in_raises():
    from heal_b200.utils import eval_utils as ev
    point, segment = np.zeros((1, 8, 3), np.float32), rect(0, 4, 0, 0)[None]
    status, _, _ = _run(point, [0.5], segment, (0.5,))
    assert status == 1
    stat = oev.new_result_stat((0.5,))
    with pytest.raises(ZeroDivisionError):
        ev.caluclate_tp_fp(_cuda(point), _cuda([0.5]), _cuda(segment), stat, 0.5)
    assert stat[0.5] == {"tp": [], "fp": [], "gt": 0, "score": []}
    # a degenerate det against a real GT is an FP, and the next call clears the status
    status, _, tp = _run(point, [0.5], rect(0, 1, 0, 1)[None], (0.5,))
    assert status == 0 and tp.tolist() == [[0]]


def test_empty_inputs():
    from heal_b200.utils import eval_utils as ev
    gt = np.stack([rect(0, 4, 0, 2), rect(5, 9, 0, 2)])
    status, s, tp = _run(np.zeros((0, 8, 3)), np.zeros(0), gt, (0.3, 0.5))
    assert status == 0 and s.shape == (0,) and tp.shape == (2, 0)
    status, s, tp = _run(gt, [0.4, 0.8], np.zeros((0, 8, 3)), (0.3, 0.5))
    assert status == 0 and s.tolist() == [np.float32(0.8), np.float32(0.4)] and tp.tolist() == [[0, 0], [0, 0]]
    stat = oev.new_result_stat((0.5,))
    ev.caluclate_tp_fp(_cuda(np.zeros((0, 8, 3))), _cuda(np.zeros(0)), _cuda(gt), stat, 0.5)
    ev.caluclate_tp_fp(_cuda(gt), _cuda([0.4, 0.8]), _cuda(np.zeros((0, 8, 3))), stat, 0.5)
    assert stat[0.5] == {"tp": [0, 0], "fp": [1, 1], "gt": 2, "score": [float(np.float32(0.8)), float(np.float32(0.4))]}


def test_size_limits_are_rejected():
    box = rect(0, 1, 0, 1)[None]
    many = np.repeat(box, 4097, axis=0)
    with pytest.raises(RuntimeError):
        _run(many, np.linspace(0, 1, 4097), box, (0.5,))
    with pytest.raises(RuntimeError):
        _run(box, [0.5], many, (0.5,))
    for thresholds in ((), (0.5,) * 9, (0.0,), (float("nan"),), (-0.5,)):
        with pytest.raises(RuntimeError):
            _run(box, [0.5], box, thresholds)
    status, _, tp = _run(np.repeat(box, 4096, axis=0), np.linspace(0, 1, 4096), np.repeat(box, 4096, axis=0), (0.5,) * 8)
    assert status == 0 and tp.sum(axis=1).tolist() == [4096] * 8


@pytest.fixture
def _isolate_opencood_modules():
    """the boundary test installs the reference (with QuadPolygon as shapely's Polygon) and rebinds its caluclate_tp_fp; other
    test modules import the reference under the same names, so everything opencood / shapely is restored afterwards"""
    from heal_b200.utils import eval_utils as ev
    before = {k: v for k, v in sys.modules.items() if k.startswith(("opencood", "shapely"))}
    ref = ev.caluclate_tp_fp.reference
    yield
    ev.caluclate_tp_fp.reference = ref
    for k in [k for k in sys.modules if k.startswith(("opencood", "shapely"))]:
        del sys.modules[k]
    sys.modules.update(before)


def test_reference_eval_utils_drives_the_gpu_path(golden, tmp_path, _isolate_opencood_modules):
    if not ref_shim.available():
        pytest.skip("oracle/_ref not built")
    from oracle.make_golden_eval import install_reference
    eu = install_reference()
    original = eu.caluclate_tp_fp
    from heal_b200 import install
    fn = install.install_gpu_eval()
    assert eu.caluclate_tp_fp is fn and fn.reference is original
    assert install.install_gpu_eval() is fn and fn.reference is original          # idempotent
    calls = []

    def counting(*a):
        calls.append(a)
        return original(*a)
    fn.reference = counting
    thr = golden["thresholds"]
    total = oev.new_result_stat(thr)
    for f in golden["frames"]:
        per = oev.new_result_stat(thr)
        cu = lambda t: None if t is None else t.cuda()              # noqa: E731
        for t in thr:
            for stat in (per, total):
                eu.caluclate_tp_fp(cu(f["det"]), cu(f["score"]), cu(f["gt"]), stat, t)
        assert per == f["result_stat"], f["name"]
    assert total == golden["result_stat"]
    # det_boxes None is the only golden frame the reference function handled
    assert len(calls) == 2 * len(thr) and all(c[0] is None for c in calls)
    ap = eu.eval_final_results(total, str(tmp_path))
    assert tuple(ap) == tuple(golden["ap"][t] for t in thr)
    # CPU tensors and (N, 4, 2) boxes go to the reference function
    f = next(f for f in golden["frames"] if f["name"] == "k60_g40")
    stat = oev.new_result_stat(thr)
    eu.caluclate_tp_fp(f["det"], f["score"], f["gt"], stat, 0.5)
    eu.caluclate_tp_fp(f["det"][:, :4, :2].cuda(), f["score"].cuda(), f["gt"][:, :4, :2].cuda(), stat, 0.7)
    assert len(calls) == 2 * len(thr) + 2
    assert stat[0.5] == f["result_stat"][0.5] and stat[0.7] == f["result_stat"][0.7]
