"""CPU checks of the evaluation in the captured scene path: heal_eval_tp_fp_counted is exported with the declared arguments, the
shared `result_stat` append (heal_b200.utils.eval_utils.append_frame / append_packed) reproduces the reference's lists for given
flags, and the GT refusals of check_scene / SceneGraphCache fire on the host before anything is copied."""
import os
import re

import numpy as np
import pytest
import torch

from oracle import eval as oev
from oracle.make_golden_eval import rect

from test_scene_stream_cpu import _batch, _cache

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_args(name):
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "heal_b200.h")).read(), flags=re.S)
    m = re.search(rf"\b{name}\s*\(([^)]*)\)\s*;", src)
    assert m, f"{name} is not declared"
    return len([a for a in m.group(1).split(",") if a.strip()])


def test_counted_entry_point_is_exported_with_its_declared_arguments():
    import __graft_entry__
    __graft_entry__.build()
    from heal_b200 import _lib
    for name in ("heal_eval_tp_fp_counted", "heal_eval_tp_fp"):
        assert hasattr(_lib.lib, name)
        assert len(_lib.SIGNATURES[name][1]) == _declared_args(name), name
    assert _declared_args("heal_eval_tp_fp_counted") == 15


def _packed(scores, tp, K_cap, status=0, seed=0):
    """A host copy of EvalBuffers.packed at capacity K_cap: the frame's scores and flags, then garbage up to the capacity."""
    rng = np.random.default_rng(seed)
    n_thr, K = tp.shape
    s = rng.uniform(-5, 5, K_cap).astype(np.float32)
    f = rng.integers(0, 255, (n_thr, K_cap)).astype(np.uint8)
    s[:K], f[:, :K] = scores, tp
    return torch.from_numpy(np.concatenate([np.int32([status]).view(np.uint8), s.view(np.uint8), f.reshape(-1)]))


@pytest.fixture(scope="module")
def golden():
    return torch.load(os.path.join(ROOT, "tests", "golden", "eval_tp_fp.pt"), weights_only=False)


def test_append_packed_gives_the_reference_s_lists(golden):
    """Flags from the CPU restatement, packed at a larger capacity with garbage beyond K, appended frame by frame: the lists the
    unmodified reference wrote per frame and over the whole golden (K = 0, G = 0 and det_boxes None included)."""
    from heal_b200.utils import eval_utils as ev
    thr = golden["thresholds"]
    n = 0
    for i, f in enumerate(golden["frames"]):
        K = 0 if f["det"] is None else f["det"].shape[0]
        G = f["gt"].shape[0]
        if K * G > 20000:                                   # the restatement's polygon loop is slow; those frames run on the GPU
            continue
        if K:
            scores, tp = oev.tp_fp(f["det"].numpy(), f["score"].numpy(), f["gt"].numpy(), thr)
        else:
            scores, tp = np.zeros(0, np.float32), np.zeros((len(thr), 0), np.uint8)
        per = oev.new_result_stat(thr)
        packed = _packed(scores, tp, K + 37, seed=i)
        ev.append_packed(per, thr, packed, K, K + 37, G)
        assert per == f["result_stat"], f["name"]
        for t in thr:
            assert all(type(v) is int for v in per[t]["tp"] + per[t]["fp"]) and type(per[t]["gt"]) is int
            assert all(type(v) is float for v in per[t]["score"])
        n += 1
    assert n >= 20
    assert any(f["det"] is None for f in golden["frames"])


def test_append_frame_k0_and_g0():
    from heal_b200.utils import eval_utils as ev
    stat = oev.new_result_stat((0.5,))
    ev.append_frame(stat, 0.5, torch.zeros(0), torch.zeros(0, dtype=torch.uint8), 4)       # no box: 'gt' only
    assert stat[0.5] == {"tp": [], "fp": [], "score": [], "gt": 4}
    ev.append_frame(stat, 0.5, torch.tensor([0.9, 0.25]), torch.tensor([0, 0], dtype=torch.uint8), 0)    # no GT: all FP
    assert stat[0.5] == {"tp": [0, 0], "fp": [1, 1], "score": [float(np.float32(0.9)), 0.25], "gt": 4}
    # the reference restatement on the same frames
    ref = oev.new_result_stat((0.5,))
    oev.caluclate_tp_fp(None, None, np.zeros((4, 8, 3), np.float32), ref, 0.5)
    oev.caluclate_tp_fp(np.stack([rect(0, 1, 0, 1), rect(2, 3, 0, 1)]), np.float32([0.25, 0.9]), np.zeros((0, 8, 3), np.float32),
                        ref, 0.5)
    assert ref == stat


def test_append_packed_status_raises_and_appends_nothing():
    from heal_b200.utils import eval_utils as ev
    stat = oev.new_result_stat((0.3, 0.7))
    tp = np.ones((2, 3), np.uint8)
    with pytest.raises(ZeroDivisionError):
        ev.append_packed(stat, (0.3, 0.7), _packed(np.float32([3, 2, 1]), tp, 8, status=1), 3, 8, 5)
    with pytest.raises(RuntimeError, match="capacity"):
        ev.append_packed(stat, (0.3, 0.7), _packed(np.float32([3, 2, 1]), tp, 8, status=2), 3, 8, 5)
    assert stat == oev.new_result_stat((0.3, 0.7))
    ev.append_packed(stat, (0.3, 0.7), _packed(np.float32([3, 2, 1]), tp, 8), 3, 8, 5)
    assert stat[0.7] == {"tp": [1, 1, 1], "fp": [0, 0, 0], "score": [3.0, 2.0, 1.0], "gt": 5}


def test_eval_setup():
    from heal_b200.graph import eval_setup
    params = {"max_num": 100}
    assert eval_setup(params, None, None) == (None, None)
    assert eval_setup(params, (0.3, 0.5, 0.7), None) == ((0.3, 0.5, 0.7), 100)
    assert eval_setup({}, [0.5], 250) == ((0.5,), 250)
    with pytest.raises(ValueError, match="needs postprocess_params"):
        eval_setup(None, (0.3,), 10)
    with pytest.raises(ValueError, match="no 'max_num'"):
        eval_setup({}, (0.3,), None)
    for bad in (0, 4097, 2.5, True):
        with pytest.raises(ValueError, match="gt_capacity"):
            eval_setup(params, (0.3,), bad)
    for thr in ((), (0.5,) * 9, (0.0,), (float("nan"),)):
        with pytest.raises(ValueError, match="eval_thresholds"):
            eval_setup(params, thr, None)
    with pytest.raises(ValueError, match="without eval_thresholds"):
        eval_setup(params, None, 100)


def _gt(n, dtype=torch.float32):
    return torch.zeros((n, 8, 3), dtype=dtype)


@pytest.mark.parametrize("gt,match", [
    (None, "gt_boxes .* required"),
    (torch.zeros((3, 4, 2)), r"shape \(3, 4, 2\)"),
    (torch.zeros((3, 8)), r"shape \(3, 8\)"),
    (np.zeros((3, 8, 3), np.float32), "shape"),
    (_gt(3, torch.float64), "float64"),
    (_gt(101), "101 GT boxes, the graph's gt_capacity is 100"),
])
def test_check_scene_gt_refusals_leave_the_stream_untouched(gt, match):
    """A stream that evaluates (GT capacity 100): each refusal fires in the cache's host check, before any graph is captured or
    anything is copied."""
    c, made = _cache()
    c.gt_capacity = 100
    b = _batch(["m1", "m4", "m2", "m1"])
    assert c.check(b, _gt(100)) == ("m1", "m4", "m2", "m1") and c.check(b, _gt(0)) == ("m1", "m4", "m2", "m1")
    with pytest.raises(ValueError, match=match):
        c.check(b, gt)
    assert made == [] and c.captures == 0 and c.graphs_captured == 0


def test_gt_is_refused_without_evaluation_and_counted_in_the_copy():
    from heal_b200.graph import check_scene, scene_spec
    from test_scene_stream_cpu import CAPS, LIMITS, SENSORS
    c, made = _cache()
    b = _batch(["m1", "m3"])
    with pytest.raises(ValueError, match="without eval_thresholds"):
        c.check(b, _gt(2))
    assert made == []
    spec = scene_spec(SENSORS, ["m1", "m3"], CAPS)
    plain = check_scene(spec, ["m1", "m3"], LIMITS, b)
    assert check_scene(spec, ["m1", "m3"], LIMITS, b, _gt(7), 100) == plain + 7 * 96 + 4


def test_decode_kwargs_of_the_scene_postprocess_block():
    """decode_kwargs on the scenes' `postprocess:` block: the keyword arguments of the box decodes of VoxelPostprocessor,
    SceneGraph and LateFusionGraph, with a dir head (the `dir_args` correction) and without one (no correction)."""
    import scene_fixtures
    from heal_b200.data_utils.post_processor.voxel_postprocessor import decode_kwargs
    common = {"score_threshold": 0.2, "nms_threshold": 0.15, "order": "hwl", "gt_range": [-12.8, -12.8, -3, 12.8, 12.8, 1],
              "top": 1000}
    assert decode_kwargs(scene_fixtures.postprocess_params(), True) == {**common, "dir_offset": 0.7853, "num_bins": 2}
    assert decode_kwargs(scene_fixtures.postprocess_params(), False) == {**common, "dir_offset": 0.0, "num_bins": 2}
