"""GPU detection post-processing (heal_box_decode_nms through heal_b200.data_utils.post_processor.VoxelPostprocessor) against
(a) tests/golden/postprocess.pt, produced by the UNMODIFIED reference VoxelPostprocessor.post_process, and (b) the oracle on a
full-size 256 x 256 x 2 anchor map.  Integer results (how many boxes, which ones, in which order) must match exactly; corner
coordinates and scores are fp32 results of exp / sin / cos / sigmoid -> 1e-4 absolute on metres, 1e-6 on scores."""
import copy
import os

import numpy as np
import pytest
import torch

from oracle import golden

from oracle import make_golden
from oracle import postprocess as opp

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gold(golden_dir):
    return golden.load(os.path.join(golden_dir, "postprocess.pt"))


def _run_gpu(params, anchors, cls, reg, dirp, T):
    from heal_b200.data_utils.post_processor import build_postprocessor
    pp = build_postprocessor(copy.deepcopy(params), train=False)
    data = {"ego": {"transformation_matrix": T, "anchor_box": anchors}}
    out = {"ego": {"cls_preds": cls.cuda(), "reg_preds": reg.cuda(), "dir_preds": None if dirp is None else dirp.cuda()}}
    if dirp is None:
        del out["ego"]["dir_preds"]
    return pp, pp.post_process(data, out)


def test_anchor_box_equals_reference(gold):
    from heal_b200.data_utils.post_processor import build_postprocessor
    pp = build_postprocessor(copy.deepcopy(gold["params"]), train=False)
    assert np.array_equal(pp.generate_anchor_box(), gold["anchors"].numpy())


@pytest.mark.parametrize("case", ["dense", "sparse"])
def test_post_process_vs_reference_golden(gold, case):
    c = gold["cases"][case]
    pp, (boxes, scores) = _run_gpu(gold["params"], gold["anchors"], c["cls"], c["reg"], c["dir"], c["T"])
    assert boxes.shape == c["boxes"].shape, (boxes.shape, c["boxes"].shape)
    torch.testing.assert_close(scores.cpu(), c["scores"], rtol=0, atol=1e-6)
    torch.testing.assert_close(boxes.cpu(), c["boxes"], rtol=0, atol=1e-4)
    st = next(iter(pp._buffers.values())).stats.cpu().tolist()
    assert st[0] == int((torch.sigmoid(c["cls"]) > gold["params"]["target_args"]["score_threshold"]).sum())


def test_no_box_above_threshold_returns_none(gold):
    c = gold["cases"]["sparse"]
    _, (boxes, scores) = _run_gpu(gold["params"], gold["anchors"], c["cls"] - 20.0, c["reg"], c["dir"], c["T"])
    assert boxes is None and scores is None


def test_full_size_map_vs_oracle():
    """BASELINE config 2 geometry: +-102.4 m, 256 x 256 x 2 anchors, ~3 k boxes above the threshold (top-1000 cut active),
    no direction head on this one."""
    params = make_golden.postprocess_params(rng=(-102.4, -102.4, -3, 102.4, 102.4, 1))
    anchors = torch.from_numpy(opp.generate_anchor_box(params["anchor_args"], params["order"]))
    cls, reg, _, T = make_golden.postprocess_inputs(params, seed=11, logit_mean=-4.5)
    ref_b, ref_s = opp.post_process(cls.clone(), reg.clone(), None, anchors, T, params)
    _, (boxes, scores) = _run_gpu(params, anchors, cls, reg, None, T)
    assert boxes.shape == ref_b.shape and boxes.shape[0] > 100
    torch.testing.assert_close(scores.cpu(), ref_s, rtol=0, atol=1e-6)
    torch.testing.assert_close(boxes.cpu(), ref_b, rtol=0, atol=1e-4)


def test_model_heads_feed_the_postprocessor_without_copies(gold):
    """channels-last head outputs (what the engine produces) and contiguous NCHW tensors give the same boxes."""
    c = gold["cases"]["dense"]
    _, (b0, s0) = _run_gpu(gold["params"], gold["anchors"], c["cls"], c["reg"], c["dir"], c["T"])
    cl = lambda t: t.cuda().contiguous(memory_format=torch.channels_last)
    from heal_b200.data_utils.post_processor import build_postprocessor
    pp = build_postprocessor(copy.deepcopy(gold["params"]), train=False)
    b1, s1 = pp.post_process({"ego": {"transformation_matrix": c["T"], "anchor_box": gold["anchors"]}},
                             {"ego": {"cls_preds": cl(c["cls"]), "reg_preds": cl(c["reg"]), "dir_preds": cl(c["dir"])}})
    assert torch.equal(b0, b1) and torch.equal(s0, s1)


@pytest.mark.parametrize("case", ["late2", "iou"])
def test_late_fusion_and_iou_rescoring_vs_reference_golden(gold, case):
    """heal_box_decode_nms_multi: two cavs with their own cav->ego transforms (late fusion, one NMS over both box sets) and
    `iou_preds` rescoring, against the UNMODIFIED reference VoxelPostprocessor.post_process (tests/golden/postprocess.pt `multi`)."""
    from heal_b200.data_utils.post_processor import build_postprocessor
    c = gold["multi"][case]
    pp = build_postprocessor(copy.deepcopy(gold["params"]), train=False)
    names = ["ego"] + [f"cav{i}" for i in range(1, len(c["cavs"]))]
    data = {n: {"transformation_matrix": cav["T"], "anchor_box": gold["anchors"]} for n, cav in zip(names, c["cavs"])}
    out = {}
    for n, cav in zip(names, c["cavs"]):
        out[n] = {"cls_preds": cav["cls"].cuda(), "reg_preds": cav["reg"].cuda(), "dir_preds": cav["dir"].cuda()}
        if "iou" in cav:
            out[n]["iou_preds"] = cav["iou"].cuda()
    boxes, scores = pp.post_process(data, out)
    assert boxes.shape == c["boxes"].shape, (boxes.shape, c["boxes"].shape)
    torch.testing.assert_close(scores.cpu(), c["scores"], rtol=0, atol=1e-6)
    torch.testing.assert_close(boxes.cpu(), c["boxes"], rtol=0, atol=1e-4)
