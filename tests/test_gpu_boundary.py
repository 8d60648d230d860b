"""Drop-in boundary, end to end through the REFERENCE's own callers (SURVEY.md 8b): with the unmodified `opencood` package of
oracle/_ref importable and `heal_b200.install.install_into_opencood()` applied,

  opencood.tools.train_utils.create_model(hypes)                 (tools/train_utils.py:141-174)  builds the heal_b200 class,
  model.load_state_dict(<reference-keyed checkpoint>, strict)    loads with zero missing / unexpected keys,
  opencood.tools.inference_utils.inference_intermediate_fusion   (tools/inference_utils.py:142) = model(batch['ego']) +
        dataset.post_process -> the registry's post-processor     (install_gpu_postprocessor: a subclass of the reference class)

and the boxes equal the oracle's (oracle.nets heads -> oracle.postprocess) on the same scene."""
import copy
import os
import sys
import types

import numpy as np
import pytest
import torch

from oracle import golden

from oracle import make_golden, nets, ref_shim
from oracle import postprocess as opp
from workloads import procedural

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _isolate_opencood_modules():
    """install_into_opencood() aliases heal_b200 mirrors under `opencood.models.*` in sys.modules; other test modules import the
    UNMODIFIED reference under those names (oracle.ref_runner), so everything opencood / shapely is restored afterwards."""
    before = {k: v for k, v in sys.modules.items() if k.startswith(("opencood", "shapely"))}
    yield
    for k in [k for k in sys.modules if k.startswith(("opencood", "shapely"))]:
        del sys.modules[k]
    sys.modules.update(before)


def _install_reference_with_quad_polygon():
    from unittest.mock import MagicMock
    sg = types.ModuleType("shapely.geometry")
    sg.Polygon = opp.QuadPolygon                  # shapely is absent: same stand-in make_golden.py pins the reference with
    sg.Point, sg.MultiPoint = MagicMock(), MagicMock()          # imported (unused on this path) by opencood/utils/camera_utils.py
    sh = types.ModuleType("shapely")
    sh.geometry = sg
    sys.modules["shapely"], sys.modules["shapely.geometry"] = sh, sg
    sys.modules.setdefault("opencood.utils.box_overlaps", MagicMock())
    ref_shim.install()


def test_reference_callers_drive_the_b200_path(golden_dir):
    if not ref_shim.available():
        pytest.skip("oracle/_ref not built")
    _install_reference_with_quad_polygon()
    from heal_b200 import install
    done = install.install_into_opencood()
    assert "opencood.models.heter_pyramid_collab" in done
    from opencood.tools.train_utils import create_model
    from opencood.tools import inference_utils
    g = golden.load(os.path.join(golden_dir, "heter_pyramid_collab_small.pt"))
    rng_ = list(g["args"]["lidar_range"])
    params = make_golden.postprocess_params(rng=tuple(rng_))
    params["target_args"]["score_threshold"] = 0.5
    hypes = {"model": {"core_method": "heter_pyramid_collab", "args": copy.deepcopy(g["args"])}, "postprocess": params}
    model = create_model(hypes)
    assert type(model).__module__ == "heal_b200.models.heter_pyramid_collab"
    sd = procedural.make_state_dict(g["shapes"])                 # g["shapes"] = the UNMODIFIED reference model's key/shape table
    res = model.load_state_dict(sd, strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    model = model.cuda().eval()

    cls = install.install_gpu_postprocessor()
    from opencood.data_utils.post_processor import build_postprocessor
    from opencood.data_utils.post_processor.voxel_postprocessor import VoxelPostprocessor as RefPP
    pp = build_postprocessor(copy.deepcopy(params), train=False)
    assert isinstance(pp, cls) and isinstance(pp, RefPP)
    for name in ("generate_gt_bbx", "generate_label", "generate_object_center", "collate_batch", "generate_anchor_box"):
        assert callable(getattr(pp, name)), name

    class Dataset:                                                # intermediate_heter_fusion_dataset.py:760-783, verbatim logic
        post_processor = pp

        def post_process(self, data_dict, output_dict):
            pred_box_tensor, pred_score = self.post_processor.post_process(data_dict, output_dict)
            gt_box_tensor = self.post_processor.generate_gt_bbx(data_dict)
            return pred_box_tensor, pred_score, gt_box_tensor

    data = g["data"]
    anchors = torch.from_numpy(pp.generate_anchor_box())
    gt = torch.zeros(1, 100, 7)
    gt[0, 0] = torch.tensor([2.0, 1.0, -1.0, 1.6, 1.6, 3.9, 0.3])
    gt[0, 1] = torch.tensor([-4.0, 3.0, -1.0, 1.6, 1.6, 3.9, 1.2])
    mask = torch.zeros(1, 100)
    mask[0, :2] = 1
    ego = {"inputs_m1": {k: v.cuda() for k, v in data["inputs_m1"].items()}, "agent_modality_list": data["agent_modality_list"],
           "record_len": data["record_len"], "pairwise_t_matrix": data["pairwise_t_matrix"].cuda(),
           "anchor_box": anchors, "transformation_matrix": torch.eye(4), "transformation_matrix_clean": torch.eye(4),
           "object_bbx_center": gt, "object_bbx_mask": mask, "object_ids": [11, 12]}
    with torch.no_grad():
        ret = inference_utils.inference_intermediate_fusion({"ego": ego}, model, Dataset())
    assert ret["gt_box_tensor"].shape == (2, 8, 3)
    # oracle: CPU network + CPU post-processing of the same scene
    with torch.no_grad():
        ref_heads = nets.heter_pyramid_collab(sd, g["args"], copy.deepcopy(data))
    ref_b, ref_s = opp.post_process(ref_heads["cls_preds"], ref_heads["reg_preds"], ref_heads["dir_preds"], anchors, torch.eye(4), params)
    if ref_b is None:
        assert ret["pred_box_tensor"] is None
        return
    assert ret["pred_box_tensor"].shape == ref_b.shape, (ret["pred_box_tensor"].shape, ref_b.shape)
    torch.testing.assert_close(ret["pred_score"].cpu(), ref_s, rtol=0, atol=1e-4)
    torch.testing.assert_close(ret["pred_box_tensor"].cpu(), ref_b, rtol=0, atol=2e-3)


def test_postprocessor_subclass_falls_back_to_the_reference_for_cpu_and_late_fusion(golden_dir):
    """CPU tensors (and more than one cav) are not GPU-eligible: the installed class answers with the reference implementation."""
    if not ref_shim.available():
        pytest.skip("oracle/_ref not built")
    _install_reference_with_quad_polygon()
    from heal_b200 import install
    cls = install.install_gpu_postprocessor()
    gold = golden.load(os.path.join(golden_dir, "postprocess.pt"))
    pp = cls(copy.deepcopy(gold["params"]), train=False)
    c = gold["cases"]["sparse"]
    data = {"ego": {"transformation_matrix": c["T"], "anchor_box": gold["anchors"]}}
    out = {"ego": {"cls_preds": c["cls"].clone(), "reg_preds": c["reg"].clone(), "dir_preds": c["dir"].clone()}}
    boxes, scores = pp.post_process(data, out)                    # CPU tensors -> reference path
    assert torch.equal(boxes, c["boxes"]) and torch.equal(scores, c["scores"])
    out_gpu = {"ego": {k: v.cuda() for k, v in out["ego"].items()}}
    b2, s2 = pp.post_process(data, out_gpu)                       # CUDA tensors -> heal_box_decode_nms
    torch.testing.assert_close(b2.cpu(), c["boxes"], rtol=0, atol=1e-4)
