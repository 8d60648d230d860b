"""Golden vectors for the single-agent models and late fusion (TEST INFRASTRUCTURE ONLY): the UNMODIFIED reference
HeterModelLate, HeterPyramidSingle, VoxelPostprocessor and inference_utils.inference_late_fusion run on the CPU with procedural
weights (the camera trunk over the `efficientnet_pytorch` stand-in of oracle/efficientnet.py).

    python -m oracle.make_golden_late        (needs the reference package: oracle/_ref or HEAL_REFERENCE_ROOT)

Writes under tests/golden/ (inputs are regenerated from seeds by oracle/late.py, not stored):
  heter_model_late_m1_small.pt.xz                 PointPillars (Single/m1_pointpillar_pretrain.yaml shapes, small range)
  heter_model_late_m2eff_small.pt.xz              LSS + EfficientNet, camera map center-cropped 48 -> 32
  heter_pyramid_single_m1_small.pt.xz             identity aligner
  heter_pyramid_single_m2_convnext_small.pt.xz    LSS + EfficientNet camera agent with a ConvNeXt aligner
  late_fusion_scene_small.pt.xz                   three m1 cavs with different poses: every cav's heads and the boxes and
                                                  scores of the reference's inference_late_fusion
SECOND (m3) is not among them: the reference's VoxelBackBone8x needs spconv, which the CPU build does not have."""
import copy
import os
import sys
import types
from unittest.mock import MagicMock

import torch

from oracle import efficientnet

efficientnet.install()          # before ref_shim.install(): the stand-in takes the place of the MagicMock stub

from oracle import golden, late, make_golden, ref_shim  # noqa: E402
from oracle.make_golden_coalign import _cuda_moves_stay_on_cpu  # noqa: E402

OUT = make_golden.OUT
HEAD_KEYS = ("cls_preds", "reg_preds", "dir_preds")
SCENE_CLS_BIAS = 2.0     # added to the procedural cls_head bias so that a few hundred anchors pass the 0.2 score threshold


def _inputs(mod):
    return {"inputs_m1": late.lidar_cav(31)} if mod == "m1" else {"inputs_m2": efficientnet.cam_inputs()}


def _build(cls, args):
    with _cuda_moves_stay_on_cpu():
        m = cls(copy.deepcopy(args)).eval()
    shapes = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    m.load_state_dict(efficientnet.state_dict_of(shapes), strict=True)
    return m, shapes


def model_goldens():
    from opencood.models.heter_model_late import HeterModelLate
    from opencood.models.heter_pyramid_single import HeterPyramidSingle
    for name, cls, args, mod in (("heter_model_late_m1", HeterModelLate, late.late_args("m1"), "m1"),
                                 ("heter_model_late_m2eff", HeterModelLate, late.late_args("m2eff"), "m2"),
                                 ("heter_pyramid_single_m1", HeterPyramidSingle, late.pyramid_single_args("m1"), "m1"),
                                 ("heter_pyramid_single_m2_convnext", HeterPyramidSingle, late.pyramid_single_args("m2_convnext"), "m2")):
        m, shapes = _build(cls, args)
        with torch.no_grad():
            out = m(copy.deepcopy(_inputs(mod)))
        keep = {k: out[k] for k in HEAD_KEYS}
        if "occ_single_list" in out:
            keep["occ_single_list"] = list(out["occ_single_list"])
        golden.save({"args": args, "shapes": shapes, "out": keep, "keys": sorted(out.keys())},
                    os.path.join(OUT, f"{name}_small.pt"))
        print(name, {k: tuple(v.shape) for k, v in out.items() if torch.is_tensor(v)}, float(out["cls_preds"].abs().max()))


def scene_golden():
    """inference_late_fusion over three m1 cavs, through a dataset stand-in whose post_process is the late dataset's
    (late_heter_fusion_dataset.py:524-548) minus the ground truth."""
    from oracle import postprocess as opp
    sg = types.ModuleType("shapely.geometry")
    sg.Polygon = opp.QuadPolygon
    sg.Point = sg.MultiPoint = MagicMock()     # imported by opencood.utils.camera_utils, unused on this path
    sh = types.ModuleType("shapely")
    sh.geometry = sg
    sys.modules["shapely"], sys.modules["shapely.geometry"] = sh, sg
    sys.modules.setdefault("opencood.utils.box_overlaps", MagicMock())      # cython, training labels only
    for k in [k for k in sys.modules if k.startswith("opencood.utils.common_utils") or k.startswith("opencood.utils.box_utils")]:
        del sys.modules[k]
    ref_shim.install()
    from opencood.models.heter_model_late import HeterModelLate
    from opencood.data_utils.post_processor.voxel_postprocessor import VoxelPostprocessor
    from opencood.tools import inference_utils
    args = late.late_args("m1")
    m, shapes = _build(HeterModelLate, args)
    with torch.no_grad():
        m.cls_head_m1.bias += SCENE_CLS_BIAS
    params = make_golden.postprocess_params(rng=late.SMALL_RANGE)
    pp = VoxelPostprocessor(copy.deepcopy(params), train=False)
    anchors = torch.from_numpy(pp.generate_anchor_box())

    class Dataset:
        def post_process(self, data_dict, output_dict):
            boxes, scores = pp.post_process(data_dict, output_dict)
            return boxes, scores, None

    batch = late.scene_batch(anchors)
    heads = {}
    with torch.no_grad():
        for cav, content in batch.items():
            heads[cav] = {k: v for k, v in m(copy.deepcopy(content)).items() if k in HEAD_KEYS}
        res = inference_utils.inference_late_fusion(copy.deepcopy(batch), m, Dataset())
    golden.save({"args": args, "shapes": shapes, "cls_bias": SCENE_CLS_BIAS, "params": params, "anchors": anchors,
                 "transforms": {c: v["transformation_matrix"] for c, v in batch.items()}, "heads": heads,
                 "boxes": res["pred_box_tensor"], "scores": res["pred_score"]}, os.path.join(OUT, "late_fusion_scene_small.pt"))
    print("late_fusion_scene_small: kept", None if res["pred_box_tensor"] is None else tuple(res["pred_box_tensor"].shape))


def main():
    ref_shim.install()
    torch.set_num_threads(8)
    if "--scene-only" not in sys.argv:
        model_goldens()
    scene_golden()
    for f in sorted(os.listdir(OUT)):
        if f.startswith(("heter_model_late", "heter_pyramid_single", "late_fusion")):
            print(f, os.path.getsize(os.path.join(OUT, f)) // 1024, "KiB")


if __name__ == "__main__":
    main()
