"""Single-agent models and late fusion on the GPU: HeterModelLate / HeterPyramidSingle against the goldens made from the unmodified
reference, `forward_late` (one batched forward per modality) against the per-cav loop of the reference's inference_late_fusion,
heal_box_decode_nms_late against heal_box_decode_nms_multi, LateFusionGraph replayed for scenes with different poses, and the
reference's own callers (create_model, load_state_dict, inference_late_fusion / inference_no_fusion) driving the mirrors."""
import copy
import os
import sys
from collections import OrderedDict

import pytest
import torch

from oracle import efficientnet as oe
from oracle import golden, late, ref_shim

pytestmark = pytest.mark.gpu

MODELS = ("heter_model_late_m1", "heter_model_late_m2eff", "heter_pyramid_single_m1", "heter_pyramid_single_m2_convnext")
HEADS = ("cls_preds", "reg_preds", "dir_preds")


@pytest.fixture(autouse=True)
def _restore_precision():
    from heal_b200 import engine
    old = engine.PRECISION
    yield
    engine.set_precision(old)


def _cuda(d):
    return {k: (v.cuda() if torch.is_tensor(v) else _cuda(v) if isinstance(v, dict) else v) for k, v in d.items()}


def _model(name_or_args, sd=None, shapes=None):
    from heal_b200.models.heter_model_late import HeterModelLate
    from heal_b200.models.heter_pyramid_single import HeterPyramidSingle
    args = name_or_args
    cls = HeterModelLate if "layers_args" in str(args) else HeterPyramidSingle
    m = cls(copy.deepcopy(args)).eval()
    sd = sd if sd is not None else oe.state_dict_of(shapes or {k: tuple(v.shape) for k, v in m.state_dict().items()})
    r = m.load_state_dict(sd, strict=True)
    assert not r.missing_keys and not r.unexpected_keys
    return m.cuda()


def _inputs(name):
    return {"inputs_m1": late.lidar_cav(31)} if name.endswith("_m1") else {"inputs_m2": oe.cam_inputs()}


@pytest.mark.parametrize("prec,tol", [("tc32", 1e-3), ("bf16", 2.5e-2)])
@pytest.mark.parametrize("name", MODELS)
def test_mirror_vs_reference_golden(golden_dir, name, prec, tol):
    from heal_b200 import engine
    engine.set_precision(prec)
    g = golden.load(os.path.join(golden_dir, f"{name}_small.pt"))
    m = _model(g["args"], shapes=g["shapes"])
    with torch.no_grad():
        out = m(_cuda(_inputs(name)))
    assert sorted(out.keys()) == g["keys"]
    pairs = [(k, out[k], g["out"][k]) for k in HEADS]
    pairs += [(f"occ{i}", a, b) for i, (a, b) in enumerate(zip(out.get("occ_single_list", []), g["out"].get("occ_single_list", [])))]
    for k, a, ref in pairs:
        err = (a.cpu() - ref).abs().max().item()
        scale = max(ref.abs().max().item(), 1.0)
        print(f"{name} {prec}/{k}: max|ref|={scale:.3f} err={err:.3e}")
        assert a.shape == ref.shape and err < tol * scale, (k, err, scale)


def _mixed_late_args():
    a = late.late_args("m1")
    a["m2"] = late.late_args("m2eff")["m2"]
    return a


def _lidar_batch(seeds, anchors=None):
    return OrderedDict((f"cav{i}", {"inputs_m1": _cuda(late.lidar_cav(s)), "anchor_box": anchors,
                                    "transformation_matrix": torch.eye(4)}) for i, s in enumerate(seeds))


# Lidar cavs: bit-identical, the batched forward runs the same kernels on more images and no output element's reduction order
# depends on the batch size.  Camera cavs: the Lift-Splat-Shoot pooling (heal_lss_pool_sorted) sums each BEV cell's frustum points
# in 128-point chunks of the WHOLE batch's sorted points, so where a cell's points are cut into chunks (and so the order of its
# sum) moves with the points of the cavs before it; the image trunk and heads stay bit-identical.  Those cavs are held to the
# tc32 bar, 1e-3 of max(1, max|ref|).
@pytest.mark.parametrize("kind", ["late_m1", "late_mixed", "single_m1", "single_m2_convnext"])
def test_forward_late_equals_the_per_cav_loop(kind):
    from heal_b200 import engine
    engine.set_precision("tc32")
    if kind == "late_m1":
        m, batch = _model(late.late_args("m1")), _lidar_batch((21, 22, 23, 24, 25))
    elif kind == "single_m1":
        m, batch = _model(late.pyramid_single_args("m1")), _lidar_batch((21, 22, 23))
    else:
        m = _model(_mixed_late_args() if kind == "late_mixed" else late.pyramid_single_args("m2_convnext"))
        cams = [{"inputs_m2": _cuda(oe.cam_inputs(s))} for s in (53, 54)]
        if kind == "late_mixed":      # m2 cavs interleaved with m1 cavs: the copy path, and a contiguous m1 run
            lid = list(_lidar_batch((21, 22, 23)).values())
            batch = OrderedDict([("ego", cams[0]), ("a", lid[0]), ("b", cams[1]), ("c", lid[1]), ("d", lid[2])])
        else:
            batch = OrderedDict([("ego", cams[0]), ("a", cams[1])])
    with torch.no_grad():
        got = m.forward_late(batch)
        loop = OrderedDict((c, m(content)) for c, content in batch.items())
    assert list(got) == list(loop) == list(batch)
    for c in batch:
        assert sorted(got[c]) == sorted(loop[c]), c
        pairs = [(k, got[c][k], loop[c][k]) for k in HEADS]
        pairs += [(f"occ{i}", a, b) for i, (a, b) in enumerate(zip(got[c].get("occ_single_list", []), loop[c].get("occ_single_list", [])))]
        for k, a, b in pairs:
            d = (a - b).abs().max().item()
            if "inputs_m2" in batch[c]:
                print(f"forward_late {kind} camera cav {c} {k}: max|diff| {d:.3e}")
                assert d <= 1e-3 * max(1.0, b.abs().max().item()), (kind, c, k, d)
            else:
                assert torch.equal(a, b), (kind, c, k, d)


def _anchors_dev(params):
    from heal_b200.data_utils.post_processor.voxel_postprocessor import VoxelPostprocessor
    return torch.from_numpy(VoxelPostprocessor(params, False).generate_anchor_box()).float().cuda().contiguous()


def _late_vs_multi(params, cavs, anchors):
    from heal_b200 import ops
    dargs = params["dir_args"]
    kw = dict(dir_offset=dargs["dir_offset"], num_bins=dargs["num_bins"], order=params["order"], gt_range=params["gt_range"])
    thr, nms = params["target_args"]["score_threshold"], params["nms_thresh"]
    multi = ops.box_decode_nms_multi([{"cls": c["cls"].cuda(), "reg": c["reg"].cuda(), "dir": c["dir"].cuda(), "anchors": anchors,
                                       "transform": c["T"]} for c in cavs], thr, nms, **kw)
    T = torch.stack([torch.as_tensor(c["T"]).reshape(4, 4).float() for c in cavs]).cuda()
    stacked = ops.box_decode_nms_late(*(torch.cat([c[h] for c in cavs]).cuda() for h in ("cls", "reg", "dir")), anchors, T, thr, nms, **kw)
    fused = ops.to_act(torch.cat([torch.cat([c[h] for c in cavs]) for h in ("cls", "reg", "dir")], 1).cuda())
    A = cavs[0]["cls"].shape[1]
    viewed = ops.box_decode_nms_late(fused, fused, fused, anchors, T, thr, nms, coffsets=(0, A, 8 * A), **kw)
    torch.cuda.synchronize()
    k = int(multi.count.item())
    assert k > 0
    for b in (stacked, viewed):
        assert int(b.count.item()) == k
        assert torch.equal(b.boxes[:k], multi.boxes[:k]) and torch.equal(b.scores[:k], multi.scores[:k])
        assert torch.equal(b.stats, multi.stats)
    return multi.boxes[:k].cpu(), multi.scores[:k].cpu()


def test_late_decode_equals_multi_on_the_late2_golden(golden_dir):
    g = golden.load(os.path.join(golden_dir, "postprocess.pt"))
    c = g["multi"]["late2"]
    boxes, scores = _late_vs_multi(g["params"], c["cavs"], g["anchors"].float().cuda().contiguous())
    torch.testing.assert_close(scores, c["scores"], rtol=0, atol=1e-6)
    torch.testing.assert_close(boxes, c["boxes"], rtol=0, atol=1e-4)


def test_late_decode_equals_multi_on_the_scene_golden(golden_dir):
    g = golden.load(os.path.join(golden_dir, "late_fusion_scene_small.pt"))
    cavs = [{"cls": h["cls_preds"], "reg": h["reg_preds"], "dir": h["dir_preds"], "T": g["transforms"][c]} for c, h in g["heads"].items()]
    boxes, scores = _late_vs_multi(g["params"], cavs, _anchors_dev(g["params"]))
    assert boxes.shape == g["boxes"].shape
    torch.testing.assert_close(scores, g["scores"], rtol=0, atol=1e-6)
    torch.testing.assert_close(boxes, g["boxes"], rtol=0, atol=1e-4)


def _scene_model(g):
    sd = oe.state_dict_of(g["shapes"])
    sd["cls_head_m1.bias"] = sd["cls_head_m1.bias"] + g["cls_bias"]
    return _model(g["args"], sd=sd), sd


def _raw_scene(poses):
    """The scene golden's three clouds as raw points (voxelised on the GPU) under the given (x, y, yaw) poses."""
    out = OrderedDict()
    for i, (seed, p) in enumerate(zip(late.SCENE_SEEDS, poses)):
        pts = torch.from_numpy(late.scene_points(seed)).cuda()
        out["ego" if i == 0 else f"cav{i}"] = {
            "inputs_m1": {"points": pts, "agent_offsets": torch.tensor([0, pts.shape[0]], dtype=torch.int32, device="cuda")},
            "transformation_matrix": late.pose(*p).float()}
    return out


def _eager_boxes(m, scene, params, anchors):
    from heal_b200 import ops
    with torch.no_grad():
        heads = m.forward_late(scene)
    dargs = params["dir_args"]
    b = ops.box_decode_nms_multi([{"cls": h["cls_preds"], "reg": h["reg_preds"], "dir": h["dir_preds"], "anchors": anchors,
                                   "transform": scene[c]["transformation_matrix"]} for c, h in heads.items()],
                                 params["target_args"]["score_threshold"], params["nms_thresh"], dir_offset=dargs["dir_offset"],
                                 num_bins=dargs["num_bins"], order=params["order"], gt_range=params["gt_range"])
    k = int(b.count.item())
    return b.boxes[:k].clone(), b.scores[:k].clone()


def test_late_fusion_graph_replays_new_poses_and_matches_the_reference(golden_dir):
    from heal_b200 import engine
    from heal_b200.graph import LateFusionGraph
    engine.set_precision("tc32")
    g = golden.load(os.path.join(golden_dir, "late_fusion_scene_small.pt"))
    m, _ = _scene_model(g)
    params = g["params"]
    anchors = _anchors_dev(params)
    lg = LateFusionGraph(m, ["m1"] * 3, {"m1": 3 * 1500}, params)
    poses_b = ((0.0, 0.0, 0.0), (-6.0, 1.0, 80.0), (3.0, 5.0, 170.0))
    results = []
    for poses in (late.SCENE_POSES, poses_b, late.SCENE_POSES):
        scene = _raw_scene(poses)
        lg.load(scene)
        out = lg.replay()
        torch.cuda.synchronize()
        k = int(out.count.item())
        eb, es = _eager_boxes(m, scene, params, anchors)
        assert k == eb.shape[0] > 0
        assert torch.equal(out.boxes[:k], eb) and torch.equal(out.scores[:k], es)
        results.append((out.boxes[:k].cpu().clone(), out.scores[:k].cpu().clone()))
    assert results[0][0].shape != results[1][0].shape or not torch.equal(results[0][0], results[1][0])   # the poses moved the boxes
    assert torch.equal(results[0][0], results[2][0])
    print(f"LateFusionGraph: {lg.kernels_per_replay} kernels per replay, {results[0][0].shape[0]} boxes")
    # the golden's clouds were voxelised on the host by the reference's voxeliser; the graph voxelises them on the GPU
    b, s = results[0]
    assert b.shape == g["boxes"].shape, (b.shape, g["boxes"].shape)
    torch.testing.assert_close(s, g["scores"], rtol=0, atol=1e-4)
    torch.testing.assert_close(b, g["boxes"], rtol=0, atol=2e-3)


@pytest.fixture
def _isolate_opencood_modules():
    before = {k: v for k, v in sys.modules.items() if k.startswith(("opencood", "shapely"))}
    yield
    for k in [k for k in sys.modules if k.startswith(("opencood", "shapely"))]:
        del sys.modules[k]
    sys.modules.update(before)


def test_reference_callers_drive_the_late_path(golden_dir, _isolate_opencood_modules):
    """create_model on a Single/m1_pointpillar_pretrain.yaml-shaped hypes, load_state_dict, then inference_late_fusion and
    inference_no_fusion with the registry's GPU post-processor; the boxes equal the reference's (golden) and the oracle's."""
    if not ref_shim.available():
        pytest.skip("oracle/_ref not built")
    import types
    from unittest.mock import MagicMock
    from oracle import postprocess as opp
    sg = types.ModuleType("shapely.geometry")
    sg.Polygon = opp.QuadPolygon                  # shapely is absent: the stand-in the goldens pin the reference with
    sg.Point, sg.MultiPoint = MagicMock(), MagicMock()          # imported (unused on this path) by opencood/utils/camera_utils.py
    sh = types.ModuleType("shapely")
    sh.geometry = sg
    sys.modules["shapely"], sys.modules["shapely.geometry"] = sh, sg
    sys.modules.setdefault("opencood.utils.box_overlaps", MagicMock())
    ref_shim.install()
    from heal_b200 import engine, install
    engine.set_precision("tc32")
    done = install.install_into_opencood()
    assert {"opencood.models.heter_model_late", "opencood.models.heter_pyramid_single"} <= set(done)
    from opencood.tools.train_utils import create_model
    from opencood.tools import inference_utils
    g = golden.load(os.path.join(golden_dir, "late_fusion_scene_small.pt"))
    params = g["params"]
    model = create_model({"model": {"core_method": "heter_model_late", "args": copy.deepcopy(g["args"])}, "postprocess": params})
    assert type(model).__module__ == "heal_b200.models.heter_model_late"
    sd = oe.state_dict_of(g["shapes"])
    sd["cls_head_m1.bias"] = sd["cls_head_m1.bias"] + g["cls_bias"]
    r = model.load_state_dict(sd, strict=True)
    assert not r.missing_keys and not r.unexpected_keys
    model = model.cuda().eval()
    install.install_gpu_postprocessor()
    from opencood.data_utils.post_processor import build_postprocessor
    pp = build_postprocessor(copy.deepcopy(params), train=False)

    class Dataset:                     # late_heter_fusion_dataset.py:524-558 without the ground truth
        post_processor = pp

        def post_process(self, data_dict, output_dict):
            return (*self.post_processor.post_process(data_dict, output_dict), None)

        def post_process_no_fusion(self, data_dict, output_dict_ego):
            return (*self.post_processor.post_process(OrderedDict(ego=data_dict["ego"]), output_dict_ego), None)

    batch = late.scene_batch(torch.from_numpy(pp.generate_anchor_box()))
    batch = OrderedDict((c, dict(v, inputs_m1=_cuda(v["inputs_m1"]))) for c, v in batch.items())
    with torch.no_grad():
        ret = inference_utils.inference_late_fusion(batch, model, Dataset())
        ret_no = inference_utils.inference_no_fusion(batch, model, Dataset())
    assert ret["pred_box_tensor"].shape == g["boxes"].shape
    torch.testing.assert_close(ret["pred_score"].cpu(), g["scores"], rtol=0, atol=1e-4)
    torch.testing.assert_close(ret["pred_box_tensor"].cpu(), g["boxes"], rtol=0, atol=2e-3)
    ego = late.heter_model_late(sd, g["args"], late.scene_batch(None)["ego"])
    ref_b, ref_s = opp.post_process(ego["cls_preds"], ego["reg_preds"], ego["dir_preds"],
                                    torch.from_numpy(pp.generate_anchor_box()), batch["ego"]["transformation_matrix"], params)
    assert ret_no["pred_box_tensor"].shape == ref_b.shape
    torch.testing.assert_close(ret_no["pred_score"].cpu(), ref_s, rtol=0, atol=1e-4)
    torch.testing.assert_close(ret_no["pred_box_tensor"].cpu(), ref_b, rtol=0, atol=2e-3)
