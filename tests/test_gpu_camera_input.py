"""heal_camera_input on the GPU: both output layouts bit-equal to oracle/camera_input.py (the numpy restatement pinned to PIL and
torchvision by tests/test_camera_input_cpu.py) and to the reference's own golden, and the camera encoders, a C4-shaped
HeterPyramidCollab and the captured graphs fed raw uint8 frames bit-identical to the same models fed the normalised images."""
import copy
import os
from collections import OrderedDict

import numpy as np
import pytest
import torch

from oracle import camera_input as oci
from oracle import efficientnet as oe
from oracle import golden, late, procedural

pytestmark = pytest.mark.gpu

# (frame H0 x W0, resize_dims (W, H), crop box, frames in one launch): tests/test_camera_input_cpu.py's cases
CASES = [
    ((600, 800), (512, 384), (0, -10, 512, 374), 3),
    ((600, 800), (448, 336), (0, -9, 448, 327), 3),
    ((1080, 1920), (512, 288), (0, -8, 512, 280), 2),
    ((600, 800), (704, 528), (0, 258, 704, 514), 3),
    ((50, 70), (134, 96), (3, -5, 120, 91), 9),
    ((37, 53), (29, 21), (1, 2, 28, 19), 9),
    ((40, 56), (56, 24), (4, 0, 52, 24), 9),
    ((40, 56), (32, 40), (0, 4, 32, 36), 9),
    ((33, 47), (40, 24), (-5, 0, 35, 24), 9),
    ((33, 47), (40, 24), (8, 0, 48, 24), 9),
    ((33, 47), (40, 24), (0, -6, 40, 18), 9),
    ((33, 47), (40, 24), (0, 8, 40, 32), 9),
    ((33, 47), (40, 24), (-9, -7, 49, 33), 9),
]
CONF_RAW = {"H": 600, "W": 800, "bot_pct_lim": [0.0, 0.05]}


@pytest.fixture(autouse=True)
def _restore_precision():
    from heal_b200 import engine
    old = engine.PRECISION
    yield
    engine.set_precision(old)


def _plan(H0, W0, dims, box):
    from heal_b200.data_utils.camera_input import CameraPlan
    return CameraPlan(H0, W0, (box[3] - box[1], box[2] - box[0]), 1.0, dims, box, torch.eye(2), torch.zeros(2))


def _frames(n, H0, W0, seed):
    return np.random.default_rng(seed).integers(0, 256, (n, H0, W0, 3), dtype=np.uint8)


def _bits_equal(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


@pytest.mark.parametrize("case", range(len(CASES)))
def test_both_layouts_equal_the_oracle_and_repeat(case):
    from heal_b200 import ops
    (H0, W0), dims, box, n = CASES[case]
    f = _frames(n, H0, W0, 100 + case)
    ref = torch.from_numpy(np.stack([oci.camera_input(x, dims, box) for x in f]))
    plan = _plan(H0, W0, dims, box)
    frames = torch.from_numpy(f).cuda()
    a = ops.camera_input(frames, plan, "nchw")
    a2 = ops.camera_input(frames, plan, "nchw")
    torch.cuda.synchronize()
    assert _bits_equal(a.cpu(), ref), f"nchw: {(a.cpu() != ref).sum().item()} values differ"
    assert _bits_equal(a, a2)
    fH, fW = plan.final_dim
    if fH % 8 == 0 and fW % 8 == 0:
        s = ops.camera_input(frames, plan, "s2d")
        s2 = ops.camera_input(frames, plan, "s2d")
        torch.cuda.synchronize()
        assert (s.fmt, s.N, s.H, s.W, s.C) == ("f32", n, fH // 4, fW // 4, 64)
        ref_s = torch.from_numpy(np.stack([oci.to_s2d(r.numpy()) for r in ref]))
        assert _bits_equal(s.t.cpu(), ref_s)
        assert _bits_equal(s.t, s2.t)
        # the layout the ResNet-101 stem built before: zeros, copy, pixel_unshuffle, to_act
        x4 = torch.zeros((n, 4, fH, fW), device="cuda")
        x4[:, :3] = a
        assert _bits_equal(ops.to_act(torch.nn.functional.pixel_unshuffle(x4, 4)).t, s.t)


def test_reference_golden(golden_dir):
    from heal_b200 import ops
    from heal_b200.data_utils.camera_input import inference_plan
    g = torch.load(os.path.join(golden_dir, "camera_input.pt"))
    assert len(g["cases"]) == 3
    for c in g["cases"]:
        frames = c["frames"]
        n, H0, W0, _ = frames.shape
        plan = inference_plan(c["conf"], H0, W0)
        assert (plan.resize_dims, plan.crop) == (c["resize_dims"], c["crop"])
        assert torch.equal(plan.post_rot, c["post_rot"]) and torch.equal(plan.post_tran, c["post_tran"])
        got = ops.camera_input(frames.cuda(), plan, "nchw").cpu()
        assert _bits_equal(got, c["imgs"]), (c["conf"], (got != c["imgs"]).sum().item())
        s = ops.camera_input(frames.cuda(), plan, "s2d").t.cpu()
        assert _bits_equal(s, torch.from_numpy(np.stack([oci.to_s2d(x.numpy()) for x in c["imgs"]])))


def _normalised(frames_u8, plan):
    """(B, N, H0, W0, 3) uint8 -> (B, N, 3, fH, fW) fp32 through the oracle, as the reference's DataLoader makes them."""
    B, N = frames_u8.shape[:2]
    out = [oci.camera_input(f, plan.resize_dims, plan.crop) for f in frames_u8.reshape(B * N, *frames_u8.shape[2:])]
    return torch.from_numpy(np.stack(out)).view(B, N, 3, *plan.final_dim)


def _cam_batch(B, N, H0, W0, plan, seed):
    from workloads import synth
    fH, fW = plan.final_dim
    rots, trans, intr, _, _ = [torch.from_numpy(a) for a in synth.camera_rig(B, N, fH, fW)]
    f = _frames(B * N, H0, W0, seed).reshape(B, N, H0, W0, 3)
    raw = {"imgs": torch.from_numpy(f), "rots": rots, "trans": trans, "intrins": intr,
           "post_rots": plan.post_rot3().expand(B, N, 3, 3).contiguous(), "post_trans": plan.post_tran3().expand(B, N, 3).contiguous()}
    return raw, dict(raw, imgs=_normalised(f, plan))


def _cuda(d):
    return {k: (v.cuda() if torch.is_tensor(v) else _cuda(v) if isinstance(v, dict) else v) for k, v in d.items()}


def _lss(cfg):
    from heal_b200.models.heter_encoders import LiftSplatShoot
    m = LiftSplatShoot(copy.deepcopy(cfg)).eval()
    m.load_state_dict(oe.state_dict_of({k: tuple(v.shape) for k, v in m.state_dict().items()}), strict=True)
    return m.cuda()


def _eff_cfg():
    cfg = oe.lss_cfg()
    cfg["data_aug_conf"].update({"H": 90, "W": 160, "bot_pct_lim": [0.0, 0.05]})   # 90x160 -> 72x128, crop rows 6 .. 70
    return cfg


def _resnet_cfg():
    from workloads import configs as wcfg
    cfg = wcfg.lss_encoder_args((256, 704))
    cfg["data_aug_conf"].update(CONF_RAW)                                         # C4: 600x800 -> 528x704, crop rows 258 .. 514
    return cfg


@pytest.mark.parametrize("prec", ["tc32", "bf16", "fp32"])
@pytest.mark.parametrize("encoder", ["EfficientNet", "Resnet101"])
def test_lss_from_raw_frames_equals_lss_from_normalised_images(encoder, prec):
    from heal_b200 import engine
    engine.set_precision(prec)
    cfg = _eff_cfg() if encoder == "EfficientNet" else _resnet_cfg()
    m = _lss(cfg)
    conf = cfg["data_aug_conf"]
    H0, W0 = (90, 160) if encoder == "EfficientNet" else (600, 800)
    plan = m.camera_plan(H0, W0)
    raw, ref = _cam_batch(2 if encoder == "EfficientNet" else 1, 2, H0, W0, plan, 7)
    with torch.no_grad():
        a = m({"inputs_m2": _cuda(raw)}, "m2")
        b = m({"inputs_m2": _cuda(ref)}, "m2")
    torch.cuda.synchronize()
    assert plan.final_dim == tuple(conf["final_dim"])
    assert a.abs().sum().item() > 0 and _bits_equal(a, b), (a - b).abs().max().item()


def test_c4_heter_pyramid_collab_from_raw_frames():
    """configs[3] shapes: agents [PointPillars, LSS-ResNet101 4 x 600x800 frames, LSS], bf16 as bench.py runs C4."""
    from heal_b200 import engine, synth
    from heal_b200.models.heter_pyramid_collab import HeterPyramidCollab
    from workloads import configs as wcfg
    engine.set_precision("bf16")
    args = wcfg.c4_args()
    args["m2"]["encoder_args"]["data_aug_conf"].update(CONF_RAW)
    m = HeterPyramidCollab(copy.deepcopy(args)).eval()
    m.load_state_dict(procedural.make_state_dict(procedural.shapes_of(m)), strict=True)
    m = m.cuda()
    sc = synth.scene(323, n_agents=3, max_cav=5, rings=32, azimuth=512)
    cloud = torch.from_numpy(sc["points"][0]).cuda()
    plan = m.encoder_m2.camera_plan(600, 800)
    raw, ref = _cam_batch(2, 4, 600, 800, plan, 11)
    outs = []
    for cam in (raw, ref):
        with torch.no_grad():
            outs.append(m({"inputs_m1": {"points": cloud, "agent_offsets": torch.tensor([0, cloud.shape[0]], dtype=torch.int32).cuda()},
                           "inputs_m2": _cuda(cam), "agent_modality_list": ["m1", "m2", "m2"], "record_len": torch.tensor([3]),
                           "pairwise_t_matrix": torch.from_numpy(sc["pairwise_t_matrix"]).cuda()}))
    torch.cuda.synchronize()
    for k in ("cls_preds", "reg_preds", "dir_preds"):
        assert _bits_equal(outs[0][k], outs[1][k]), k


def test_raw_frame_encoder_captured_with_graphed_call_replays_equal_to_eager():
    from heal_b200 import engine
    from heal_b200.graph import GraphedCall
    engine.set_precision("bf16")
    cfg = _resnet_cfg()
    m = _lss(cfg)
    plan = m.camera_plan(600, 800)
    raw, _ = _cam_batch(1, 4, 600, 800, plan, 21)
    spec = {k: (tuple(v.shape), v.dtype) for k, v in raw.items()}
    gc = GraphedCall(lambda d: m(d, "m2"), spec, lambda bufs: {"inputs_m2": bufs}, torch.device("cuda"), init=raw)
    for seed in (22, 23):
        nxt, _ = _cam_batch(1, 4, 600, 800, plan, seed)
        gc.load(**_cuda(nxt))
        out = gc.replay()
        with torch.no_grad():
            eager = m({"inputs_m2": _cuda(nxt)}, "m2")
        torch.cuda.synchronize()
        assert _bits_equal(out, eager), seed
    print(f"raw-frame LSS-ResNet101 graph: {gc.kernels_per_replay} kernels per replay")


def test_late_fusion_graph_with_raw_frames_equals_eager_and_the_normalised_graph(golden_dir):
    from heal_b200 import engine, ops
    from heal_b200.graph import LateFusionGraph
    from heal_b200.models.heter_model_late import HeterModelLate
    from heal_b200.data_utils.post_processor.voxel_postprocessor import VoxelPostprocessor
    engine.set_precision("tc32")
    params = golden.load(os.path.join(golden_dir, "late_fusion_scene_small.pt"))["params"]
    args = late.late_args("m2eff")
    args["m2"]["encoder_args"]["data_aug_conf"].update({"H": 90, "W": 160, "bot_pct_lim": [0.0, 0.05]})
    m = HeterModelLate(copy.deepcopy(args)).eval()
    sd = oe.state_dict_of({k: tuple(v.shape) for k, v in m.state_dict().items()})
    for k in [k for k in sd if k.startswith("cls_head") and k.endswith("bias")]:
        sd[k] = sd[k] + 3.0                                                        # enough scores over the threshold to keep boxes
    m.load_state_dict(sd, strict=True)
    m = m.cuda()
    plan = m.encoder_m2.camera_plan(90, 160)
    raw_g = LateFusionGraph(m, ["m2", "m2"], {"m2": (2, 90, 160, torch.uint8)}, params)
    ref_g = LateFusionGraph(m, ["m2", "m2"], {"m2": (2, 64, 128)}, params)
    anchors = torch.from_numpy(VoxelPostprocessor(params, False).generate_anchor_box()).float().cuda().contiguous()
    for seed in (31, 32):
        raw_scene, ref_scene = OrderedDict(), OrderedDict()
        for i, p in enumerate(((0.0, 0.0, 0.0), (3.0, -2.0, 40.0))):
            raw, ref = _cam_batch(1, 2, 90, 160, plan, seed + 10 * i)
            T = late.pose(*p).float()
            raw_scene[f"cav{i}"] = {"inputs_m2": _cuda(raw), "transformation_matrix": T}
            ref_scene[f"cav{i}"] = {"inputs_m2": _cuda(ref), "transformation_matrix": T}
        raw_g.load(raw_scene)
        a = raw_g.replay()
        ref_g.load(ref_scene)
        b = ref_g.replay()
        torch.cuda.synchronize()
        k = int(a.count.item())
        assert k == int(b.count.item()) > 0
        assert torch.equal(a.boxes[:k], b.boxes[:k]) and torch.equal(a.scores[:k], b.scores[:k])
        with torch.no_grad():
            heads = m.forward_late(raw_scene)
        dargs = params["dir_args"]
        e = ops.box_decode_nms_multi([{"cls": h["cls_preds"], "reg": h["reg_preds"], "dir": h["dir_preds"], "anchors": anchors,
                                       "transform": raw_scene[c]["transformation_matrix"]} for c, h in heads.items()],
                                     params["target_args"]["score_threshold"], params["nms_thresh"], dir_offset=dargs["dir_offset"],
                                     num_bins=dargs["num_bins"], order=params["order"], gt_range=params["gt_range"])
        assert int(e.count.item()) == k
        assert torch.equal(a.boxes[:k], e.boxes[:k]) and torch.equal(a.scores[:k], e.scores[:k])
    assert plan.final_dim == (64, 128)
