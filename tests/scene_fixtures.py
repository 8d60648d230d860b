"""Small mixed-modality scenes for the SceneGraph / heal_agent_stack tests: model arguments at the goldens' sizes (lidar range
+-12.8 m, 64 x 64 pillars, 32 x 32 fusion map), procedural weights and seeded raw clouds, camera rigs and images."""
import copy

import numpy as np
import torch

from oracle import make_golden, procedural
from oracle import efficientnet as oe

RANGE = make_golden.SMALL_RANGE
CONVNEXT = {"core_method": "convnext", "spatial_align": False, "args": {"num_of_blocks": 3, "dim": 64}}
CAMS, IMG_H, IMG_W = 2, 64, 128
FRAME_H, FRAME_W = 90, 160

AML = {
    "c4": ["m1", "m2", "m2"],                              # PointPillars + LSS-ResNet101, camera map zero-padded
    "four": ["m1", "m2", "m3", "m4", "m1"],                # PointPillars, LSS-EfficientNet (cropped), SECOND, LSS-ResNet101 (padded)
    "baseline": ["m2", "m1", "m2"],                        # HeterModelBaseline att: LSS-ResNet101 (padded) + PointPillars
}
LIDAR_CAPACITY = 4 * 2200
SECOND_CAPACITY = 8192


def _raw_frames(enc):
    """data_aug_conf of 90 x 160 raw frames (resized to 72 x 128, rows 6 .. 70 kept), so the encoder also takes uint8 frames."""
    enc["data_aug_conf"].update({"H": FRAME_H, "W": FRAME_W, "bot_pct_lim": [0.0, 0.05]})
    return enc


def _resnet_cam(half=6.4, C=64):
    c = make_golden.lss_small_cfg()
    c["grid_conf"]["xbound"] = [-half, half, 0.4]
    c["grid_conf"]["ybound"] = [-half, half, 0.4]
    c["img_features"] = C
    return c


def _cam_block(enc, backbone, **extra):
    return {"core_method": "lift_splat_shoot", "sensor_type": "camera", "encoder_args": _raw_frames(enc),
            "camera_mask_args": {"grid_conf": copy.deepcopy(enc["grid_conf"])}, "backbone_args": backbone, **extra}


def collab_args(kind):
    a = make_golden.small_model_args()
    if kind == "c4":
        a["m2"] = _cam_block(_resnet_cam(), {"layer_nums": [3], "layer_strides": [2], "num_filters": [64], "inplanes": 64},
                             aligner_args={"core_method": "identity"})
        return a
    eff = oe.lss_cfg()
    eff["grid_conf"]["xbound"] = [-19.2, 19.2, 0.4]       # 96 cells -> 48 after the backbone -> center-cropped to 32
    eff["grid_conf"]["ybound"] = [-19.2, 19.2, 0.4]
    eff["img_features"] = 64
    a["m1"]["aligner_args"] = copy.deepcopy(CONVNEXT)
    a["m2"] = _cam_block(eff, {"layer_nums": [3], "layer_strides": [2], "num_filters": [64], "inplanes": 64},
                         aligner_args=copy.deepcopy(CONVNEXT))
    a["m3"] = {"core_method": "second", "sensor_type": "lidar",
               "encoder_args": {"voxel_size": [0.1, 0.1, 0.1], "lidar_range": list(RANGE), "mean_vfe": {"num_point_features": 4},
                                "spconv": {"num_features_in": 4, "num_features_out": 64}, "map2bev": {"feature_num": 128}},
               "backbone_args": {"layer_nums": [3], "layer_strides": [1], "num_filters": [64], "inplanes": 128},
               "aligner_args": copy.deepcopy(CONVNEXT)}
    a["m4"] = _cam_block(_resnet_cam(), {"layer_nums": [3], "layer_strides": [2], "num_filters": [64], "inplanes": 64},
                         aligner_args=copy.deepcopy(CONVNEXT))
    return a


def baseline_args():
    a = make_golden.baseline_att_args()
    a["m2"] = _cam_block(_resnet_cam(), copy.deepcopy(a["m1"]["backbone_args"]), shrink_header=copy.deepcopy(a["m1"]["shrink_header"]))
    return a


def model(kind):
    from heal_b200.models.heter_pyramid_collab import HeterPyramidCollab
    from heal_b200.models.heter_model_baseline import HeterModelBaseline
    m = (HeterModelBaseline(baseline_args()) if kind == "baseline" else HeterPyramidCollab(collab_args(kind))).eval()
    m.load_state_dict(oe.state_dict_of(procedural.shapes_of(m)), strict=True)
    return m.cuda()


def baseline_camera_model():
    return model("baseline")


def _cloud(rng, n):
    return np.concatenate([rng.uniform(-14, 14, (n, 2)), rng.uniform(-3.5, 1.5, (n, 1)), rng.uniform(0, 1, (n, 1))],
                          1).astype(np.float32)


def scene_batch(kind, seed, raw=False):
    """The collated ego batch of one scene on the GPU: raw clouds (point counts vary with the seed), poses, camera rigs and
    fp32 images or, with `raw`, uint8 (H0, W0, 3) frames."""
    from workloads import synth
    aml = AML[kind]
    rng = np.random.default_rng(100 + seed)
    batch = {"agent_modality_list": list(aml), "record_len": torch.tensor([len(aml)])}
    for m in dict.fromkeys(aml):
        k = aml.count(m)
        sensor = "camera" if (kind, m) in {("c4", "m2"), ("four", "m2"), ("four", "m4"), ("baseline", "m2")} else "lidar"
        if sensor == "lidar" and (kind, m) == ("four", "m3"):       # SECOND: a 32-ring cloud (~7000 points)
            clouds = [synth.lidar_cloud(rng, 32, 256) for _ in range(k)]
        elif sensor == "lidar":
            clouds = [_cloud(rng, int(rng.integers(1200, 2200))) for _ in range(k)]
        if sensor == "lidar":
            offs = np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds])]).astype(np.int32)
            batch[f"inputs_{m}"] = {"points": torch.from_numpy(np.concatenate(clouds)).cuda(),
                                    "agent_offsets": torch.from_numpy(offs).cuda()}
        else:
            rots, trans, intr, post_rots, post_trans = [torch.from_numpy(a).cuda() for a in synth.camera_rig(k, CAMS, IMG_H, IMG_W)]
            trans = trans + torch.from_numpy(rng.uniform(-0.3, 0.3, tuple(trans.shape)).astype(np.float32)).cuda()
            gen = torch.Generator().manual_seed(1000 + seed)
            imgs = torch.randint(0, 256, (k, CAMS, FRAME_H, FRAME_W, 3), generator=gen, dtype=torch.uint8) if raw else \
                torch.randn(k, CAMS, 3, IMG_H, IMG_W, generator=gen)
            batch[f"inputs_{m}"] = {"imgs": imgs.cuda(), "rots": rots, "trans": trans, "intrins": intr, "post_rots": post_rots,
                                    "post_trans": post_trans}
    poses = [[0, 0, 0, 0, 0, 0]] + [[rng.uniform(-5, 5), rng.uniform(-5, 5), 0, 0, rng.uniform(-180, 180), 0]
                                    for _ in range(len(aml) - 1)]
    batch["pairwise_t_matrix"] = torch.from_numpy(synth.pairwise_t_matrix(poses, 5)[None]).cuda()
    return batch


def capacities(kind, raw=False):
    caps = {}
    for m in dict.fromkeys(AML[kind]):
        if (kind, m) in {("c4", "m2"), ("four", "m2"), ("four", "m4"), ("baseline", "m2")}:
            caps[m] = (CAMS, FRAME_H, FRAME_W, torch.uint8) if raw else (CAMS, IMG_H, IMG_W)
        else:
            caps[m] = SECOND_CAPACITY if (kind, m) == ("four", "m3") else LIDAR_CAPACITY
    return caps


PAIRWISE_SHAPE = (1, 5, 5, 4, 4)


def postprocess_params():
    return make_golden.postprocess_params(rng=tuple(RANGE))
