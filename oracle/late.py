"""ORACLE — TEST INFRASTRUCTURE ONLY.  CPU restatements of the single-agent models behind HEAL's `Single/*` and stage-2 configs,
built on oracle/nets.py, oracle/coalign.py, oracle/lss.py and oracle/efficientnet.py:

  heter_model_late      opencood/models/heter_model_late.py:70-112: encoder -> ResNetBEVBackbone -> camera CenterCrop ->
                        levels 1.. of `layers_<m>` (layer0 never runs) -> `layers_<m>` deblocks -> shrink -> per-modality heads
  heter_pyramid_single  opencood/models/heter_pyramid_single.py:99-136: encoder -> ResNetBEVBackbone -> aligner -> camera
                        CenterCrop -> PyramidFusion.forward_single -> shrink -> shared heads

plus the configs, inputs and weights oracle/make_golden_late.py and the tests share.  Nothing here imports heal_b200.
"""
import copy

import numpy as np
import torch
import torch.nn.functional as F
import torchvision

from oracle import coalign, nets, lss, efficientnet as oe, make_golden

SMALL_RANGE, VOXEL = make_golden.SMALL_RANGE, make_golden.VOXEL
HEAD = {"anchor_number": 2, "dir_args": {"dir_offset": 0.7853, "num_bins": 2, "anchor_yaw": [0, 90]}}
LAYERS = {"layer_nums": [3, 5, 8], "layer_strides": [2, 2, 2], "num_filters": [64, 128, 256],
          "upsample_strides": [1, 2, 4], "num_upsample_filter": [128, 128, 128]}
SHRINK = {"kernal_size": [3], "stride": [1], "padding": [1], "dim": [256], "input_dim": 384}


def _m1():
    return copy.deepcopy(make_golden.small_model_args()["m1"])


def _m2_eff():
    """m2 of opv2v/Single/m2_LSSeff48_pretrain.yaml scaled down: Lift-Splat-Shoot with the EfficientNet trunk on a +-19.2 m camera
    grid, so the 48 x 48 backbone map is center-cropped to the lidar range's 32 x 32."""
    return copy.deepcopy(oe.collab_args()["m2"])


def late_args(mod):
    """`model.args` of a Single/* config (heter_model_late) with one modality: 'm1' PointPillars or 'm2eff' LSS-EfficientNet."""
    m = _m1() if mod == "m1" else _m2_eff()
    m["layers_args"] = copy.deepcopy(LAYERS)
    m["shrink_header"] = copy.deepcopy(SHRINK)
    m["head_args"] = {"in_head": 256}
    return {"lidar_range": list(SMALL_RANGE), "ego_modality": "m1" if mod == "m1" else "m2",
            ("m1" if mod == "m1" else "m2"): m, **copy.deepcopy(HEAD)}


def pyramid_single_args(mod):
    """`model.args` of a HEAL stage-2 *_single_pyramid.yaml: 'm1' (identity aligner) or 'm2_convnext' (LSS-EfficientNet camera
    agent with a 3-block ConvNeXt aligner)."""
    a = make_golden.small_model_args()
    a.pop("supervise_single")
    if mod != "m1":
        a.pop("m1")
        a["m2"] = _m2_eff()
        a["m2"]["aligner_args"] = {"core_method": "convnext", "spatial_align": False, "args": {"num_of_blocks": 3, "dim": 64}}
    return a


def lidar_cav(seed):
    """One cav's `inputs_m1` as the late dataset collates it (voxels of one cloud, agent index 0 in voxel_coords)."""
    return make_golden.small_scene(seed=seed, n_agents=1)["inputs_m1"]


def scene_points(seed, n=1500):
    """The raw cloud small_scene(seed, n_agents=1) voxelises (same generator draws)."""
    rng = np.random.default_rng(seed)
    return np.concatenate([rng.uniform(-14, 14, (n, 2)), rng.uniform(-3.5, 1.5, (n, 1)), rng.uniform(0, 1, (n, 1))],
                          1).astype(np.float32)


def pose(x, y, yaw_deg, z=0.0):
    c, s = np.cos(np.radians(yaw_deg)), np.sin(np.radians(yaw_deg))
    return torch.tensor([[c, -s, 0, x], [s, c, 0, y], [0, 0, 1, z], [0, 0, 0, 1]], dtype=torch.float64)


SCENE_SEEDS = (21, 22, 23)
SCENE_POSES = ((0.0, 0.0, 0.0), (4.0, -3.0, 35.0), (-5.0, 2.5, -120.0))


def scene_batch(anchors):
    """The late scene: three m1 cavs with different poses, as the late dataset's collate hands them to inference_late_fusion."""
    out = {}
    for i, (seed, p) in enumerate(zip(SCENE_SEEDS, SCENE_POSES)):
        out["ego" if i == 0 else f"cav{i}"] = {"inputs_m1": lidar_cav(seed), "anchor_box": anchors,
                                               "transformation_matrix": pose(*p).float()}
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# restatements
# ---------------------------------------------------------------------------------------------------------------------------
def modality_of(data_dict):
    """heter_model_late.py:72-74: the one `inputs_*` key through str.lstrip('inputs_')."""
    names = [k for k in data_dict if k.startswith("inputs_")]
    assert len(names) == 1
    return names[0].lstrip("inputs_")


def _up(x1, x2, sd, p):
    """lss_submodule.py:17-36 (Up): bilinear x2 align_corners of x1, cat([x2, x1]), 2 x (conv3x3 + BN(1e-5) + ReLU)."""
    x = torch.cat([x2, F.interpolate(x1, scale_factor=2, mode="bilinear", align_corners=True)], 1)
    x = F.relu(nets.bn_eval(nets.conv(x, sd, p + ".conv.0", 1, 1), sd, p + ".conv.1", 1e-5))
    return F.relu(nets.bn_eval(nets.conv(x, sd, p + ".conv.3", 1, 1), sd, p + ".conv.4", 1e-5))


def eff_cam_heads(sd, p, imgs, downsample):
    """CamEncode (EfficientNet) depth logits and image features (lss_submodule.py:87-134) over oracle/efficientnet's trunk."""
    trunk = oe.EfficientNet().eval()
    trunk.load_state_dict({k[len(p) + 7:]: v for k, v in sd.items() if k.startswith(p + ".trunk.")}, strict=True)
    with torch.no_grad():
        x = trunk._swish(trunk._bn0(trunk._conv_stem(imgs[:, :3])))
        ends, prev = [], x
        for blk in trunk._blocks:
            x = blk(x)
            if prev.shape[2] > x.shape[2]:
                ends.append(prev)
            prev = x
        ends.append(x)
        f = _up(ends[4], ends[3], sd, p + ".up1")
        if downsample == 8:
            f = _up(f, ends[2], sd, p + ".up2")
        return nets.conv(f, sd, p + ".depth_head"), nets.conv(f, sd, p + ".image_head")


def lss_eff_encoder(sd, p, enc_args, cam):
    imgs = cam["imgs"]
    B, N = imgs.shape[:2]
    dl, ft = eff_cam_heads(sd, p + ".camencode", imgs.reshape(B * N, *imgs.shape[2:]), enc_args["img_downsample"])
    g = enc_args["grid_conf"]
    fr = lss.create_frustum(g, enc_args["data_aug_conf"]["final_dim"], enc_args["img_downsample"])
    dx, bx, nx = lss.gen_dx_bx(g["xbound"], g["ybound"], g["zbound"])
    geom = lss.get_geometry(fr, cam["rots"], cam["trans"], cam["intrins"], cam["post_rots"], cam["post_trans"])
    x = lss.outer_product(dl, ft).view(B, N, -1, *fr.shape[:3]).permute(0, 1, 3, 4, 5, 2)
    return lss.voxel_pooling(geom, x, dx, bx, nx, exact=True)


def _encode(sd, args, m, data_dict):
    s = args[m]
    if s["core_method"] == "point_pillar":
        f = nets.point_pillar_encoder(sd, f"encoder_{m}", s["encoder_args"], data_dict[f"inputs_{m}"])
    else:
        assert s["core_method"] == "lift_splat_shoot" and s["encoder_args"]["camera_encoder"] == "EfficientNet"
        f = lss_eff_encoder(sd, f"encoder_{m}", s["encoder_args"], data_dict[f"inputs_{m}"])
    return nets.resnet_bev_backbone(f, sd, f"backbone_{m}", s["backbone_args"])


def _crop(f, args, m):
    if args[m]["sensor_type"] != "camera":
        return f
    g, rng_ = args[m]["camera_mask_args"]["grid_conf"], args["lidar_range"]
    rw, rh = rng_[3] / g["xbound"][1], rng_[4] / g["ybound"][1]
    return torchvision.transforms.CenterCrop((int(f.shape[2] * rh), int(f.shape[3] * rw)))(f)


def heter_model_late(sd, args, data_dict):
    m = modality_of(data_dict)
    with torch.no_grad():
        f = _crop(_encode(sd, args, m, data_dict), args, m)
        la = args[m]["layers_args"]
        feats = [f]
        for i in range(1, len(la["num_upsample_filter"])):
            f = coalign.resnet_layer(f, sd, f"layers_{m}", la, i)
            feats.append(f)
        f = nets.deblocks(feats, sd, f"layers_{m}", la["upsample_strides"])
        f = nets.downsample_conv(f, sd, f"shrink_conv_{m}", args[m]["shrink_header"])
        return {k: nets.conv(f, sd, f"{k[:3]}_head_{m}") for k in ("cls_preds", "reg_preds", "dir_preds")}


def heter_pyramid_single(sd, args, data_dict):
    m = modality_of(data_dict)
    with torch.no_grad():
        f = _encode(sd, args, m, data_dict)
        al = args[m]["aligner_args"]
        if al["core_method"] == "convnext":
            f = nets.convnext_aligner(f, sd, f"aligner_{m}", al["args"]["num_of_blocks"], al["args"].get("kernel_size", 7))
        f = _crop(f, args, m)
        cfg = args["fusion_backbone"]
        feats = nets.resnet_modified(f, sd, "pyramid_backbone.resnet", "bottleneck", cfg["layer_nums"], cfg["layer_strides"],
                                     cfg["num_filters"], cfg.get("inplanes", 64), groups=32)
        occ = [nets.conv(x, sd, f"pyramid_backbone.single_head_{i}") for i, x in enumerate(feats)]
        f = nets.deblocks(feats, sd, "pyramid_backbone", cfg["upsample_strides"])
        if "shrink_header" in args:
            f = nets.downsample_conv(f, sd, "shrink_conv", args["shrink_header"])
        out = {k: nets.conv(f, sd, k.replace("_preds", "_head")) for k in ("cls_preds", "reg_preds", "dir_preds")}
        out["occ_single_list"] = occ
        return out
