"""ORACLE — TEST INFRASTRUCTURE ONLY.  Literal restatement of the reference's HeterModelBaselineMs
(opencood/models/heter_model_baseline_ms.py:26-220), the multi-scale model of every `*_coalign.yaml`, in plain functional PyTorch
over a flat state_dict, built from the pieces of oracle/nets.py (encoders, ResNet blocks, deblocks, shrink header), oracle/hetero.py
(Lift-Splat-Shoot) and oracle/fusion_methods.py (MaxFusion, the device-agnostic warp).  Pinned against the reference's own model
by oracle/make_golden_coalign.py -> tests/golden/heter_model_baseline_ms_*.pt.xz.

AttFusion here scales the scores by 1/sqrt(feat_dim) as the reference's ScaledDotProductAttention(feat_dim[i]) does, not by
1/sqrt(C) as nets.att_fusion does: the two agree only when the yaml's feat_dim matches the level's channel count.

The reference's `*_coalign.yaml` files do not parse (`fusion_method: att` is followed by a more-indented `feat_dim:` with the
`att:` key missing); coalign_args() builds the args dict at their values with `att: {feat_dim: [64, 128, 256]}`, as the
indentation intends.
"""
import os
from collections import Counter

import numpy as np
import torch
import torch.nn.functional as F
import torchvision

from oracle import fusion_methods, golden, hetero, nets

SMALL_RANGE = [-12.8, -12.8, -3, 12.8, 12.8, 1]     # 64 x 64 pillars @ 0.4 m -> 32 x 32 level-0 maps
VOXEL = [0.4, 0.4, 4]
GOLDENS = ("att_small", "max_small", "att_two_scenes", "att_hetero")
HETERO_AML = ["m1", "m4", "m1"]


def coalign_args(method="att", supervise_single=False, lidar_range=None):
    """The `model.args` of opv2v/LiDAROnly/lidar_coalign.yaml on a small range (the fusion stage's channel counts and strides as
    in the yaml: levels of 64, 128 and 256 channels at strides 1, 2, 4 of the level-0 map)."""
    rng = list(lidar_range or SMALL_RANGE)
    a = {
        "ego_modality": "m1", "lidar_range": rng, "supervise_single": supervise_single,
        "m1": {"core_method": "point_pillar", "sensor_type": "lidar",
               "encoder_args": {"voxel_size": VOXEL, "lidar_range": rng,
                                "pillar_vfe": {"use_norm": True, "with_distance": False, "use_absolute_xyz": True,
                                               "num_filters": [64]},
                                "point_pillar_scatter": {"num_features": 64}},
               "backbone_args": {"layer_nums": [3], "layer_strides": [2], "num_filters": [64]},
               "aligner_args": {"core_method": "identity"}},
        "fusion_method": method,
        "fusion_backbone": {"layer_nums": [3, 5, 8], "layer_strides": [1, 2, 2], "num_filters": [64, 128, 256],
                            "upsample_strides": [1, 2, 4], "num_upsample_filter": [128, 128, 128]},
        "shrink_header": {"kernal_size": [3], "stride": [1], "padding": [1], "dim": [256], "input_dim": 384},
        "in_head": 256, "anchor_number": 2, "dir_args": {"dir_offset": 0.7853, "num_bins": 2, "anchor_yaw": [0, 90]},
    }
    if method == "att":
        a["att"] = {"feat_dim": [64, 128, 256]}
    if supervise_single:
        a["in_head_single"] = 64
    return a


def hetero_args():
    """m1 PointPillar + m4 of m1m2m3m4_coalign.yaml (Lift-Splat-Shoot, Resnet101 trunk) at lss_small_cfg() sizes, with a camera
    grid of +-19.2 m against the +-12.8 m lidar range: the camera's 48 x 48 level-0 map is center-cropped to 32 x 32."""
    from oracle import make_golden
    a = coalign_args("att")
    lcfg = make_golden.lss_small_cfg()
    lcfg["grid_conf"]["xbound"] = [-19.2, 19.2, 0.4]
    lcfg["grid_conf"]["ybound"] = [-19.2, 19.2, 0.4]
    lcfg["img_features"] = 64
    a["m4"] = {"core_method": "lift_splat_shoot", "sensor_type": "camera", "encoder_args": lcfg,
               "camera_mask_args": {"grid_conf": lcfg["grid_conf"]},
               "backbone_args": {"layer_nums": [3], "layer_strides": [2], "num_filters": [64]},
               "aligner_args": {"core_method": "identity"}}
    return a


def hetero_cam_inputs():
    """The camera agent's inputs (1 agent, 2 cameras, 64 x 128 images), seeded; the golden does not store them."""
    from workloads import synth
    rots, trans, intr, post_rots, post_trans = [torch.from_numpy(a) for a in synth.camera_rig(1, 2, 64, 128)]
    imgs = torch.randn(1, 2, 3, 64, 128, generator=torch.Generator().manual_seed(47))
    return {"imgs": imgs, "rots": rots, "trans": trans, "intrins": intr, "post_rots": post_rots, "post_trans": post_trans}


def load_golden(golden_dir, name):
    """tests/golden/heter_model_baseline_ms_<name>.pt with the seeded camera inputs put back."""
    d = golden.load(os.path.join(golden_dir, f"heter_model_baseline_ms_{name}.pt"))
    if "m4" in d["args"]:
        d["data"]["inputs_m4"] = hetero_cam_inputs()
    return d


# ------------------------------------------------------------------------------------------------ pieces
def resnet_layer(x, sd, p, cfg, i):
    """resblock.py:178-203 layer i of a BasicBlock ResNetModified run on its own (ResNetBEVBackbone.get_layer_i_feature)."""
    nf, ln, ls = cfg["num_filters"], cfg["layer_nums"], cfg["layer_strides"]
    inplanes = cfg.get("inplanes", 64) if i == 0 else nf[i - 1]
    for b in range(ln[i]):
        st = ls[i] if b == 0 else 1
        down = b == 0 and (ls[i] != 1 or inplanes != nf[i])
        x = nets.basic_block(x, sd, f"{p}.resnet.layer{i}.{b}", st, down)
    return x


def att_fusion(xx, record_len, affine_matrix, feat_dim):
    """fusion_in_one.py:126-151 (AttFusion(feat_dim)) + ScaledDotProductAttention :41-45, on xx's device."""
    _, C, H, W = xx.shape
    out = []
    for b, xb in enumerate(fusion_methods._regroup(xx, record_len)):
        N = xb.shape[0]
        x = fusion_methods.warp_affine_simple(xb, affine_matrix[b][0, :N], (H, W))
        x = x.view(N, C, -1).permute(2, 0, 1)
        score = torch.bmm(x, x.transpose(1, 2)) / np.sqrt(feat_dim)
        h = torch.bmm(F.softmax(score, -1), x)
        out.append(h.permute(1, 2, 0).view(N, C, H, W)[0])
    return torch.stack(out)


def fuse_levels(levels, args, record_len, affine):
    """Per-level fusion of heter_model_baseline_ms.py:204-206."""
    out = []
    for i, f in enumerate(levels):
        if args["fusion_method"] == "att":
            out.append(att_fusion(f, record_len, affine, args["att"]["feat_dim"][i]))
        elif args["fusion_method"] == "max":
            out.append(fusion_methods.max_fusion(f, record_len, affine))
        else:
            raise NotImplementedError(args["fusion_method"])
    return out


# ------------------------------------------------------------------------------------------------ the model
def heter_model_baseline_ms(sd, args, data_dict):
    """heter_model_baseline_ms.py:133-220 on the CPU for PointPillar and Lift-Splat-Shoot modalities."""
    mods = [k for k in args.keys() if k.startswith("m") and k[1:].isdigit()]
    rng = args["lidar_range"]
    affine = nets.normalize_pairwise_tfm(data_dict["pairwise_t_matrix"], rng[4] - rng[1], rng[3] - rng[0], 1)
    aml = data_dict["agent_modality_list"]
    cnt = Counter(aml)
    feats = {}
    for m in mods:
        if m not in cnt:
            continue
        s = args[m]
        if s["sensor_type"] == "lidar":
            f = nets.point_pillar_encoder(sd, f"encoder_{m}", s["encoder_args"], data_dict[f"inputs_{m}"])
        else:
            f = hetero.lss_encoder(sd, f"encoder_{m}", s["encoder_args"], data_dict[f"inputs_{m}"])
        f = nets.resnet_bev_backbone(f, sd, f"backbone_{m}", s["backbone_args"])
        al = s["aligner_args"]
        if al["core_method"] == "convnext":
            f = nets.convnext_aligner(f, sd, f"aligner_{m}", al["args"]["num_of_blocks"], al["args"].get("kernel_size", 7))
        else:
            assert al["core_method"] == "identity"
        if s["sensor_type"] == "camera":
            g = s["camera_mask_args"]["grid_conf"]
            rh, rw = rng[4] / g["ybound"][1], rng[3] / g["xbound"][1]
            f = torchvision.transforms.CenterCrop((int(f.shape[2] * rh), int(f.shape[3] * rw)))(f)
        feats[m] = f
    counting = {m: 0 for m in mods}
    lst = []
    for m in aml:
        lst.append(feats[m][counting[m]])
        counting[m] += 1
    x = torch.stack(lst)
    out = {}
    if args.get("supervise_single", False):
        out.update({k + "_single": nets.conv(x, sd, k.replace("_preds", "_head_single"))
                    for k in ("cls_preds", "reg_preds", "dir_preds")})
    fb = args["fusion_backbone"]
    levels = [x]
    for i in range(1, len(fb["layer_nums"])):
        levels.append(resnet_layer(levels[-1], sd, "backbone", fb, i))
    fused = nets.deblocks(fuse_levels(levels, args, data_dict["record_len"], affine), sd, "backbone", fb["upsample_strides"])
    if "shrink_header" in args:
        fused = nets.downsample_conv(fused, sd, "shrink_conv", args["shrink_header"])
    out.update({k: nets.conv(fused, sd, k.replace("_preds", "_head")) for k in ("cls_preds", "reg_preds", "dir_preds")})
    return out
