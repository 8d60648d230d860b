"""ORACLE — TEST INFRASTRUCTURE ONLY.  A literal restatement of the reference's V2X-ViT fusion (opencood/models/fuse_modules/
fusion_in_one.py:320-372 V2XViTFusion; sub_modules/v2xvit_basic.py STTF / V2XFusionBlock / V2XTEncoder / V2XTransformer;
hmsa.py HGTCavAttention; mswin.py BaseWindowAttention / PyramidWindowAttention; split_attn.py SplitAttn; base_transformer.py
PreNorm / FeedForward; torch_transformation_utils.py warp_affine, get_roi_and_cav_mask and the matrix chain) and of
HeterModelBaseline with `fusion_method: v2xvit`, in plain functional PyTorch over a flat state_dict.  The einops rearranges are
reshape / permute, the relation einsums matmuls; runs on any device.  Pinned against the reference's own modules by
oracle/make_golden_v2xvit.py -> tests/golden/{fusion_v2xvit,heter_model_baseline_v2xvit_small}.pt.xz.
"""
import os
from collections import Counter

import numpy as np
import torch
import torch.nn.functional as F

from oracle import cobevt, fusion_methods, golden, nets

MODULE_GOLDEN = "fusion_v2xvit.pt"


def v2xvit_args(dim=256, depth=3):
    """`v2xvit:` block of opv2v/LiDAROnly/lidar_v2xvit.yaml (every shipped v2xvit config uses the same encoder)."""
    return {"transformer": {"encoder": {
        "num_blocks": 1, "depth": depth, "use_roi_mask": True, "use_RTE": False, "RTE_ratio": 0,
        "cav_att_config": {"dim": dim, "use_hetero": True, "use_RTE": False, "RTE_ratio": 0, "heads": 8, "dim_head": 32,
                           "dropout": 0.3},
        "pwindow_att_config": {"dim": dim, "heads": [16, 8, 4], "dim_head": [16, 32, 64], "dropout": 0.3,
                               "window_size": [4, 8, 16], "relative_pos_embedding": True, "fusion_method": "split_attn"},
        "feed_forward": {"mlp_dim": 256, "dropout": 0.3},
        "sttf": {"voxel_size": [0.4, 0.4, 4], "downsample_rate": 4}}}}


def module_cases():
    """name -> (args, seeded input shape, record_len, pairwise-pose scenes, L) of fusion_v2xvit.pt."""
    two = [[[0, 0, 0, 0, 0, 0], [3.0, -1.5, 0, 0, 35, 0], [-4.0, 2.5, 0, 0, -120, 0]],
           [[0, 0, 0, 0, 0, 0], [0.07, 0.05, 0, 0, 0, 0]]]
    return {
        "c256": (v2xvit_args(), (5, 256, 16, 32), [3, 2], two, 5),
        "l2": (v2xvit_args(depth=2), (3, 256, 16, 16), [2, 1],
               [[[0, 0, 0, 0, 0, 0], [2.0, 1.0, 0, 0, 60, 0]], [[0, 0, 0, 0, 0, 0]]], 2),
    }


def case_inputs(name):
    """(x, record_len, pairwise_t_matrix) of case `name`: x is drawn from a seeded generator (not stored in the golden)."""
    from workloads import synth
    args, shape, rl, scenes, L = module_cases()[name]
    seed = {"c256": 61, "l2": 62}[name]
    x = torch.randn(*shape, generator=torch.Generator().manual_seed(seed))
    pw = np.stack([synth.pairwise_t_matrix(p, L) for p in scenes])
    return x, torch.tensor(rl), torch.from_numpy(pw)


def case_affine(pw):
    return nets.normalize_pairwise_tfm(pw, 9.6, 16.0, 1)


def load_module_golden(golden_dir):
    return golden.load(os.path.join(golden_dir, MODULE_GOLDEN))


# ---- torch_transformation_utils.py ------------------------------------------------------------------------------------
def get_discretized_transformation_matrix(matrix, discrete_ratio, downsample_rate):
    matrix = matrix[:, :, [0, 1], :][:, :, :, [0, 1, 3]]
    matrix[:, :, :, -1] = matrix[:, :, :, -1] / (discrete_ratio * downsample_rate)
    return matrix.type(dtype=torch.float)


def normal_transform_pixel(height, width, device, dtype, eps=1e-14):
    tr_mat = torch.tensor([[1.0, 0.0, -1.0], [0.0, 1.0, -1.0], [0.0, 0.0, 1.0]], device=device, dtype=dtype)
    width_denom = eps if width == 1 else width - 1.0
    height_denom = eps if height == 1 else height - 1.0
    tr_mat[0, 0] = tr_mat[0, 0] * 2.0 / width_denom
    tr_mat[1, 1] = tr_mat[1, 1] * 2.0 / height_denom
    return tr_mat.unsqueeze(0)


def normalize_homography(dst_pix_trans_src_pix, dsize_src, dsize_dst):
    src_h, src_w = dsize_src
    dst_h, dst_w = dsize_dst
    dev, dt = dst_pix_trans_src_pix.device, dst_pix_trans_src_pix.dtype
    src_norm_trans_src_pix = normal_transform_pixel(src_h, src_w, dev, dt)
    src_pix_trans_src_norm = torch.inverse(src_norm_trans_src_pix)
    dst_norm_trans_dst_pix = normal_transform_pixel(dst_h, dst_w, dev, dt)
    return dst_norm_trans_dst_pix @ (dst_pix_trans_src_pix @ src_pix_trans_src_norm)


def get_transformation_matrix(M, dsize):
    """get_rotation_matrix2d (shift @ rotation @ shift^-1 about the map centre) plus the translation of M."""
    H, W = dsize
    B = M.shape[0]
    center = torch.Tensor([W / 2, H / 2]).to(M.dtype).to(M.device).unsqueeze(0)
    shift_m = torch.eye(3, device=M.device, dtype=M.dtype)[None].repeat(B, 1, 1)
    shift_m[:, :2, 2] = center
    shift_m_inv = torch.eye(3, device=M.device, dtype=M.dtype)[None].repeat(B, 1, 1)
    shift_m_inv[:, :2, 2] = -center
    rotat_m = torch.eye(3, device=M.device, dtype=M.dtype)[None].repeat(B, 1, 1)
    rotat_m[:, :2, :2] = M[:, :2, :2]
    T = (shift_m @ rotat_m @ shift_m_inv)[:, :2, :]
    T[..., 2] += M[..., 2]
    return T


def warp_affine_matrix(M, dsize_src, dsize_dst):
    """The 2x3 matrix warp_affine hands F.affine_grid: inverse of the normalised homography of M."""
    M3 = F.pad(M, [0, 0, 0, 1], "constant", value=0.0)
    M3[..., -1, -1] += 1.0
    return torch.inverse(normalize_homography(M3, dsize_src, dsize_dst))[:, :2, :]


def warp_affine(src, M, dsize, mode="bilinear"):
    """torch_transformation_utils.py:334-374 (align_corners=True, zeros padding)."""
    B, C, H, W = src.shape
    theta = warp_affine_matrix(M, (H, W), dsize)
    grid = F.affine_grid(theta, [B, C, dsize[0], dsize[1]], align_corners=True).to(src.dtype)   # fp32 grid, as in the reference
    return F.grid_sample(src, grid, align_corners=True, mode=mode, padding_mode="zeros")


def sttf_matrix(spatial_correction_matrix, H, W, discrete_ratio, downsample_rate):
    """(B*(L-1), 2, 3): the matrices STTF warps the non-ego agents by (v2xvit_basic.py:12-33)."""
    d = get_discretized_transformation_matrix(spatial_correction_matrix, discrete_ratio, downsample_rate)
    return get_transformation_matrix(d[:, 1:, :, :].reshape(-1, 2, 3), (H, W))


def get_roi_and_cav_mask(shape, cav_mask, spatial_correction_matrix, discrete_ratio, downsample_rate):
    """(B, H, W, 1, L): the nearest-warped all-ones ROI of every agent times its cav mask."""
    B, L, H, W, _ = shape
    d = get_discretized_transformation_matrix(spatial_correction_matrix, discrete_ratio, downsample_rate)
    T = get_transformation_matrix(d.reshape(-1, 2, 3), (H, W))
    ones = torch.ones((B * L, 1, H, W), dtype=T.dtype, device=T.device)
    roi = warp_affine(ones, T, (H, W), mode="nearest").reshape(B, L, 1, H, W)
    com = roi * cav_mask[:, :, None, None, None].expand(roi.shape)
    return com.permute(0, 3, 4, 2, 1)


# ---- the encoder ---------------------------------------------------------------------------------------------------
def layer_norm(x, sd, p):
    return F.layer_norm(x, (x.shape[-1],), sd[p + ".weight"], sd[p + ".bias"], 1e-5)


def linear(x, sd, p, bias=True):
    return F.linear(x, sd[p + ".weight"], sd[p + ".bias"] if bias else None)


def hgt_cav_attention(x, mask, types, sd, p, heads, dim_head):
    """hmsa.py HGTCavAttention.forward.  x (B, L, H, W, C); mask (B, H, W, 1, L); types (B, L) int."""
    x = x.permute(0, 2, 3, 1, 4)                                          # B H W L C
    B, H, W, L, _ = x.shape
    mask = mask.unsqueeze(1)                                              # B 1 H W 1 L
    q, k, v = (torch.stack([torch.stack([linear(x[b, :, :, i], sd, f"{p}.{n}_linears.{int(types[b, i])}")
                                         for i in range(L)], dim=2) for b in range(B)])
               for n in ("q", "k", "v"))                                  # B H W L inner
    num_types = 2
    w_att = torch.stack([torch.stack([torch.stack([sd[p + ".relation_att"][int(types[b, i]) * num_types + int(types[b, j])]
                                                   for j in range(L)]) for i in range(L)]) for b in range(B)])
    w_msg = torch.stack([torch.stack([torch.stack([sd[p + ".relation_msg"][int(types[b, i]) * num_types + int(types[b, j])]
                                                   for j in range(L)]) for i in range(L)]) for b in range(B)])
    w_att = w_att.permute(0, 3, 1, 2, 4, 5)                               # B M L L p q
    w_msg = w_msg.permute(0, 3, 1, 2, 4, 5)
    q, k, v = (t.reshape(B, H, W, L, heads, dim_head).permute(0, 4, 1, 2, 3, 5) for t in (q, k, v))   # B M H W L c
    # att[b,m,h,w,i,j] = sum_{p,q} q[b,m,h,w,i,p] w_att[b,m,i,j,p,q] k[b,m,h,w,j,q]
    qw = (q[:, :, :, :, :, None, None, :] @ w_att[:, :, None, None]).squeeze(-2)   # B M H W i j q
    att = (qw * k.unsqueeze(4)).sum(-1) * dim_head ** -0.5                        # B M H W i j
    att = att.masked_fill(mask == 0, -float("inf")).softmax(dim=-1)
    # v_msg[b,m,h,w,i,j,c] = sum_p w_msg[b,m,i,j,p,c] v[b,m,h,w,j,p]
    v_msg = (v[:, :, :, :, None, :, None, :] @ w_msg[:, :, None, None]).squeeze(-2)  # B M H W i j c
    out = (att.unsqueeze(-1) * v_msg).sum(5)                                      # B M H W i c
    out = out.permute(0, 2, 3, 4, 1, 5).reshape(B, H, W, L, heads * dim_head)
    out = torch.stack([torch.stack([linear(out[b, :, :, i], sd, f"{p}.a_linears.{int(types[b, i])}") for i in range(L)], dim=2)
                       for b in range(B)])
    return out.permute(0, 3, 1, 2, 4)                                             # B L H W C


def relative_indices(ws):
    idx = torch.tensor(np.array([[x, y] for x in range(ws) for y in range(ws)]))
    return idx[None, :, :] - idx[:, None, :] + ws - 1


def base_window_attention(x, sd, p, heads, dim_head, ws):
    """mswin.py BaseWindowAttention.forward with relative_pos_embedding.  x (b, l, h, w, c)."""
    b, l, h, w, _ = x.shape
    inner = heads * dim_head
    q, k, v = F.linear(x, sd[p + ".to_qkv.weight"]).chunk(3, dim=-1)
    nh, nw = h // ws, w // ws
    # 'b l (new_h w_h) (new_w w_w) (m c) -> b l m (new_h new_w) (w_h w_w) c'
    q, k, v = (t.reshape(b, l, nh, ws, nw, ws, heads, dim_head).permute(0, 1, 6, 2, 4, 3, 5, 7)
               .reshape(b, l, heads, nh * nw, ws * ws, dim_head) for t in (q, k, v))
    dots = q @ k.transpose(-1, -2) * dim_head ** -0.5
    ri = relative_indices(ws).to(x.device)
    dots = dots + sd[p + ".pos_embedding"][ri[:, :, 0], ri[:, :, 1]]
    out = dots.softmax(dim=-1) @ v
    out = out.reshape(b, l, heads, nh, nw, ws, ws, dim_head).permute(0, 1, 3, 5, 4, 6, 2, 7).reshape(b, l, h, w, inner)
    return linear(out, sd, p + ".to_out.0")


def split_attn(window_list, sd, p):
    """split_attn.py SplitAttn.forward (RadixSoftmax(3, 1))."""
    sw, mw, bw = window_list
    B, L = sw.shape[:2]
    x_gap = (sw + mw + bw).mean((2, 3), keepdim=True)
    x_gap = F.relu(layer_norm(F.linear(x_gap, sd[p + ".fc1.weight"]), sd, p + ".bn1"))
    x_attn = F.linear(x_gap, sd[p + ".fc2.weight"])
    x_attn = F.softmax(x_attn.view(B, L, 1, 3, -1), dim=3).reshape(B, -1).view(B, L, 1, 1, -1)
    C = sw.shape[-1]
    return sw * x_attn[..., 0:C] + mw * x_attn[..., C:2 * C] + bw * x_attn[..., 2 * C:]


def feed_forward(x, sd, p):
    return linear(F.gelu(linear(x, sd, p + ".net.0")), sd, p + ".net.3")


def v2xt_encoder(x, mask, scm, sd, p, enc):
    """v2xvit_basic.py V2XTEncoder.forward (no RTE).  x (B, L, H, W, C + 3)."""
    prior = x[..., -3:]
    x = x[..., :-3]
    B, L, H, W, C = x.shape
    ratio, rate = enc["sttf"]["voxel_size"][0], enc["sttf"]["downsample_rate"]
    # STTF
    xs = x.permute(0, 1, 4, 2, 3)
    T = sttf_matrix(scm, H, W, ratio, rate)
    cav = warp_affine(xs[:, 1:].reshape(-1, C, H, W), T, (H, W)).reshape(B, -1, C, H, W)
    x = torch.cat([xs[:, :1], cav], dim=1).permute(0, 1, 3, 4, 2)
    com_mask = get_roi_and_cav_mask(x.shape, mask, scm, ratio, rate) if enc["use_roi_mask"] else \
        mask[:, None, None, None, :]
    types = prior[:, :, 0, 0, 2].to(torch.int)
    cav_cfg, pw = enc["cav_att_config"], enc["pwindow_att_config"]
    for i in range(enc["depth"]):
        lp = f"{p}.layers.{i}"
        for blk in range(enc["num_blocks"]):
            bp = f"{lp}.0.layers.{blk}"
            x = hgt_cav_attention(layer_norm(x, sd, bp + ".0.norm"), com_mask, types, sd, bp + ".0.fn", cav_cfg["heads"],
                                  cav_cfg["dim_head"]) + x
            y = layer_norm(x, sd, bp + ".1.norm")
            outs = [base_window_attention(y, sd, f"{bp}.1.fn.pwmsa.{k}", hd, dh, ws)
                    for k, (hd, dh, ws) in enumerate(zip(pw["heads"], pw["dim_head"], pw["window_size"]))]
            x = split_attn(outs, sd, bp + ".1.fn.split_attn") + x
        x = feed_forward(layer_norm(x, sd, lp + ".1.norm"), sd, lp + ".1.fn") + x
    return x


def v2xvit_fusion(x, sd, p, args, record_len, affine_matrix):
    """fusion_in_one.py:320-372 (V2XViTFusion.forward) in eval; `args` = the yaml's `v2xvit:` block."""
    _, C, H, W = x.shape
    B, L = affine_matrix.shape[:2]
    feats, mask = cobevt.regroup(x, record_len, L)
    prior = torch.zeros(len(record_len), L, 3, H, W, dtype=x.dtype, device=x.device)
    feats = torch.cat([feats, prior], dim=2)
    feats = torch.stack([fusion_methods.warp_affine_simple(feats[b], affine_matrix[b, 0], (H, W)) for b in range(B)])
    feats = feats.permute(0, 1, 3, 4, 2)
    scm = torch.eye(4, device=x.device).expand(len(record_len), L, 4, 4)
    out = v2xt_encoder(feats, mask, scm, sd, p + ".fusion_net.encoder", args["transformer"]["encoder"])
    return out[:, 0].permute(0, 3, 1, 2)


def heter_model_baseline(sd, args, data_dict):
    """heter_model_baseline.py:155-236 for PointPillars modalities with fusion_method v2xvit."""
    mods = [k for k in args.keys() if k.startswith("m") and k[1:].isdigit()]
    rng = args["lidar_range"]
    affine = nets.normalize_pairwise_tfm(data_dict["pairwise_t_matrix"], rng[4] - rng[1], rng[3] - rng[0], 1)
    aml = data_dict["agent_modality_list"]
    cnt = Counter(aml)
    feats = {}
    for m in mods:
        if m not in cnt:
            continue
        f = nets.point_pillar_encoder(sd, f"encoder_{m}", args[m]["encoder_args"], data_dict[f"inputs_{m}"])
        f = nets.base_bev_backbone(f, sd, f"backbone_{m}", args[m]["backbone_args"])
        feats[m] = nets.downsample_conv(f, sd, f"shrinker_{m}", args[m]["shrink_header"])
    counting = {m: 0 for m in mods}
    lst = []
    for m in aml:
        lst.append(feats[m][counting[m]])
        counting[m] += 1
    x = torch.stack(lst)
    assert args["fusion_method"] == "v2xvit"
    fused = v2xvit_fusion(x, sd, "fusion_net", args["v2xvit"], data_dict["record_len"], affine)
    if "shrink_header" in args:
        fused = nets.downsample_conv(fused, sd, "shrink_conv", args["shrink_header"])
    return {"cls_preds": nets.conv(fused, sd, "cls_head"), "reg_preds": nets.conv(fused, sd, "reg_head"),
            "dir_preds": nets.conv(fused, sd, "dir_head"), "fused_feature": fused}
