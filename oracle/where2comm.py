"""ORACLE — TEST INFRASTRUCTURE ONLY.  Restatements of the reference's Where2commFusion and Who2comFusion
(opencood/models/fuse_modules/fusion_in_one.py:431-539, where2comm_attn.py:64-103 EncodeLayer) and of HeterModelBaseline with
fusion_method where2comm / who2com, in plain functional PyTorch over a flat state_dict, on any device and in any float dtype.
Pinned against the reference's own modules by oracle/make_golden_where2comm.py -> tests/golden/fusion_where2comm_who2com.pt.xz
and heter_model_baseline_{where2comm,who2com}_small.pt.xz.

`where2comm_fusion` is literal: every agent is warped to the ego, then nn.MultiheadAttention's math path (in-projection with bias,
q * dim_head^-0.5, softmax over the agents, out_proj), LayerNorm, FFN, LayerNorm.  `where2comm_fusion_projected` is the
GPU path's form: the bias-free k | v projection of the UNWARPED maps, sampled, plus the bias.  Tests hold the two equal in
float64, which is what lets the GPU path run the projection before the warp.
"""
import os
from collections import Counter

import torch
import torch.nn.functional as F

from oracle import golden, nets
from oracle.fusion_methods import warp_affine_simple

MODULE_GOLDEN = "fusion_where2comm_who2com.pt"
HEADS = 8


def fusion_x():
    """The seeded input of fusion_where2comm_who2com.pt: 7 agents (record_len [3, 2, 2]), C = 256, a ragged 24 x 40 map."""
    return torch.randn(7, 256, 24, 40, generator=torch.Generator().manual_seed(43))


def load_module_golden(golden_dir):
    """fusion_where2comm_who2com.pt with its seeded input `x` put back (the stored file leaves it out)."""
    d = golden.load(os.path.join(golden_dir, MODULE_GOLDEN))
    d["x"] = fusion_x()
    return d


def _regroup(x, record_len):
    return list(torch.split(x, [int(n) for n in record_len]))


def _mha_tail(x0, ctx, sd, p, C):
    """ctx (HW, C) merged heads -> out_proj -> LN1(x0 + .) -> FFN -> LN2, x0 (HW, C) the warped ego; p = the EncodeLayer."""
    a = F.linear(ctx, sd[p + ".attn.out_proj.weight"], sd[p + ".attn.out_proj.bias"])
    y1 = F.layer_norm(x0 + a, (C,), sd[p + ".norm1.weight"], sd[p + ".norm1.bias"], 1e-5)
    f = F.linear(F.relu(F.linear(y1, sd[p + ".linear1.weight"], sd[p + ".linear1.bias"])),
                 sd[p + ".linear2.weight"], sd[p + ".linear2.bias"])
    return F.layer_norm(y1 + f, (C,), sd[p + ".norm2.weight"], sd[p + ".norm2.bias"], 1e-5)


def _attend(q, k, v, C):
    """q (HW, C) projected ego, k / v (n, HW, C) -> (HW, C): per pixel and head softmax_j((q * dh^-0.5) . k_j) v_j."""
    dh = C // HEADS
    n, HW = k.shape[:2]
    qh = (q * (1.0 / dh) ** 0.5).view(HW, HEADS, dh)
    kh, vh = k.view(n, HW, HEADS, dh), v.view(n, HW, HEADS, dh)
    s = torch.einsum("phd,nphd->phn", qh, kh)
    a = torch.softmax(s, dim=-1)
    return torch.einsum("phn,nphd->phd", a, vh).reshape(HW, C)


def where2comm_fusion(x, sd, p, record_len, affine_matrix):
    """fusion_in_one.py:431-484 (Where2commFusion) as written: x (sumN, C, H, W) -> (B, C, H, W)."""
    _, C, H, W = x.shape
    p = p + ".mha_fusion"
    w, b = sd[p + ".attn.in_proj_weight"], sd[p + ".attn.in_proj_bias"]
    out = []
    for bi, xb in enumerate(_regroup(x, record_len)):
        n = xb.shape[0]
        X = warp_affine_simple(xb, affine_matrix[bi][0, :n], (H, W)).permute(0, 2, 3, 1).reshape(n, H * W, C)
        q = F.linear(X[0], w[:C], b[:C])
        k = F.linear(X, w[C:2 * C], b[C:2 * C])
        v = F.linear(X, w[2 * C:], b[2 * C:])
        y = _mha_tail(X[0], _attend(q, k, v, C), sd, p, C)
        out.append(y.t().reshape(C, H, W))
    return torch.stack(out)


def where2comm_fusion_projected(x, sd, p, record_len, affine_matrix):
    """The GPU path's formulation: k | v = warp([W_k; W_v] x_j) + [b_k; b_v], the projection run on the unwarped maps."""
    _, C, H, W = x.shape
    p = p + ".mha_fusion"
    w, b = sd[p + ".attn.in_proj_weight"], sd[p + ".attn.in_proj_bias"]
    out = []
    for bi, xb in enumerate(_regroup(x, record_len)):
        n = xb.shape[0]
        X0 = warp_affine_simple(xb[:1], affine_matrix[bi][0, :1], (H, W)).permute(0, 2, 3, 1).reshape(H * W, C)
        kv = F.conv2d(xb, w[C:, :, None, None])
        kv = warp_affine_simple(kv, affine_matrix[bi][0, :n], (H, W)).permute(0, 2, 3, 1).reshape(n, H * W, 2 * C) + b[C:]
        q = F.linear(X0, w[:C], b[:C])
        y = _mha_tail(X0, _attend(q, kv[..., :C], kv[..., C:], C), sd, p, C)
        out.append(y.t().reshape(C, H, W))
    return torch.stack(out)


def who2com_fusion(x, sd, p, record_len, affine_matrix):
    """fusion_in_one.py:486-539 (Who2comFusion): decode_layer(cat[x_0 unwarped, ego row of the attention over the warped agents])."""
    _, C, H, W = x.shape
    out = []
    for bi, xb in enumerate(_regroup(x, record_len)):
        n = xb.shape[0]
        X = warp_affine_simple(xb, affine_matrix[bi][0, :n], (H, W)).reshape(n, C, H * W).permute(2, 0, 1)
        s = torch.bmm(X, X.transpose(1, 2)) / (C ** 0.5)
        a = torch.bmm(torch.softmax(s, -1), X).permute(1, 2, 0).reshape(n, C, H, W)[0]
        out.append(nets.conv(torch.cat([xb[0], a])[None], sd, p + ".decode_layer", padding=1))
    return torch.cat(out)


FUSIONS = {"where2comm": where2comm_fusion, "who2com": who2com_fusion}


def heter_model_baseline(sd, args, data_dict):
    """heter_model_baseline.py:155-236 for PointPillars modalities with fusion_method where2comm or who2com: encoder ->
    BaseBEVBackbone -> per-agent shrinker -> fusion -> (shrink) -> heads."""
    mods = [k for k in args.keys() if k.startswith("m") and k[1:].isdigit()]
    rng = args["lidar_range"]
    affine = nets.normalize_pairwise_tfm(data_dict["pairwise_t_matrix"], rng[4] - rng[1], rng[3] - rng[0], 1)
    aml = data_dict["agent_modality_list"]
    feats = {}
    for m in mods:
        if m not in Counter(aml):
            continue
        f = nets.point_pillar_encoder(sd, f"encoder_{m}", args[m]["encoder_args"], data_dict[f"inputs_{m}"])
        f = nets.base_bev_backbone(f, sd, f"backbone_{m}", args[m]["backbone_args"])
        feats[m] = nets.downsample_conv(f, sd, f"shrinker_{m}", args[m]["shrink_header"])
    counting = {m: 0 for m in mods}
    lst = []
    for m in aml:
        lst.append(feats[m][counting[m]])
        counting[m] += 1
    fused = FUSIONS[args["fusion_method"]](torch.stack(lst), sd, "fusion_net", data_dict["record_len"], affine)
    if "shrink_header" in args:
        fused = nets.downsample_conv(fused, sd, "shrink_conv", args["shrink_header"])
    return {"cls_preds": nets.conv(fused, sd, "cls_head"), "reg_preds": nets.conv(fused, sd, "reg_head"),
            "dir_preds": nets.conv(fused, sd, "dir_head"), "fused_feature": fused}
