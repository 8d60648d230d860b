"""ORACLE — TEST INFRASTRUCTURE ONLY.  Literal restatements of the reference's MaxFusion and V2VNetFusion
(opencood/models/fuse_modules/fusion_in_one.py:87-124, :203-318; sub_modules/convgru.py) and of HeterModelBaseline with every
fusion method the mirror builds, in plain functional PyTorch over a flat state_dict.  Unlike oracle/nets.py these run on any
device, so the full-size checks can run the oracle on the GPU.  Pinned against the reference's own modules by
oracle/make_golden_fusion_methods.py -> tests/golden/{fusion_max_v2vnet,heter_model_baseline_{max,v2vnet}_small}.pt.xz.

V2VNet is restated as written: every node updated in every iteration from the concat message conv
msg_cnn(cat[warp(x_j), x_i]) * roi_mask, and the full ConvGRU cell with its zero initial hidden state.  The GPU path's
shortcuts are therefore checked against the reference's structure, not against themselves.
"""
import os
from collections import Counter

import torch
import torch.nn.functional as F

from oracle import golden, nets

MODULE_GOLDEN = "fusion_max_v2vnet.pt"


def fusion_x():
    """The seeded input of fusion_max_v2vnet.pt: 5 agents (record_len [3, 2]), C = 64, a ragged 24 x 40 map."""
    return torch.randn(5, 64, 24, 40, generator=torch.Generator().manual_seed(41))


def load_module_golden(golden_dir):
    """fusion_max_v2vnet.pt with its seeded input `x` put back (the stored file leaves it out)."""
    d = golden.load(os.path.join(golden_dir, MODULE_GOLDEN))
    d["x"] = fusion_x()
    return d


def warp_affine_simple(src, M, dsize):
    """torch_transformation_utils.py:323-332 with align_corners=False, as oracle/nets.py restates it (fp64 theta through the
    grid, grid cast to src.dtype, bilinear taps, zeros padding), on src's device."""
    B, C, H, W = src.shape
    Ho, Wo = dsize
    th = M.to(device=src.device, dtype=torch.float64)
    xb = ((torch.arange(Wo, dtype=torch.float64, device=src.device) * 2 + 1) / Wo - 1).view(1, 1, Wo).expand(B, Ho, Wo)
    yb = ((torch.arange(Ho, dtype=torch.float64, device=src.device) * 2 + 1) / Ho - 1).view(1, Ho, 1).expand(B, Ho, Wo)
    gx = (th[:, 0, 0].view(B, 1, 1) * xb + th[:, 0, 1].view(B, 1, 1) * yb + th[:, 0, 2].view(B, 1, 1)).to(src.dtype)
    gy = (th[:, 1, 0].view(B, 1, 1) * xb + th[:, 1, 1].view(B, 1, 1) * yb + th[:, 1, 2].view(B, 1, 1)).to(src.dtype)
    ix = ((gx + 1) * W - 1) / 2
    iy = ((gy + 1) * H - 1) / 2
    x0, y0 = torch.floor(ix), torch.floor(iy)
    out = torch.zeros(B, C, Ho, Wo, dtype=src.dtype, device=src.device)
    flat = src.reshape(B, C, H * W)
    for dy, dx in ((0, 0), (0, 1), (1, 0), (1, 1)):
        xi, yi = x0 + dx, y0 + dy
        wx = (ix - x0) if dx == 1 else (x0 + 1 - ix)
        wy = (iy - y0) if dy == 1 else (y0 + 1 - iy)
        ok = (xi >= 0) & (xi < W) & (yi >= 0) & (yi < H)
        idx = (yi.clamp(0, H - 1) * W + xi.clamp(0, W - 1)).long().view(B, 1, Ho * Wo).expand(B, C, Ho * Wo)
        out = out + torch.gather(flat, 2, idx).view(B, C, Ho, Wo) * (wx * wy * ok.to(src.dtype)).unsqueeze(1)
    return out


def _regroup(x, record_len):
    rl = [int(n) for n in record_len]
    return list(torch.split(x, rl))


def max_fusion(x, record_len, affine_matrix):
    """fusion_in_one.py:87-124 (MaxFusion): warp every agent to the ego, max over agents (zeros warped in from outside count)."""
    _, C, H, W = x.shape
    out = []
    for b, xb in enumerate(_regroup(x, record_len)):
        N = xb.shape[0]
        out.append(torch.max(warp_affine_simple(xb, affine_matrix[b][0, :N], (H, W)), dim=0)[0])
    return torch.stack(out)


def conv_gru_cell(x, h, sd, p, hidden_dim, padding):
    """sub_modules/convgru.py:47-68 (ConvGRUCell.forward)."""
    cc = F.conv2d(torch.cat([x, h], 1), sd[p + ".conv_gates.weight"], sd.get(p + ".conv_gates.bias"), padding=padding)
    gamma, beta = torch.split(cc, hidden_dim, dim=1)
    reset_gate, update_gate = torch.sigmoid(gamma), torch.sigmoid(beta)
    cnm = torch.tanh(F.conv2d(torch.cat([x, reset_gate * h], 1), sd[p + ".conv_can.weight"], sd.get(p + ".conv_can.bias"),
                              padding=padding))
    return (1 - update_gate) * h + update_gate * cnm


def conv_gru(x, sd, p, hidden_dims, paddings):
    """sub_modules/convgru.py:133-190 on a length-1 batch-first sequence with hidden_state=None, i.e. the zero initial state of
    _init_hidden; x (b, c, h, w) -> the last layer's h."""
    cur = x
    for layer, (hd, pad) in enumerate(zip(hidden_dims, paddings)):
        h = torch.zeros(x.shape[0], hd, x.shape[2], x.shape[3], dtype=x.dtype, device=x.device)
        cur = conv_gru_cell(cur, h, sd, f"{p}.cell_list.{layer}", hd, pad)
    return cur


def v2vnet_fusion(x, sd, p, args, record_len, affine_matrix):
    """fusion_in_one.py:203-318 (V2VNetFusion) as written; `args` = the yaml's `v2vnet:` block."""
    _, C, H, W = x.shape
    B, L = affine_matrix.shape[:2]
    if (args["conv_gru"]["H"], args["conv_gru"]["W"]) != (H, W):
        raise ValueError(f"conv_gru H/W {(args['conv_gru']['H'], args['conv_gru']['W'])} != feature map {(H, W)}")
    nl = args["conv_gru"]["num_layers"]
    ks = args["conv_gru"]["kernel_size"]
    ks = ks if isinstance(ks, list) else [ks] * nl
    paddings = [(k[0] // 2, k[1] // 2) for k in ks]
    roi_mask = torch.zeros((B, L, L, 1, H, W), dtype=x.dtype, device=x.device)
    for b in range(B):
        for i in range(int(record_len[b])):
            roi_mask[b, i] = warp_affine_simple(torch.ones((L, 1, H, W), dtype=x.dtype, device=x.device), affine_matrix[b][i], (H, W))
    feats = _regroup(x, record_len)
    for _ in range(args["num_iteration"]):
        new = []
        for b in range(B):
            N = int(record_len[b])
            t = affine_matrix[b][:N, :N]
            upd = []
            for i in range(N):
                mask = roi_mask[b, i, :N]
                nb = warp_affine_simple(feats[b], t[i], (H, W))
                ego = feats[b][i].unsqueeze(0).repeat(N, 1, 1, 1)
                msg = nets.conv(torch.cat([nb, ego], 1), sd, p + ".msg_cnn", padding=1) * mask
                if args["agg_operator"] == "avg":
                    agg = torch.mean(msg, dim=0)
                elif args["agg_operator"] == "max":
                    agg = torch.max(msg, dim=0)[0]
                else:
                    raise ValueError("agg_operator has wrong value")
                if args["gru_flag"]:
                    out = conv_gru(torch.cat([feats[b][i], agg], 0).unsqueeze(0), sd, p + ".conv_gru", [C] * nl, paddings)[0]
                else:
                    out = feats[b][i] + agg
                upd.append(out.unsqueeze(0))
            new.append(torch.cat(upd, 0))
        feats = new
    out = torch.cat([f[0:1] for f in feats], 0)
    return F.linear(out.permute(0, 2, 3, 1), sd[p + ".mlp.weight"], sd[p + ".mlp.bias"]).permute(0, 3, 1, 2)


def heter_model_baseline(sd, args, data_dict):
    """heter_model_baseline.py:155-236 for PointPillars modalities with fusion_method att, max or v2vnet: encoder ->
    BaseBEVBackbone -> per-agent shrinker -> fusion -> (shrink) -> heads (the building blocks of oracle/nets.py)."""
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
    rl, fm = data_dict["record_len"], args["fusion_method"]
    if fm == "att":
        fused = nets.att_fusion(x, rl, affine)
    elif fm == "max":
        fused = max_fusion(x, rl, affine)
    elif fm == "v2vnet":
        fused = v2vnet_fusion(x, sd, "fusion_net", args["v2vnet"], rl, affine)
    else:
        raise NotImplementedError(fm)
    if "shrink_header" in args:
        fused = nets.downsample_conv(fused, sd, "shrink_conv", args["shrink_header"])
    return {"cls_preds": nets.conv(fused, sd, "cls_head"), "reg_preds": nets.conv(fused, sd, "reg_head"),
            "dir_preds": nets.conv(fused, sd, "dir_head"), "fused_feature": fused}
