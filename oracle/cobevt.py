"""ORACLE — TEST INFRASTRUCTURE ONLY.  A literal restatement of the reference's CoBEVT fusion (opencood/models/fuse_modules/
fusion_in_one.py:374-429; swap_fusion_modules.py:13-192 Attention / SwapFusionBlockMask; sub_modules/base_transformer.py
PreNormResidual / FeedForward; fuse_utils.py:13-64 regroup) and of HeterModelBaseline with `fusion_method: cobevt`, in plain
functional PyTorch over a flat state_dict.  The einops rearranges are written as reshape / permute; runs on any device.
Pinned against the reference's own modules by oracle/make_golden_cobevt.py -> tests/golden/{fusion_cobevt,
heter_model_baseline_cobevt_small}.pt.xz.

The state dict holds the float parameters only: relative_position_index is rebuilt here, as the reference builds it.
"""
import os
from collections import Counter

import numpy as np
import torch
import torch.nn.functional as F

from oracle import fusion_methods, golden, nets

MODULE_GOLDEN = "fusion_cobevt.pt"
INDEX_KEY = "relative_position_index"


def cobevt_args(C, depth, agent_size, mlp_dim=None):
    """`cobevt:` block of opv2v/LiDAROnly/lidar_cobevt.yaml (input_dim 256, mlp_dim 256, window 4, dim_head 32, depth 3) with the
    channel count, depth and agent_size of a test."""
    return {"input_dim": C, "mlp_dim": mlp_dim or C, "agent_size": agent_size, "window_size": 4, "dim_head": 32,
            "drop_out": 0.1, "depth": depth}


def module_cases():
    """name -> (args, seeded input shape, record_len, pairwise-pose scenes) of fusion_cobevt.pt."""
    two = [[[0, 0, 0, 0, 0, 0], [3.0, -1.5, 0, 0, 35, 0], [-4.0, 2.5, 0, 0, -120, 0]],
           [[0, 0, 0, 0, 0, 0], [0.07, 0.05, 0, 0, 0, 0]]]
    return {
        "c64": (cobevt_args(64, 2, 5, mlp_dim=128), (5, 64, 24, 40), [3, 2], two, 5),
        "c256": (cobevt_args(256, 3, 5), (5, 256, 16, 24), [3, 2], two, 5),
        "l2": (cobevt_args(64, 2, 2, mlp_dim=128), (3, 64, 24, 40), [2, 1],
               [[[0, 0, 0, 0, 0, 0], [2.0, 1.0, 0, 0, 60, 0]], [[0, 0, 0, 0, 0, 0]]], 2),
    }


def case_inputs(name):
    """(x, record_len, pairwise_t_matrix) of case `name`: x is drawn from a seeded generator (not stored in the golden)."""
    from workloads import synth
    args, shape, rl, scenes, L = module_cases()[name]
    seed = {"c64": 51, "c256": 52, "l2": 53}[name]
    x = torch.randn(*shape, generator=torch.Generator().manual_seed(seed))
    pw = np.stack([synth.pairwise_t_matrix(p, L) for p in scenes])
    return x, torch.tensor(rl), torch.from_numpy(pw)


def case_affine(pw):
    return nets.normalize_pairwise_tfm(pw, 9.6, 16.0, 1)


def load_module_golden(golden_dir):
    return golden.load(os.path.join(golden_dir, MODULE_GOLDEN))


def float_shapes(shapes):
    """The procedural part of a parameter table: every key but the int64 relative_position_index buffers."""
    return {k: v for k, v in shapes.items() if not k.endswith(INDEX_KEY)}


def relative_position_index(agent_size, window_size):
    """swap_fusion_modules.py:61-83: token pairs (i, j), tokens (agent, w1, w2) -> index into the (Δagent, Δw1, Δw2) table."""
    ws = [agent_size, window_size, window_size]
    coords = torch.stack(torch.meshgrid(torch.arange(ws[0]), torch.arange(ws[1]), torch.arange(ws[2]), indexing="ij"))
    coords_flatten = torch.flatten(coords, 1)
    rel = coords_flatten[:, :, None] - coords_flatten[:, None, :]
    rel = rel.permute(1, 2, 0).contiguous()
    rel[:, :, 0] += ws[0] - 1
    rel[:, :, 1] += ws[1] - 1
    rel[:, :, 2] += ws[2] - 1
    rel[:, :, 0] *= (2 * ws[1] - 1) * (2 * ws[2] - 1)
    rel[:, :, 1] *= 2 * ws[2] - 1
    return rel.sum(-1)


def regroup(x, record_len, max_len):
    """fuse_utils.py:13-64: (sumN, C, H, W) -> (B, L, C, H, W) zero-padded, mask (B, L)."""
    feats, mask = [], []
    for f in torch.split(x, [int(n) for n in record_len]):
        pad = max_len - f.shape[0]
        mask.append([1] * f.shape[0] + [0] * pad)
        feats.append(torch.cat([f, torch.zeros(pad, *f.shape[1:], dtype=f.dtype, device=f.device)], 0))
    return torch.stack(feats), torch.tensor(mask, device=x.device)


def attention(x, sd, p, dim_head, agent_size, window_size, mask):
    """swap_fusion_modules.py:87-128.  x (b, l, X, Y, w1, w2, d); mask (b, X, Y, w1, w2, 1, l)."""
    b, l, X, Y, w1, w2, d = x.shape
    h = d // dim_head
    t = x.permute(0, 2, 3, 1, 4, 5, 6).reshape(b * X * Y, l * w1 * w2, d)         # (b x y) (l w1 w2) d
    q, k, v = F.linear(t, sd[p + ".to_qkv.weight"]).chunk(3, dim=-1)
    q, k, v = (u.reshape(u.shape[0], u.shape[1], h, dim_head).permute(0, 2, 1, 3) for u in (q, k, v))
    q = q * dim_head ** -0.5
    sim = torch.einsum("bhid,bhjd->bhij", q, k)
    idx = relative_position_index(agent_size, window_size).to(x.device)
    bias = F.embedding(idx, sd[p + ".relative_position_bias_table.weight"])        # i j h
    sim = sim + bias.permute(2, 0, 1)
    m = mask.permute(0, 1, 2, 5, 6, 3, 4).reshape(b * X * Y, mask.shape[5], l * w1 * w2).unsqueeze(1)
    sim = sim.masked_fill(m == 0, -float("inf"))
    attn = sim.softmax(dim=-1)
    out = torch.einsum("bhij,bhjd->bhid", attn, v)
    out = out.permute(0, 2, 1, 3).reshape(b * X * Y, l, w1, w2, d)                # b l w1 w2 (h d)
    out = F.linear(out, sd[p + ".to_out.0.weight"])
    return out.reshape(b, X, Y, l, w1, w2, d).permute(0, 3, 1, 2, 4, 5, 6)


def layer_norm(x, sd, p):
    return F.layer_norm(x, (x.shape[-1],), sd[p + ".weight"], sd[p + ".bias"], 1e-5)


def feed_forward(x, sd, p):
    """base_transformer.py:27-39 in eval (Dropout = identity): Linear -> exact GELU -> Linear."""
    y = F.gelu(F.linear(x, sd[p + ".net.0.weight"], sd[p + ".net.0.bias"]))
    return F.linear(y, sd[p + ".net.3.weight"], sd[p + ".net.3.bias"])


def _sublayers(x, mask, sd, p, kind, args):
    x = attention(layer_norm(x, sd, f"{p}.{kind}_attention.norm"), sd, f"{p}.{kind}_attention.fn", args["dim_head"],
                  args["agent_size"], args["window_size"], mask) + x
    return feed_forward(layer_norm(x, sd, f"{p}.{kind}_ffd.norm"), sd, f"{p}.{kind}_ffd.fn") + x


def swap_fusion_block_mask(x, mask, sd, p, args):
    """swap_fusion_modules.py:165-192.  x (b, m, d, H, W); mask (b, H, W, 1, l)."""
    b, m, d, H, W = x.shape
    w, L = args["window_size"], mask.shape[-1]
    # window: 'b (x w1) (y w2) e l -> b x y w1 w2 e l', 'b m d (x w1) (y w2) -> b m x y w1 w2 d'
    mw = mask.reshape(b, H // w, w, W // w, w, 1, L).permute(0, 1, 3, 2, 4, 5, 6)
    xw = x.reshape(b, m, d, H // w, w, W // w, w).permute(0, 1, 3, 5, 4, 6, 2)
    xw = _sublayers(xw, mw, sd, p, "window", args)
    x = xw.permute(0, 1, 6, 2, 4, 3, 5).reshape(b, m, d, H, W)
    # grid: 'b (w1 x) (w2 y) e l -> b x y w1 w2 e l', 'b m d (w1 x) (w2 y) -> b m x y w1 w2 d'
    mg = mask.reshape(b, w, H // w, w, W // w, 1, L).permute(0, 2, 4, 1, 3, 5, 6)
    xg = x.reshape(b, m, d, w, H // w, w, W // w).permute(0, 1, 4, 6, 3, 5, 2)
    xg = _sublayers(xg, mg, sd, p, "grid", args)
    return xg.permute(0, 1, 6, 4, 2, 5, 3).reshape(b, m, d, H, W)


def cobevt_fusion(x, sd, p, args, record_len, affine_matrix):
    """fusion_in_one.py:409-429 (CoBEVT.forward) in eval; `args` = the yaml's `cobevt:` block."""
    _, C, H, W = x.shape
    B, L = affine_matrix.shape[:2]
    feats, mask = regroup(x, record_len, L)
    com_mask = mask[:, None, None, None, :].expand(B, H, W, 1, L)
    x = torch.stack([fusion_methods.warp_affine_simple(feats[b], affine_matrix[b, 0], (H, W)) for b in range(B)])
    for i in range(args["depth"]):
        x = swap_fusion_block_mask(x, com_mask, sd, f"{p}.layers.{i}", args)
    y = layer_norm(x.mean(dim=1).permute(0, 2, 3, 1), sd, p + ".mlp_head.2")
    return F.linear(y, sd[p + ".mlp_head.3.weight"], sd[p + ".mlp_head.3.bias"]).permute(0, 3, 1, 2)


def heter_model_baseline(sd, args, data_dict):
    """heter_model_baseline.py:155-236 for PointPillars modalities with fusion_method cobevt (the building blocks of
    oracle/nets.py, as oracle/fusion_methods.heter_model_baseline uses them for the other methods)."""
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
    assert args["fusion_method"] == "cobevt"
    fused = cobevt_fusion(x, sd, "fusion_net", args["cobevt"], data_dict["record_len"], affine)
    if "shrink_header" in args:
        fused = nets.downsample_conv(fused, sd, "shrink_conv", args["shrink_header"])
    return {"cls_preds": nets.conv(fused, sd, "cls_head"), "reg_preds": nets.conv(fused, sd, "reg_head"),
            "dir_preds": nets.conv(fused, sd, "dir_head"), "fused_feature": fused}
