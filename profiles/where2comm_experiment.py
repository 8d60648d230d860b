"""Where2comm and Who2com at the C3 fusion shape (5 agents, 256 x 256 fused map, C = 256).

1. `heal_ego_mha` per call (CUDA events) for fp32, split-bf16 and bf16 storage, with its algorithmic bytes (q and out once,
   the k | v projection once per agent) as bytes/s against the 3.35 TB/s HBM3 data-sheet rate.
2. A/B of Where2comm's attention stage, alternating, three rounds, in tc32 and bf16:
     fused:       warp the ego -> q 1x1 conv -> bias-free k|v 1x1 conv on the unwarped maps -> heal_ego_mha
     composition: warp every agent -> one C -> 3C 1x1 conv (q rows pre-scaled) -> heal_cav_attention(ego_only=1)
   with the outputs of the two compared.
3. Graph-captured HeterModelBaseline frames (heal_b200.graph.FrameGraph) with att, where2comm and who2com in tc32 and bf16.
Prints the card's name and power limit first; --out DIR writes the records as DIR/where2comm.json."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))

from bottleneck_experiment import card, time_us  # noqa: E402
from fusion_methods_experiment import frame_inputs, load_procedural, model_args  # noqa: E402

HBM_TBPS = 3.35          # H100 SXM HBM3, data sheet
N_AGENTS, HW, C = 5, 256, 256


def scene():
    from heal_b200 import synth
    from oracle import nets
    pw = torch.from_numpy(synth.scene(7, n_agents=N_AGENTS, rings=4, azimuth=16)["pairwise_t_matrix"])
    aff = nets.normalize_pairwise_tfm(pw, 204.8, 204.8, 1).cuda()
    return aff[:, 0, :N_AGENTS].reshape(N_AGENTS, 2, 3).contiguous()


def ego_mha_bytes(fmt):
    from heal_b200.ops import BPE
    return HW * HW * C * (2 * BPE[fmt] + N_AGENTS * 2 * BPE[fmt])


def time_kernel(iters, theta):
    from heal_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(1)
    rec = {}
    for fmt in ("f32", "split", "bf16"):
        q = ops.convert(ops.Act(torch.randn(1, HW, HW, C, device="cuda", generator=g), "f32"), fmt)
        kv = ops.convert(ops.Act(torch.randn(N_AGENTS, HW, HW, 2 * C, device="cuda", generator=g), "f32"), fmt)
        bias = torch.randn(2 * C, device="cuda", generator=g)
        out = ops.act_empty(1, HW, HW, C, fmt, q.device)
        fn = lambda: ops.ego_mha(q, kv, bias, theta, [N_AGENTS], out=out)      # noqa: E731
        for _ in range(3):
            fn()
        us = time_us(fn, iters)
        nbytes = ego_mha_bytes(fmt)
        rec[fmt] = {"us": us, "bytes": nbytes, "GBps": nbytes / us / 1e3, "share_of_hbm": nbytes / us / 1e6 / HBM_TBPS}
        print(f"heal_ego_mha {fmt:5s}: {us:8.1f} us  {nbytes / 1e6:7.1f} MB  {nbytes / us / 1e3:7.1f} GB/s "
              f"({100 * rec[fmt]['share_of_hbm']:.1f}% of {HBM_TBPS} TB/s)")
        del q, kv, out
    return rec


def ab(precision, iters, theta):
    from heal_b200 import engine, ops
    from heal_b200.engine import conv_bn_act
    from heal_b200.models.fuse_modules.fusion_in_one import Where2commFusion, _conv_from
    from workloads import procedural
    engine.set_precision(precision)
    fmt = engine.act_fmt()
    m = Where2commFusion(C).eval()
    m.load_state_dict(procedural.make_state_dict(procedural.shapes_of(m)), strict=True)
    m = m.cuda()
    q_conv, kv_conv, kv_bias, _, _, _ = m._packed()
    w = m.mha_fusion.attn.in_proj_weight.detach().double()
    b = m.mha_fusion.attn.in_proj_bias.detach().double()
    s = (1.0 / (C // 8)) ** 0.5
    qkv_conv = _conv_from(torch.cat([w[:C] * s, w[C:]]).float()[:, :, None, None], torch.cat([b[:C] * s, b[C:]]).float(), 0)
    x = ops.convert(ops.Act(torch.randn(N_AGENTS, HW, HW, C, device="cuda", generator=torch.Generator(device="cuda")
                                        .manual_seed(2)), "f32"), fmt)
    rl = [N_AGENTS]

    def fused():
        ego = ops.warp_affine(x, [0], theta[:1], out_fmt=fmt)
        return ops.ego_mha(conv_bn_act(ego, q_conv), conv_bn_act(x, kv_conv), kv_bias, theta, rl, out_fmt=fmt)

    def composition():
        X = ops.warp_affine(x, list(range(N_AGENTS)), theta, out_fmt=fmt)
        return ops.cav_attention(conv_bn_act(X, qkv_conv), rl, ego_only=True, out_fmt=fmt)

    with torch.no_grad():
        a, c = ops.act_to_nchw(fused()), ops.act_to_nchw(composition())
        err = (a - c).abs().max().item() / max(c.abs().max().item(), 1e-30)
        for fn in (fused, composition):
            for _ in range(3):
                fn()
        rounds = {"fused": [], "composition": []}
        for _ in range(3):
            rounds["fused"].append(time_us(fused, iters))
            rounds["composition"].append(time_us(composition, iters))
    print(f"A/B {precision}: fused {[round(v, 1) for v in rounds['fused']]} us, composition "
          f"{[round(v, 1) for v in rounds['composition']]} us, max rel diff of the outputs {err:.2e}")
    return {"rounds_us": rounds, "max_rel_diff": err}


def frame(method, precision, iters, pts, offs, pw):
    from heal_b200 import engine
    from heal_b200.graph import FrameGraph
    from heal_b200.models.heter_model_baseline import HeterModelBaseline
    engine.set_precision(precision)
    args = model_args("att", 1)
    if method != "att":
        args["fusion_method"] = method
        del args["att"]
        args[method] = C
    m = load_procedural(HeterModelBaseline(args).eval()).cuda()
    fg = FrameGraph(m, N_AGENTS, (pts.shape[0] + 4095) // 4096 * 4096, pw.shape)
    fg.load(pts, offs, pw)
    for _ in range(3):
        fg.replay()
    us = time_us(fg.replay, iters)
    del fg, m
    torch.cuda.empty_cache()
    print(f"frame {method:10s} {precision}: {us / 1e3:.3f} ms (graph replay)")
    return us


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    rec = {"card": card(), "agents": N_AGENTS, "hw": HW, "C": C}
    print("card:", rec["card"])
    theta = scene()
    rec["ego_mha"] = time_kernel(a.iters * 4, theta)
    rec["ab"] = {p: ab(p, a.iters, theta) for p in ("tc32", "bf16")}
    pts, offs, pw = frame_inputs(N_AGENTS)
    rec["frames_us"] = {f"{m}/{p}": frame(m, p, a.iters, pts, offs, pw)
                        for p in ("tc32", "bf16") for m in ("att", "where2comm", "who2com")}
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "where2comm.json"), "w") as fh:
            json.dump(rec, fh, indent=1)


if __name__ == "__main__":
    main()
