"""HeterModelBaseline frames with fusion_method max (lidar_fcooper.yaml), v2vnet (lidar_v2vnet.yaml), cobevt
(lidar_cobevt.yaml) and v2xvit (lidar_v2xvit.yaml), and att at the same shapes for comparison: 5 agents, PointPillars on the
+-102.4 m range (512^2 pillar grid), BaseBEVBackbone [3,5,8] -> 256^2, per-agent shrink header stride 1 (fusion at 256^2) or
stride 2 (fusion at 128^2: lidar_v2vnet's conv_gru H/W = 128, and lidar_cobevt's and lidar_v2xvit's shape).

Each frame is captured as a CUDA graph (heal_b200.graph.FrameGraph) and replayed after warm-up, timed with CUDA events.  One
eager frame per model is then run with the `ops._Prof` counters on, and the per-family times are printed.  When the reference
has been built into oracle/_ref, its own MaxFusion / V2VNetFusion / CoBEVT / V2XViTFusion modules are timed eagerly (cuDNN, fp32) on random maps of the
same shapes.  The window attention's rate is also given as a share of the H100 SXM data-sheet dense BF16 tensor-core rate.
Prints the card's name and power limit first; --cases picks cases by name; --out DIR writes the records as
DIR/fusion_methods.json."""
import argparse
import copy
import json
import os
import sys
from collections import defaultdict

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))

from bottleneck_experiment import card, time_us  # noqa: E402


def model_args(method, shrink_stride):
    from workloads import configs as wcfg
    rng = wcfg.RANGE
    fused_hw = 256 // shrink_stride
    args = {"lidar_range": list(rng), "ego_modality": "m1",
            "m1": {"core_method": "point_pillar", "sensor_type": "lidar", "encoder_args": wcfg.pillar_encoder_args(rng),
                   "backbone_args": {"layer_nums": [3, 5, 8], "layer_strides": [2, 2, 2], "num_filters": [64, 128, 256],
                                     "upsample_strides": [1, 2, 4], "num_upsample_filter": [128, 128, 128]},
                   "shrink_header": {"kernal_size": [3], "stride": [shrink_stride], "padding": [1], "dim": [256], "input_dim": 384}},
            "fusion_method": method, "in_head": 256, "anchor_number": 2, "dir_args": copy.deepcopy(wcfg.DIR_ARGS)}
    if method == "att":
        args["att"] = {"feat_dim": 256}
    elif method == "v2vnet":
        args["v2vnet"] = {"num_iteration": 2, "in_channels": 256, "gru_flag": True, "agg_operator": "avg",
                          "conv_gru": {"H": fused_hw, "W": fused_hw, "num_layers": 1, "kernel_size": [[3, 3]]}}
    elif method == "cobevt":
        args["cobevt"] = {"input_dim": 256, "mlp_dim": 256, "agent_size": 5, "window_size": 4, "dim_head": 32, "drop_out": 0.1,
                          "depth": 3}
    elif method == "v2xvit":
        from oracle import v2xvit
        args["v2xvit"] = v2xvit.v2xvit_args()
    return args


def load_procedural(m):
    """Procedural values for every float key (CoBEVT's int64 relative_position_index buffers keep the module's own values)."""
    from workloads import procedural
    sd = m.state_dict()
    sd.update(procedural.make_state_dict({k: v for k, v in procedural.shapes_of(m).items() if sd[k].is_floating_point()}))
    m.load_state_dict(sd, strict=True)
    return m


CASES = [("fcooper", "max", 1), ("att@256", "att", 1), ("v2vnet", "v2vnet", 2), ("att@128", "att", 2), ("cobevt", "cobevt", 2),
         ("v2xvit", "v2xvit", 2)]
BF16_DATASHEET_TFLOPS = 989.0     # H100 SXM, dense, at up to 700 W


def frame_inputs(n_agents, seed=7):
    from heal_b200 import synth
    sc = synth.scene(seed, n_agents=n_agents)
    pts = np.concatenate(sc["points"]).astype(np.float32)
    offs = np.cumsum([0] + [p.shape[0] for p in sc["points"]]).astype(np.int32)
    return torch.from_numpy(pts).cuda(), torch.from_numpy(offs).cuda(), torch.from_numpy(sc["pairwise_t_matrix"]).cuda()


def run_case(method, stride, iters, pts, offs, pw, n_agents):
    from heal_b200 import ops
    from heal_b200.graph import FrameGraph
    from heal_b200.models.heter_model_baseline import HeterModelBaseline
    m = load_procedural(HeterModelBaseline(model_args(method, stride)).eval()).cuda()
    cap = (pts.shape[0] + 4095) // 4096 * 4096
    fg = FrameGraph(m, n_agents, cap, pw.shape)
    fg.load(pts, offs, pw)
    for _ in range(3):
        fg.replay()
    frame_us = time_us(fg.replay, iters)
    ops.PROFILE = []
    with torch.no_grad():
        m(fg.data)
    torch.cuda.synchronize()
    fam = defaultdict(lambda: [0.0, 0, 0.0])
    for name, flops, a, b, _nbytes, _launches in ops.PROFILE:
        f = fam[name]
        f[0] += a.elapsed_time(b) * 1e3
        f[1] += 1
        f[2] += float(flops() if callable(flops) else flops)
    ops.PROFILE = None
    del fg, m
    torch.cuda.empty_cache()
    return frame_us, dict(fam)


def reference_fusion_us(iters, n_agents, cases):
    """The reference's own fusion modules, eager PyTorch / cuDNN fp32, on random maps of the frame's fusion shapes."""
    from oracle import ref_shim
    if not os.path.isdir(os.path.join(ROOT, "oracle", "_ref", "opencood")):
        return None
    ref_shim.install()
    from opencood.models.fuse_modules.fusion_in_one import CoBEVT, MaxFusion, V2VNetFusion, V2XViTFusion
    from workloads import procedural
    from heal_b200 import synth
    from oracle import nets
    pw = torch.from_numpy(synth.scene(7, n_agents=n_agents, rings=4, azimuth=16)["pairwise_t_matrix"])
    aff = nets.normalize_pairwise_tfm(pw, 204.8, 204.8, 1).cuda()
    rl = torch.tensor([n_agents]).cuda()
    out = {}
    with torch.no_grad():
        if "fcooper" in cases:
            x = torch.randn(n_agents, 256, 256, 256, device="cuda")
            mx = MaxFusion().cuda()
            mx(x, rl, aff)
            out["reference MaxFusion @256"] = time_us(lambda: mx(x, rl, aff), iters)
        x = torch.randn(n_agents, 256, 128, 128, device="cuda")
        if "v2vnet" in cases:
            v = V2VNetFusion(model_args("v2vnet", 2)["v2vnet"]).eval()
            v.load_state_dict(procedural.make_state_dict(procedural.shapes_of(v)), strict=True)
            v = v.cuda()
            v(x, rl, aff)
            out["reference V2VNetFusion @128"] = time_us(lambda: v(x, rl, aff), max(1, iters // 10))
            del v
        if "cobevt" in cases:
            c = load_procedural(CoBEVT(model_args("cobevt", 2)["cobevt"]).eval()).cuda()
            c(x, rl, aff)
            out["reference CoBEVT @128"] = time_us(lambda: c(x, rl, aff), max(1, iters // 10))
            del c
        if "v2xvit" in cases:
            vt = load_procedural(V2XViTFusion(model_args("v2xvit", 2)["v2xvit"]).eval()).cuda()
            vt(x, rl, aff)
            out["reference V2XViTFusion @128"] = time_us(lambda: vt(x, rl, aff), max(1, iters // 10))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--agents", type=int, default=5)
    ap.add_argument("--precision", default="tc32", choices=["tc32", "bf16", "fp32"])
    ap.add_argument("--cases", default=",".join(c[0] for c in CASES), help="comma-separated case names")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    cases = a.cases.split(",")
    from heal_b200 import engine
    engine.set_precision(a.precision)
    rec = {"card": card(), "precision": a.precision, "agents": a.agents, "cases": {}}
    print("card:", rec["card"], "| precision:", a.precision, "| agents:", a.agents)
    pts, offs, pw = frame_inputs(a.agents)
    for name, method, stride in [c for c in CASES if c[0] in cases]:
        frame_us, fam = run_case(method, stride, a.iters, pts, offs, pw, a.agents)
        rec["cases"][name] = {"frame_us": frame_us, "families": fam}
        print(f"\n{name}: graph-replayed frame {frame_us / 1e3:.3f} ms")
        for k, (us, n, flops) in sorted(fam.items(), key=lambda kv: -kv[1][0]):
            tf = flops / us / 1e6 if us > 0 and flops else 0.0
            print(f"  {k:34s} {us:9.1f} us  {n:3d} calls  {flops / 1e9:9.1f} GFLOP  {tf:7.1f} TFLOP/s (eager, events)")
        if "window_attention" in fam:
            us, _, flops = fam["window_attention"]
            share = flops / us / 1e6 / BF16_DATASHEET_TFLOPS
            rec["cases"][name]["window_attention_share_of_bf16_datasheet"] = share
            print(f"  window_attention: {100 * share:.2f}% of the {BF16_DATASHEET_TFLOPS:.0f} TFLOP/s dense BF16 data-sheet rate")
    ref = reference_fusion_us(a.iters, a.agents, cases)
    if ref:
        rec["reference"] = ref
        for k, us in ref.items():
            print(f"{k}: {us / 1e3:.3f} ms (eager)")
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "fusion_methods.json"), "w") as fh:
            json.dump(rec, fh, indent=1)


if __name__ == "__main__":
    main()
