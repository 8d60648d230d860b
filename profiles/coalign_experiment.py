"""A HeterModelBaselineMs frame at the lidar_coalign.yaml shape: 5 agents, PointPillars on the +-102.4 m range (512^2 pillar
grid), ResNetBEVBackbone [3] stride 2 -> 256^2 x 64 per agent, fusion-backbone levels 256^2 x 64, 128^2 x 128 and 64^2 x 256,
attention fusion at each level, decode, shrink header, heads.

The frame is captured as a CUDA graph (heal_b200.graph.FrameGraph) and replayed after warm-up, timed with CUDA events.  One
eager frame is then run with the `ops._Prof` counters on: per-family times, and for `att_fuse` each level's time with the bytes
it must move (every agent's map read once, the fused map written once) as an achieved rate against the H100 SXM's 3.35 TB/s
data-sheet HBM3 bandwidth.  When the reference has been built into oracle/_ref, its own AttFusion is timed eagerly (PyTorch,
fp32) on random maps of the three level shapes.  Prints the card's name and power limit first; --out DIR writes the records as
DIR/coalign.json."""
import argparse
import copy
import json
import os
import sys
from collections import defaultdict

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))

from bottleneck_experiment import card, time_us  # noqa: E402
from fusion_methods_experiment import frame_inputs, load_procedural  # noqa: E402

HBM_DATASHEET_TBPS = 3.35         # H100 SXM5 80 GB
LEVELS = [(64, 256), (128, 128), (256, 64)]


def model_args(method="att"):
    from oracle import coalign
    from workloads import configs as wcfg
    args = coalign.coalign_args(method, lidar_range=list(wcfg.RANGE))
    args["m1"]["encoder_args"] = wcfg.pillar_encoder_args(list(wcfg.RANGE))
    args["dir_args"] = copy.deepcopy(wcfg.DIR_ARGS)
    return args


def run_frame(iters, pts, offs, pw, n_agents):
    from heal_b200 import ops
    from heal_b200.graph import FrameGraph
    from heal_b200.models.heter_model_baseline_ms import HeterModelBaselineMs
    m = load_procedural(HeterModelBaselineMs(model_args()).eval()).cuda()
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
    fam = defaultdict(lambda: [0.0, 0])
    att = []
    for name, _flops, a, b, nbytes, _launches in ops.PROFILE:
        us = a.elapsed_time(b) * 1e3
        fam[name][0] += us
        fam[name][1] += 1
        if name == "att_fuse":
            att.append({"us": us, "bytes": float(nbytes() if callable(nbytes) else nbytes)})
    ops.PROFILE = None
    del fg, m
    torch.cuda.empty_cache()
    return frame_us, dict(fam), att


def reference_att_us(iters, n_agents):
    """The reference's own AttFusion (eager PyTorch, fp32) at the three level shapes."""
    from oracle import ref_shim
    if not os.path.isdir(os.path.join(ROOT, "oracle", "_ref", "opencood")):
        return None
    ref_shim.install()
    from opencood.models.fuse_modules.fusion_in_one import AttFusion
    from heal_b200 import synth
    from oracle import nets
    pw = torch.from_numpy(synth.scene(7, n_agents=n_agents, rings=4, azimuth=16)["pairwise_t_matrix"])
    aff = nets.normalize_pairwise_tfm(pw, 204.8, 204.8, 1).cuda()
    rl = torch.tensor([n_agents]).cuda()
    out = {}
    with torch.no_grad():
        for C, hw in LEVELS:
            x = torch.randn(n_agents, C, hw, hw, device="cuda")
            f = AttFusion(C).cuda()
            f(x, rl, aff)
            out[f"reference AttFusion {hw}^2 x {C}"] = time_us(lambda: f(x, rl, aff), iters)
            del x
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--agents", type=int, default=5)
    ap.add_argument("--precision", default="tc32", choices=["tc32", "bf16", "fp32"])
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from heal_b200 import engine
    engine.set_precision(a.precision)
    rec = {"card": card(), "precision": a.precision, "agents": a.agents}
    print("card:", rec["card"], "| precision:", a.precision, "| agents:", a.agents)
    pts, offs, pw = frame_inputs(a.agents)
    frame_us, fam, att = run_frame(a.iters, pts, offs, pw, a.agents)
    rec.update({"frame_us": frame_us, "families": fam})
    print(f"\nlidar_coalign: graph-replayed frame {frame_us / 1e3:.3f} ms")
    for k, (us, n) in sorted(fam.items(), key=lambda kv: -kv[1][0]):
        print(f"  {k:34s} {us:9.1f} us  {n:3d} calls (eager, events)")
    rec["att_fuse_levels"] = []
    for (C, hw), r in zip(LEVELS, att):
        rate = r["bytes"] / r["us"] / 1e6
        lv = dict(r, level=f"{hw}^2 x {C}", tbps=rate, share_of_datasheet=rate / HBM_DATASHEET_TBPS)
        rec["att_fuse_levels"].append(lv)
        print(f"  att_fuse {hw:3d}^2 x {C:3d}: {r['us']:8.1f} us  {r['bytes'] / 1e6:7.1f} MB  {rate:5.2f} TB/s "
              f"({100 * rate / HBM_DATASHEET_TBPS:.0f}% of {HBM_DATASHEET_TBPS} TB/s)")
    ref = reference_att_us(a.iters, a.agents)
    if ref:
        rec["reference"] = ref
        for k, us in ref.items():
            print(f"{k}: {us / 1e3:.3f} ms (eager)")
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "coalign.json"), "w") as fh:
            json.dump(rec, fh, indent=1)


if __name__ == "__main__":
    main()
