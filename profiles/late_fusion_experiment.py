"""Late fusion of one scene: the reference-shaped eager loop (one HeterModelLate call per cav, then the post-processor, as
opencood/tools/inference_utils.py:inference_late_fusion does it) against LateFusionGraph.replay() (one batched forward for the
scene and heal_box_decode_nms_late, captured as one CUDA graph).  5 cavs of m1 (PointPillars) at the shapes of
opv2v/Single/m1_pointpillar_pretrain.yaml (+-102.4 m x +-102.4 m at 0.4 m pillars), tc32, procedural weights, synthetic 64-ring
clouds.  Needs a GPU; prints the card and its power limit, which belong beside every number taken from the output.

    python profiles/late_fusion_experiment.py [--reps 5] [--iters 20] [--out DIR]

Both arms include the host -> device copy of the raw clouds and end with the boxes on the device (the eager arm's
post-processor also reads the box count back, as the reference's does).  Times are CUDA events around blocks of `--iters`
scenes, the two arms alternating for `--reps` rounds after warm-up; the same scene gives the same boxes in both arms.
"""
import argparse
import copy
import json
import os
import subprocess
import sys
from collections import OrderedDict

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

RANGE = [-102.4, -102.4, -3, 102.4, 102.4, 1]
N_CAV = 5


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()


def m1_args():
    from oracle import late
    a = late.late_args("m1")
    a["lidar_range"] = list(RANGE)
    a["m1"]["encoder_args"]["lidar_range"] = list(RANGE)
    return a


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    opt = ap.parse_args()
    from heal_b200 import engine
    from heal_b200.graph import LateFusionGraph
    from heal_b200.data_utils.post_processor.voxel_postprocessor import VoxelPostprocessor
    from heal_b200.models.heter_model_late import HeterModelLate
    from oracle import make_golden
    from workloads import procedural, synth
    engine.set_precision("tc32")
    args = m1_args()
    model = HeterModelLate(copy.deepcopy(args)).eval()
    model.load_state_dict(procedural.make_state_dict(procedural.shapes_of(model)), strict=True)
    with torch.no_grad():
        model.cls_head_m1.bias += 2.0               # some boxes above the 0.2 score threshold
    model = model.cuda()
    params = make_golden.postprocess_params(rng=tuple(RANGE))
    pp = VoxelPostprocessor(copy.deepcopy(params), False)
    anchors = torch.from_numpy(pp.generate_anchor_box())
    sc = synth.scene(5, n_agents=N_CAV)
    poses = [synth.x_to_world(p) for p in sc["poses"]]
    ego_inv = np.linalg.inv(poses[0])
    host = OrderedDict()
    for i, pts in enumerate(sc["points"]):
        host["ego" if i == 0 else f"cav{i}"] = {
            "points": torch.from_numpy(pts).pin_memory(),
            "T": torch.from_numpy(ego_inv @ poses[i]).float()}

    def batch():
        out = OrderedDict()
        for c, h in host.items():
            p = h["points"].cuda(non_blocking=True)
            out[c] = {"inputs_m1": {"points": p, "agent_offsets": torch.tensor([0, p.shape[0]], dtype=torch.int32, device="cuda")},
                      "anchor_box": anchors, "transformation_matrix": h["T"]}
        return out

    def eager():
        b = batch()
        with torch.no_grad():
            outs = OrderedDict((c, model(v)) for c, v in b.items())
            return pp.post_process(b, outs)

    cap = sum(h["points"].shape[0] for h in host.values())
    g = LateFusionGraph(model, ["m1"] * N_CAV, {"m1": cap}, params)

    def graphed():
        g.load({c: {"inputs_m1": {"points": h["points"]}, "transformation_matrix": h["T"]} for c, h in host.items()})
        return g.replay()

    b_e, s_e = eager()
    out = graphed()
    torch.cuda.synchronize()
    k = int(out.count.item())
    same = b_e is not None and k == b_e.shape[0] and bool(torch.equal(out.boxes[:k], b_e)) and bool(torch.equal(out.scores[:k], s_e))

    def timed(fn):
        a, z = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(opt.iters):
            fn()
        z.record()
        z.synchronize()
        return a.elapsed_time(z) / opt.iters

    for _ in range(3):
        eager()
        graphed()
    torch.cuda.synchronize()
    t_e, t_g = [], []
    for _ in range(opt.reps):
        t_e.append(timed(eager))
        t_g.append(timed(graphed))
    res = {"card": card(), "cavs": N_CAV, "points_per_scene": cap, "boxes": k, "graph_boxes_equal_eager": same,
           "kernels_per_replay": g.kernels_per_replay,
           "eager_ms": [round(v, 3) for v in t_e], "graph_ms": [round(v, 3) for v in t_g],
           "eager_ms_median": round(float(np.median(t_e)), 3), "graph_ms_median": round(float(np.median(t_g)), 3)}
    print(json.dumps(res))
    if opt.out:
        os.makedirs(opt.out, exist_ok=True)
        with open(os.path.join(opt.out, "late_fusion_experiment.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
