"""Late fusion over a stream whose cav list changes from frame to frame, evaluated as inference.py does it: the eager path
(`forward_late` -> ops.box_decode_nms_multi -> the eval_utils drop-in `caluclate_tp_fp` at 0.3 / 0.5 / 0.7, per frame, what
`inference_late_fusion` + `eval_utils` run with the GPU post-processor and evaluation installed) against LateFusionStream at
depth 2 (one captured graph per cav list and slot, evaluated inside the graph).  The model is HeterModelLate with one m1
(PointPillars) at the shapes of opv2v/Single/m1_pointpillar_pretrain.yaml (+-102.4 m at 0.4 m pillars), tc32, procedural
weights; a seeded stream of `--frames` frames draws 1 to 5 cavs of synthetic 64-ring clouds from `--scenes` scenes.  Needs a
GPU; the card and its power limit are read in the same run and written beside the numbers.

    python profiles/late_stream_experiment.py [--frames 40] [--scenes 6] [--reps 3] [--out DIR]

It records frames/s over the stream (median of `--reps` alternating rounds after a warm-up round; host clock around work
that ends in a device synchronise / the stream's drain), one-frame latency (one frame in an empty pipeline: submit + flush,
against one eager frame), that both paths give identical boxes and scores for every frame, and that both `result_stat`s are
equal.  Both arms start from pinned host clouds and host poses.  Writes late_stream_experiment_h100.json under `--out`.
"""
import argparse
import copy
import json
import os
import statistics
import sys
import time
from collections import OrderedDict

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import late_fusion_experiment as lfe  # noqa: E402

THR = (0.3, 0.5, 0.7)
MAX_CAV = 5


def gt_for(boxes, seed):
    """GT corners of a frame: every second detection moved by up to 0.6 m, plus ten boxes elsewhere."""
    from oracle.make_golden_eval import rect
    rng = np.random.default_rng(seed)
    near = boxes[::2].cpu().numpy()
    near = near + rng.uniform(-0.6, 0.6, (near.shape[0], 1, 3)).astype(np.float32) * np.float32([1, 1, 0])
    far = np.stack([rect(x, x + 4, y, y + 1.8) for x, y in rng.uniform(-90, 90, (10, 2))])
    return torch.from_numpy(np.concatenate([near.reshape(-1, 8, 3), far]).astype(np.float32)[:300])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=40)
    ap.add_argument("--scenes", type=int, default=6)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    opt = ap.parse_args()
    from heal_b200 import engine, ops
    from heal_b200.data_utils.post_processor.voxel_postprocessor import VoxelPostprocessor, decode_kwargs
    from heal_b200.graph import LateFusionStream
    from heal_b200.models.heter_model_late import HeterModelLate
    from heal_b200.utils import eval_utils as ev
    from oracle import make_golden
    from workloads import procedural, synth
    engine.set_precision("tc32")
    who = lfe.card()
    print(f"card: {who}")
    model = HeterModelLate(copy.deepcopy(lfe.m1_args())).eval()
    model.load_state_dict(procedural.make_state_dict(procedural.shapes_of(model)), strict=True)
    with torch.no_grad():
        model.cls_head_m1.bias += 2.0               # some boxes above the 0.2 score threshold
    model = model.cuda()
    params = make_golden.postprocess_params(rng=tuple(lfe.RANGE))
    anchors = torch.from_numpy(VoxelPostprocessor(copy.deepcopy(params), False).generate_anchor_box()).float().cuda()
    decode = decode_kwargs(params, True)

    scenes = []
    for s in range(opt.scenes):
        sc = synth.scene(11 + s, n_agents=MAX_CAV)
        poses = [synth.x_to_world(p) for p in sc["poses"]]
        ego_inv = np.linalg.inv(poses[0])
        scenes.append([(torch.from_numpy(pts).pin_memory(), torch.from_numpy(ego_inv @ poses[i]).float())
                       for i, pts in enumerate(sc["points"])])
    rng = np.random.default_rng(3)
    stream_of = [(int(rng.integers(0, opt.scenes)), int(rng.integers(1, MAX_CAV + 1))) for _ in range(opt.frames)]
    host = []
    for s, k in stream_of:                            # the late batch of frame i: the first k cavs of scene s, pinned clouds
        host.append(OrderedDict(("ego" if i == 0 else f"cav{i}", {
            "inputs_m1": {"points": p, "agent_offsets": torch.tensor([0, p.shape[0]], dtype=torch.int32).pin_memory()},
            "transformation_matrix": T}) for i, (p, T) in enumerate(scenes[s][:k])))
    cap = (max(sum(c["inputs_m1"]["points"].shape[0] for c in b.values()) for b in host) + 4095) // 4096 * 4096

    def to_device(b):
        return OrderedDict((c, {"inputs_m1": {k: v.cuda(non_blocking=True) for k, v in v["inputs_m1"].items()},
                                "transformation_matrix": v["transformation_matrix"]}) for c, v in b.items())

    def eager_frame(b, gt, stat):
        with torch.no_grad():
            heads = model.forward_late(to_device(b))
        post = ops.box_decode_nms_multi([{"cls": h["cls_preds"], "reg": h["reg_preds"], "dir": h["dir_preds"], "anchors": anchors,
                                          "transform": b[c]["transformation_matrix"]} for c, h in heads.items()],
                                        **decode)
        n = int(post.count.item())
        boxes, scores = post.boxes[:n], post.scores[:n]
        for t in (THR if stat is not None else ()):
            if n:
                ev.caluclate_tp_fp(boxes, scores, gt, stat, t)
            else:                                     # the reference's det_boxes None: the GT count only
                ev.append_frame(stat, t, torch.zeros(0), torch.zeros(0), gt.shape[0])
        return boxes, scores

    def new_stat():
        return {t: {'tp': [], 'fp': [], 'score': [], 'gt': 0} for t in THR}

    # GT from a first eager pass, then both arms over the same frames: identical boxes and result_stat
    first = [eager_frame(b, None, None) for b in host]
    gts = [gt_for(boxes, 100 + i).cuda() for i, (boxes, _) in enumerate(first)]
    stream = LateFusionStream(model, {"m1": cap}, MAX_CAV, params, depth=2, eval_thresholds=THR, gt_capacity=300)
    for k in range(1, MAX_CAV + 1):
        stream.capture(["m1"] * k)
    captures = stream.captures
    stat_e, got_e = new_stat(), []
    for b, gt in zip(host, gts):
        boxes, scores = eager_frame(b, gt, stat_e)
        got_e.append((boxes.cpu(), scores.cpu()))
    got_s = []
    for b, gt in zip(host, gts):
        r = stream.submit(b, gt)
        if r is not None:
            got_s.append({k: v.clone() for k, v in r.items() if torch.is_tensor(v)})
    got_s += [{k: v.clone() for k, v in r.items() if torch.is_tensor(v)} for r in stream.drain()]
    same = len(got_s) == len(got_e) and all(
        int(r["count"][0]) == e[0].shape[0] and torch.equal(r["boxes"][:e[0].shape[0]], e[0])
        and torch.equal(r["scores"][:e[0].shape[0]], e[1]) for r, e in zip(got_s, got_e))
    stat_same = stream.result_stat == stat_e
    print(f"boxes identical: {same}; result_stat identical: {stat_same}")

    def eager():
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        stat = new_stat()
        for b, gt in zip(host, gts):
            eager_frame(b, gt, stat)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3 / len(host)

    def streamed():
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for b, gt in zip(host, gts):
            stream.submit(b, gt)
        stream.drain()
        return (time.perf_counter() - t0) * 1e3 / len(host)

    def latency(one):
        out = []
        for b, gt in zip(host, gts):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            one(b, gt)
            torch.cuda.synchronize()
            out.append((time.perf_counter() - t0) * 1e3)
        return statistics.median(out)

    def stream_one(b, gt):
        stream.submit(b, gt)
        stream.flush()

    arms = {"eager": eager, "late_stream": streamed}
    for fn in arms.values():                                  # warm-up round
        fn()
    runs = {k: [] for k in arms}
    for _ in range(opt.reps):
        for k, fn in arms.items():
            runs[k].append(fn())
    lat = {"eager": latency(lambda b, gt: eager_frame(b, gt, new_stat())), "late_stream": latency(stream_one)}
    assert stream.captures == captures                        # the timed rounds captured nothing
    med = {k: statistics.median(v) for k, v in runs.items()}
    res = {"card": who, "precision": "tc32", "frames": len(host), "cavs_per_frame": [k for _, k in stream_of],
           "point_capacity": cap, "boxes_per_frame": [e[0].shape[0] for e in got_e],
           "boxes_identical": bool(same), "result_stat_identical": bool(stat_same),
           "ms_per_frame": med, "ms_per_frame_all": runs, "frames_per_s": {k: 1e3 / v for k, v in med.items()},
           "one_frame_latency_ms": lat}
    print(f"{'arm':<14}{'ms/frame':>10}{'frames/s':>10}{'latency ms':>12}")
    for k, v in med.items():
        print(f"{k:<14}{v:>10.3f}{1e3 / v:>10.1f}{lat[k]:>12.3f}")
    if opt.out:
        os.makedirs(opt.out, exist_ok=True)
        with open(os.path.join(opt.out, "late_stream_experiment_h100.json"), "w") as fh:
            json.dump(res, fh, indent=1)
    if not (same and stat_same):
        raise SystemExit("the two paths disagree")


if __name__ == "__main__":
    main()
