"""Detection evaluation on the stream of scene_stream_experiment.py (the full-size m1m2m3m4 HeterPyramidCollab, tc32, procedural
weights, a seeded stream of 1-5-agent mixed-modality lists), two ways:
  (a) `boxes_then_eval`: SceneStream (depth 2) with the boxes back on the host, then per frame the boxes copied back to the device
      and eval_utils.caluclate_tp_fp (the function install_gpu_eval() installs) for IoU 0.3, 0.5 and 0.7: three heal_eval_tp_fp
      calls, each ending in a synchronising device-to-host copy;
  (b) `eval_in_graph`: SceneStream(eval_thresholds=(0.3, 0.5, 0.7)): each captured graph ends in heal_eval_tp_fp_counted and the
      stream's `result_stat` gains each frame as it comes back.
Both arms must give the same `result_stat` (checked).  The GT of a frame is synthetic: every third box of at least 1 m^2 of the
frame's own detections moved by up to 0.6 m, plus five boxes elsewhere (at most max_num = 150).  Needs a GPU; prints the card and its power
limit, which belong beside every number taken from the output.

    python profiles/eval_stream_experiment.py [--lists 6] [--frames 48] [--reps 3] [--out DIR]

It records frames/s (host clock around the submits, the per-frame evaluation and the drain, median of `--reps` alternating
rounds after a warm-up round), the bytes copied device-to-host per frame and the kernels per replay (and, for (a), the
evaluation kernels launched per frame outside the graph).
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import scene_graph_experiment as sge  # noqa: E402
import scene_stream_experiment as sse  # noqa: E402

THR = (0.3, 0.5, 0.7)


def gt_near(boxes, seed, cap=150):
    """Synthetic GT: every third detection of at least 1 m^2 (the random-weight heads also decode degenerate boxes, and a GT
    copied from one would meet it in a union of area 0), moved by up to 0.6 m, and five boxes elsewhere."""
    rng = np.random.default_rng(seed)
    b = boxes.numpy()
    x, y = b[:, :4, 0].astype(np.float64), b[:, :4, 1].astype(np.float64)
    area = 0.5 * np.abs((x * np.roll(y, -1, 1) - np.roll(x, -1, 1) * y).sum(1))
    near = b[area >= 1.0][::3]
    near = near + rng.uniform(-0.6, 0.6, (near.shape[0], 1, 3)).astype(np.float32) * np.float32([1, 1, 0])
    far = []
    for x, y in rng.uniform(-90, 90, (5, 2)):
        q = [(x, y), (x + 4, y), (x + 4, y + 1.8), (x, y + 1.8)]
        far.append([(a, b, z) for z in (-1.0, 1.0) for a, b in q])
    return torch.from_numpy(np.concatenate([near.reshape(-1, 8, 3), np.float32(far)])[:cap].astype(np.float32))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lists", type=int, default=6)
    ap.add_argument("--frames", type=int, default=48)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    opt = ap.parse_args()
    from heal_b200 import engine
    from heal_b200._lib import lib
    from heal_b200.graph import SceneStream
    from heal_b200.models.heter_pyramid_collab import HeterPyramidCollab
    from heal_b200.utils import eval_utils as ev
    from oracle import make_golden
    from workloads import configs, procedural
    engine.set_precision("tc32")
    who = sge.card()
    print(f"card: {who}")
    model = HeterPyramidCollab(sge.scene_args()).eval()
    model.load_state_dict(procedural.make_state_dict(procedural.shapes_of(model)), strict=True)
    model = model.cuda()
    params = make_golden.postprocess_params(rng=tuple(configs.RANGE))
    lists = sse.agent_lists(opt.lists)
    uniq = [(aml, sse.scene_batch(aml, 10 * i + r)) for i, aml in enumerate(lists) for r in range(2)]
    order = np.random.default_rng(7).integers(0, len(uniq), opt.frames)
    host = [sge.to(b, lambda t: t.pin_memory()) for _, b in uniq]
    caps = {m: (max([int(h[f"inputs_{m}"]["points"].shape[0]) for h in host if f"inputs_{m}" in h] + [1]) + 4095) // 4096 * 4096
            for m in ("m1", "m3")}
    caps.update({"m2": (sse.CAMS, sse.IMG_H, sse.IMG_W), "m4": (sse.CAMS, sse.IMG_H, sse.IMG_W)})
    pw_shape = tuple(host[0]["pairwise_t_matrix"].shape)
    print(f"lists: {lists}; {opt.frames} frames over {len(uniq)} distinct scenes")

    with torch.no_grad():
        plain = SceneStream(model, caps, pw_shape, postprocess_params=params, depth=2)
        evald = SceneStream(model, caps, pw_shape, postprocess_params=params, depth=2, eval_thresholds=THR)
        for aml in lists:
            plain.capture(aml)
            evald.capture(aml)
        boxes = []                                              # each distinct scene's boxes, copied before the slot is reused
        for h in host:
            r = plain.submit(h)
            if r is not None:
                boxes.append({k: v.clone() for k, v in r.items() if torch.is_tensor(v)})
        boxes += [{k: v.clone() for k, v in r.items() if torch.is_tensor(v)} for r in plain.drain()]
        assert len(boxes) == len(host)
        gts = [gt_near(b["boxes"][:int(b["count"][0])], i).pin_memory() for i, b in enumerate(boxes)]
        counts = [int(b["count"][0]) for b in boxes]

        stats = {}
        eval_launches = []

        def boxes_then_eval():
            stat = {t: {'tp': [], 'fp': [], 'score': [], 'gt': 0} for t in THR}
            l0 = lib.heal_launch_count()
            torch.cuda.synchronize()
            t0 = time.perf_counter()

            def evaluate(r, i):
                n = int(r["count"][0])
                det, score, gt = r["boxes"][:n].cuda(), r["scores"][:n].cuda(), gts[i].cuda()
                for t in THR:
                    ev.caluclate_tp_fp(det, score, gt, stat, t)
            sent = []
            for i in order:
                r = plain.submit(host[i])
                sent.append(i)
                if r is not None and len(sent) > 1:             # the first submit hands back the previous round's last frame
                    evaluate(r, sent[-2])
            for r, i in zip(plain.drain(), sent[-1:]):
                evaluate(r, i)
            ms = (time.perf_counter() - t0) * 1e3 / len(order)
            eval_launches.append((lib.heal_launch_count() - l0) / len(order))
            stats["boxes_then_eval"] = stat
            return ms

        def eval_in_graph():
            evald.result_stat = {t: {'tp': [], 'fp': [], 'score': [], 'gt': 0} for t in THR}
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for i in order:
                evald.submit(host[i], gts[i])
            evald.drain()
            ms = (time.perf_counter() - t0) * 1e3 / len(order)
            stats["eval_in_graph"] = evald.result_stat
            return ms

        arms = {"boxes_then_eval": boxes_then_eval, "eval_in_graph": eval_in_graph}
        for fn in arms.values():                                # warm-up round
            fn()
        runs = {k: [] for k in arms}
        for _ in range(opt.reps):
            for k, fn in arms.items():
                runs[k].append(fn())
                torch.cuda.synchronize()
        assert stats["boxes_then_eval"] == stats["eval_in_graph"], "the two arms disagree"
        assert plain.captures == evald.captures == 2 * len(lists)            # the timed rounds captured nothing
        kernels = {" ".join(k): (g.kernels_per_replay, evald.cache.slots[0][k].kernels_per_replay)
                   for k, g in plain.cache.slots[0].items()}
    med = {k: statistics.median(v) for k, v in runs.items()}
    det_per_frame = float(np.mean([counts[i] for i in order]))
    gt_per_frame = float(np.mean([gts[i].shape[0] for i in order]))
    d2h = {"boxes_then_eval": plain.d2h_bytes + len(THR) * (4 + 5 * det_per_frame), "eval_in_graph": evald.d2h_bytes}
    res = {"card": who, "precision": "tc32", "lists": lists, "frames": int(opt.frames),
           "detections_per_frame": det_per_frame, "gt_per_frame": gt_per_frame,
           "ms_per_frame": med, "ms_per_frame_all": runs, "frames_per_s": {k: 1e3 / v for k, v in med.items()},
           "d2h_bytes_per_frame": d2h,
           "kernels_per_replay_without_and_with_eval": kernels,
           "eval_kernels_per_frame_outside_the_graph": {"boxes_then_eval": eval_launches[-1], "eval_in_graph": 0},
           "ap": {str(t): sse_ap(stats["eval_in_graph"], t) for t in THR}}
    print(f"{'arm':<18}{'ms/frame':>10}{'frames/s':>10}{'D2H B/frame':>13}")
    for k, v in med.items():
        print(f"{k:<18}{v:>10.3f}{1e3 / v:>10.1f}{d2h[k]:>13.0f}")
    print(f"kernels per replay (without, with eval): {kernels}")
    print(f"detections / GT per frame: {det_per_frame:.1f} / {gt_per_frame:.1f}; AP {res['ap']}")
    if opt.out:
        os.makedirs(opt.out, exist_ok=True)
        with open(os.path.join(opt.out, "eval_stream_experiment.json"), "w") as fh:
            json.dump(res, fh, indent=1)


def sse_ap(stat, t):
    from oracle import eval as oev
    return oev.calculate_ap(stat, t)


if __name__ == "__main__":
    main()
