"""Per-frame detection evaluation (eval_utils.caluclate_tp_fp at IoU 0.3, 0.5 and 0.7) on the GPU against the reference's host loop.
Needs a GPU; prints the card and its power limit, which belong beside every number taken from the output.

    python profiles/eval_experiment.py [--frames 200] [--ref-frames 2] [--reps 2] [--out DIR]

Frames are OPV2V-like (oracle/make_golden_eval.random_frame): K detections after NMS and G GT boxes at four shipped-size points
(K, G) = (50, 30), (120, 60), (200, 100), (300, 150).  Per shape, alternating for `--reps` rounds:
1. drop-in: heal_b200.utils.eval_utils.caluclate_tp_fp called three times per frame as inference.py calls it, on CUDA tensors,
   including the device-to-host copy of each call; host clock over `--frames` frames after warm-up.
2. device: heal_eval_tp_fp alone (ops.eval_tp_fp, one threshold and three thresholds per launch), CUDA events over `--frames`
   launches.
3. reference: the unmodified opencood.utils.eval_utils.caluclate_tp_fp from oracle/_ref, three calls per frame on CPU tensors,
   one host thread, over `--ref-frames` frames; with real shapely when it is importable, else with the QuadPolygon stand-in of
   oracle/postprocess.py (labelled "stand-in": a numpy polygon clip, not GEOS).
Whether the drop-in's lists equal the reference's is recorded for every reference frame (`lists_equal`).
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

SHAPES = ((50, 30), (120, 60), (200, 100), (300, 150))
THR = (0.3, 0.5, 0.7)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()


def reference_module():
    """(eval_utils, label): real shapely if importable, else QuadPolygon installed as shapely.geometry.Polygon"""
    from oracle import ref_shim
    try:
        import shapely.geometry  # noqa: F401
        ref_shim.install()
        label = "shapely " + __import__("shapely").__version__
    except ImportError:
        from oracle.make_golden_eval import install_reference
        install_reference()
        label = "stand-in (oracle.postprocess.QuadPolygon, shapely not installed)"
    import opencood.utils.eval_utils as eu
    return eu, label


def stat():
    return {t: {"tp": [], "fp": [], "gt": 0, "score": []} for t in THR}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--ref-frames", type=int, default=2)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    from heal_b200 import ops
    from heal_b200.utils import eval_utils as ev
    from oracle.make_golden_eval import random_frame
    eu, label = reference_module()
    out = {"card": card(), "reference": label, "shapes": []}
    print(f"card: {out['card']}\nreference arm: {label}")
    for K, G in SHAPES:
        frames = []
        for s in range(8):
            d, sc, g = random_frame(100 * K + s, K, G, "hwl", bool(s % 2))
            frames.append((torch.from_numpy(d), torch.from_numpy(sc), torch.from_numpy(g)))
        gpu = [(d.cuda(), s.cuda(), g.cuda()) for d, s, g in frames]
        row = {"K": K, "G": G, "dropin_ms": [], "device_us_1thr": [], "device_us_3thr": [], "reference_ms": [], "lists_equal": []}
        for d, s, g in gpu:                                 # warm-up
            for t in THR:
                ev.caluclate_tp_fp(d, s, g, stat(), t)
        buf = None
        for rep in range(a.reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for i in range(a.frames):
                d, s, g = gpu[i % len(gpu)]
                st = stat()
                for t in THR:
                    ev.caluclate_tp_fp(d, s, g, st, t)
            row["dropin_ms"].append((time.perf_counter() - t0) * 1e3 / a.frames)
            for key, thr in (("device_us_1thr", THR[:1]), ("device_us_3thr", THR)):
                buf = ops.eval_tp_fp(*gpu[0], thr, buf)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for i in range(a.frames):
                    buf = ops.eval_tp_fp(*gpu[i % len(gpu)], thr, buf)
                e1.record()
                torch.cuda.synchronize()
                row[key].append(e0.elapsed_time(e1) * 1e3 / a.frames)
            t_ref = 0.0
            for i in range(a.ref_frames):
                d, s, g = frames[i % len(frames)]
                st_ref, st_gpu = stat(), stat()
                t0 = time.perf_counter()
                for t in THR:
                    eu.caluclate_tp_fp(d, s, g, st_ref, t)
                t_ref += time.perf_counter() - t0
                for t in THR:
                    ev.caluclate_tp_fp(*gpu[i % len(gpu)], st_gpu, t)
                row["lists_equal"].append(st_ref == st_gpu)
            row["reference_ms"].append(t_ref * 1e3 / a.ref_frames)
        out["shapes"].append(row)
        print(f"K={K:4d} G={G:4d}  drop-in, 3 calls / frame: {min(row['dropin_ms']):8.3f} ms   "
              f"heal_eval_tp_fp: {min(row['device_us_1thr']):7.1f} us (1 thr) {min(row['device_us_3thr']):7.1f} us (3 thr)   "
              f"reference loop, 3 calls / frame: {min(row['reference_ms']):9.1f} ms   all reps: {row}")
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "eval_experiment.json"), "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
