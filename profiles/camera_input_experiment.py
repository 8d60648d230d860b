"""The camera agent's image stage on the GPU.  Needs a GPU; prints the card and its power limit, which belong beside every
number taken from the output.

    python profiles/camera_input_experiment.py [--reps 3] [--iters 20] [--out DIR]

1. heal_camera_input per launch at the three shipped inference shapes (600x800 -> 384x512, 600x800 -> 336x448,
   1080x1920 -> 288x512) with 4 cams x 5 agents = 20 frames in one launch, both output layouts, against the bytes the kernel must
   move: every source pixel the crop window needs read once (uint8) and n_img * 3 * fH * fW * 4 B written (64/3 of that for the
   space-to-depth layout, which also writes the zero fourth plane).  CUDA events over `--iters` launches after warm-up.
2. The C4 camera encoder (Lift-Splat-Shoot, ResNet-101 trunk, 2 agents x 4 cams, 256x704, bf16 as bench.py runs C4) captured with
   GraphedCall, fed raw 600x800 uint8 frames against the same encoder fed fp32 `imgs` (n, 4, 3, 256, 704) that the host has
   already resized, cropped and normalised.  One frame = the host -> device copy of the inputs from pinned memory + replay,
   timed with CUDA events; the two arms alternate for `--reps` rounds.  The H2D bytes per frame are printed for both.
3. For context: the host time of PIL resize + crop + ToTensor + Normalize (the reference's img_transform and normalize_img) per
   600x800 camera frame on this machine's CPU, single thread as in a DataLoader worker.
"""
import argparse
import copy
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

SHAPES = (("600x800 -> 384x512", 600, 800, {"H": 600, "W": 800, "final_dim": [384, 512], "bot_pct_lim": [0.0, 0.05]}),
          ("600x800 -> 336x448", 600, 800, {"H": 600, "W": 800, "final_dim": [336, 448], "bot_pct_lim": [0.0, 0.05]}),
          ("1080x1920 -> 288x512", 1080, 1920, {"H": 1080, "W": 1920, "final_dim": [288, 512], "bot_pct_lim": [0.0, 0.05]}))
N_IMG = 20


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()


def needed_source_bytes(plan):
    """uint8 bytes of the source pixels the crop window reads: the union of its row windows x the union of its column windows."""
    from heal_b200.data_utils.camera_input import axis_table
    l, t, r, b = plan.crop
    newW, newH = plan.resize_dims
    span = []
    for in_size, out_size, first, n in ((plan.H0, newH, t, b - t), (plan.W0, newW, l, r - l)):
        tab = axis_table(in_size, out_size, first, n)
        used = np.zeros(in_size, dtype=bool)
        for s, c in tab[:, :2]:
            used[s:s + c] = True
        span.append(int(used.sum()))
    return span[0] * span[1] * 3


def time_launches(fn, iters):
    for _ in range(3):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def kernel_times(iters, out):
    from heal_b200 import ops
    from heal_b200.data_utils.camera_input import inference_plan
    rows = []
    for name, H0, W0, conf in SHAPES:
        plan = inference_plan(conf, H0, W0)
        frames = torch.randint(0, 256, (N_IMG, H0, W0, 3), dtype=torch.uint8, device="cuda")
        fH, fW = plan.final_dim
        src = N_IMG * needed_source_bytes(plan)
        for layout, wbytes in (("nchw", N_IMG * 3 * fH * fW * 4), ("s2d", N_IMG * 4 * fH * fW * 4)):
            ms = time_launches(lambda: ops.camera_input(frames, plan, layout), iters)
            nbytes = src + wbytes
            rows.append({"shape": name, "layout": layout, "n_img": N_IMG, "us": ms * 1e3, "bytes": nbytes,
                         "GB_per_s": nbytes / (ms * 1e-3) / 1e9, "share_of_3.35TB/s": nbytes / (ms * 1e-3) / 3.35e12})
            print(f"heal_camera_input {name} {layout:4s} x{N_IMG}: {ms * 1e3:8.1f} us/launch, {nbytes / 1e6:7.2f} MB "
                  f"(read {src / 1e6:.2f}, write {wbytes / 1e6:.2f}) -> {nbytes / (ms * 1e-3) / 1e9:7.1f} GB/s")
    out["kernel"] = rows


def encoder_ab(reps, iters, out):
    from heal_b200 import engine
    from heal_b200.graph import GraphedCall
    from heal_b200.models.heter_encoders import LiftSplatShoot
    from oracle import procedural
    from workloads import configs as wcfg, synth
    engine.set_precision("bf16")
    cfg = wcfg.lss_encoder_args((256, 704))
    cfg["data_aug_conf"].update({"H": 600, "W": 800, "bot_pct_lim": [0.0, 0.05]})
    m = LiftSplatShoot(copy.deepcopy(cfg)).eval()
    m.load_state_dict(procedural.make_state_dict(procedural.shapes_of(m)), strict=True)
    m = m.cuda()
    plan = m.camera_plan(600, 800)
    rots, trans, intr, _, _ = [torch.from_numpy(a) for a in synth.camera_rig(2, 4, 256, 704)]
    geo = {"rots": rots, "trans": trans, "intrins": intr, "post_rots": plan.post_rot3().expand(2, 4, 3, 3).contiguous(),
           "post_trans": plan.post_tran3().expand(2, 4, 3).contiguous()}
    g = torch.Generator().manual_seed(5)
    host = {"raw": dict(geo, imgs=torch.randint(0, 256, (2, 4, 600, 800, 3), dtype=torch.uint8, generator=g)),
            "fp32": dict(geo, imgs=torch.randn(2, 4, 3, 256, 704, generator=g))}
    host = {k: {n: t.pin_memory() for n, t in v.items()} for k, v in host.items()}
    graphs = {}
    for arm, h in host.items():
        spec = {n: (tuple(t.shape), t.dtype) for n, t in h.items()}
        graphs[arm] = GraphedCall(lambda d: m(d, "m2"), spec, lambda bufs: {"inputs_m2": bufs}, torch.device("cuda"), init=h)
    res = {arm: [] for arm in graphs}
    h2d = {arm: sum(t.numel() * t.element_size() for t in h.values()) for arm, h in host.items()}
    for r in range(reps):
        for arm in ("raw", "fp32"):
            gc = graphs[arm]

            def frame():
                gc.load(**host[arm])
                gc.replay()
            res[arm].append(time_launches(frame, iters))
    for arm in ("raw", "fp32"):
        print(f"C4 camera encoder ({arm:4s} inputs, graph): one frame {np.median(res[arm]):.3f} ms "
              f"(rounds {', '.join(f'{v:.3f}' for v in res[arm])}), H2D {h2d[arm] / 1e6:.2f} MB, "
              f"{graphs[arm].kernels_per_replay} kernels")
    out["encoder"] = {arm: {"ms_rounds": res[arm], "h2d_bytes": h2d[arm], "kernels": graphs[arm].kernels_per_replay}
                      for arm in res}


def host_pil(out):
    try:
        from PIL import Image
        import torchvision
    except ImportError:
        print("host PIL resize + crop + normalize: not measured (Pillow or torchvision missing)")
        return
    torch.set_num_threads(1)
    norm = torchvision.transforms.Compose((torchvision.transforms.ToTensor(),
                                           torchvision.transforms.Normalize(mean=[0.485, 0.456, 0.406], std=[0.229, 0.224, 0.225])))
    res = {}
    for name, H0, W0, conf in SHAPES:
        from heal_b200.data_utils.camera_input import inference_plan
        plan = inference_plan(conf, H0, W0)
        img = Image.fromarray(np.random.default_rng(0).integers(0, 256, (H0, W0, 3), dtype=np.uint8))
        norm(img.resize(plan.resize_dims).crop(plan.crop))
        t0 = time.perf_counter()
        n = 20
        for _ in range(n):
            norm(img.resize(plan.resize_dims).crop(plan.crop))
        res[name] = (time.perf_counter() - t0) / n * 1e3
        print(f"host PIL resize + crop + normalize_img, {name}: {res[name]:.2f} ms per camera frame (1 CPU thread)")
    out["host_ms_per_frame"] = res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import __graft_entry__
    __graft_entry__.build()
    out = {"card": card()}
    print(f"card: {out['card']}")
    kernel_times(max(a.iters, 50), out)
    encoder_ab(a.reps, a.iters, out)
    host_pil(out)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "camera_input_experiment.json"), "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
