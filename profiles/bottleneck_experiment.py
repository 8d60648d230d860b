"""ResNeXt bottleneck (1x1 expand -> grouped 3x3 -> 1x1 reduce + residual) of PyramidFusion at frame size: each of the
three `ops.conv2d_tc` launches of one bottleneck and the fused kernel for its level (`ops.bottleneck_tc`, expand to reduce,
at level 0; `ops.gconv_reduce_tc`, grouped to reduce, at levels 1 and 2), timed alternately with CUDA events.  Prints us,
algorithmic bytes and GB/s per launch, shape and activation format, the card's name and power limit, and (unless
--no-bench) the conv families of one `bench.py` run; --out DIR keeps the per-launch records in
DIR/bottleneck_experiment.json and that run's full result line in DIR/bench_line.json."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# (name, planes, N, H, W): levels 0, 1 and 2 of the C2 frame (5 agents)
SHAPES = [("l0_64_128_64", 64, 5, 256, 256), ("l1_128_256_128", 128, 5, 128, 128), ("l2_256_512_256", 256, 5, 64, 64)]


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip()
    except Exception as e:                      # the numbers below still stand; say what could not be read
        return f"unknown ({e!r})"


def make_block(planes, seed):
    from heal_b200.models.sub_modules.resblock import Bottleneck
    torch.manual_seed(seed)
    # PyramidFusion's shape (Bottleneck.expansion = 1 there): width = 2 * planes, out = planes
    blk = Bottleneck.__new__(Bottleneck)
    torch.nn.Module.__init__(blk)
    width = 2 * planes
    blk.conv1 = torch.nn.Conv2d(planes, width, 1, bias=False)
    blk.bn1 = torch.nn.BatchNorm2d(width)
    blk.conv2 = torch.nn.Conv2d(width, width, 3, padding=1, groups=32, bias=False)
    blk.bn2 = torch.nn.BatchNorm2d(width)
    blk.conv3 = torch.nn.Conv2d(width, planes, 1, bias=False)
    blk.bn3 = torch.nn.BatchNorm2d(planes)
    blk.downsample, blk.stride = None, 1
    for bn in (blk.bn1, blk.bn2, blk.bn3):
        bn.running_mean.uniform_(-0.2, 0.2)
        bn.running_var.uniform_(0.5, 1.5)
        bn.weight.data.uniform_(0.5, 1.5)
        bn.bias.data.uniform_(-0.2, 0.2)
    return blk.eval().cuda()


def time_us(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters * 1e3


def run_shapes(iters, reps, records):
    from heal_b200 import engine, ops
    total = {}
    for fmt in ("split", "bf16"):
        for name, planes, N, H, W in SHAPES:
            lvl0 = planes == 64
            fused3 = hasattr(ops, "bottleneck_tc") and lvl0                  # expand + grouped + reduce: level 0
            fused2 = hasattr(ops, "gconv_reduce_tc") and not lvl0            # grouped + reduce: levels 1 and 2
            blk = make_block(planes, 0)
            pcs = [engine.packed(c, b, True, kind="tc2") for c, b in ((blk.conv1, blk.bn1), (blk.conv2, blk.bn2), (blk.conv3, blk.bn3))]
            x = ops.convert(ops.to_act(torch.randn(N, planes, H, W, device="cuda")), fmt)
            width = 2 * planes
            mid = ops.act_empty(N, H, W, width, fmt, "cuda")
            g = ops.act_empty(N, H, W, width, fmt, "cuda")
            y3 = ops.act_empty(N, H, W, planes, fmt, "cuda")
            y1 = ops.act_empty(N, H, W, planes, fmt, "cuda")
            fns = {"expand": lambda: ops.conv2d_tc(x, pcs[0], out=mid),
                   "grouped": lambda: ops.conv2d_tc(mid, pcs[1], out=g),
                   "reduce": lambda: ops.conv2d_tc(g, pcs[2], residual=x, out=y3)}
            if fused3:
                fns["fused"] = lambda: ops.bottleneck_tc(x, *pcs, out=y1)
            if fused2:
                fns["fused"] = lambda: ops.gconv_reduce_tc(mid, pcs[1], pcs[2], x, out=y1)

            epb = 4 if fmt == "split" else 2
            wb = [(pc.w_diag if pc.w_diag is not None else pc.w).numel() * 2 for pc in pcs]
            px = N * H * W
            nbytes = {"expand": px * epb * (planes + width) + wb[0],                    # x, mid
                      "grouped": px * epb * (width + width) + wb[1],                    # mid, g
                      "reduce": px * epb * (width + planes + planes) + wb[2]}          # g, residual, y
            nbytes["fused"] = (px * epb * 2 * planes + sum(wb) if fused3 else
                               px * epb * (width + planes + planes) + wb[1] + wb[2])   # mid, residual, y
            for _ in range(3):
                for f in fns.values():
                    f()
            torch.cuda.synchronize()
            ts = {k: [] for k in fns}
            for _ in range(reps):                          # alternate the launches so they see the same clocks
                for k, f in fns.items():
                    ts[k].append(time_us(f, iters))
            med = {k: sorted(v)[len(v) // 2] for k, v in ts.items()}
            rec = {"fmt": fmt, "shape": name, "N": N, "H": H, "W": W}
            parts = []
            for k in fns:
                gbs = nbytes[k] / med[k] / 1e3
                rec[k] = {"us": round(med[k], 2), "MB": round(nbytes[k] / 1e6, 2), "GB_s": round(gbs, 1),
                          "share_of_3.35TB_s": round(gbs / 3350, 3)}
                parts.append(f"{k} {med[k]:7.1f} us {nbytes[k] / 1e6:6.1f} MB {gbs:6.0f} GB/s")
            if "fused" in fns:
                fns["expand"](); fns["grouped"](); fns["reduce"](); fns["fused"]()
                torch.cuda.synchronize()
                rec["equal"] = bool(torch.equal(y1.t, y3.t))
                parts.append(f"equal={rec['equal']}")
            records.append(rec)
            print(f"{fmt:5s} {name:16s} N={N} {H}x{W} | " + " | ".join(parts), flush=True)
            nblk = {"l0": 3, "l1": 4, "l2": 7}[name[:2]]
            three = med["expand"] + med["grouped"] + med["reduce"]
            best = med["fused"] if fused3 else (med["expand"] + med["fused"] if fused2 else three)
            t = total.setdefault(fmt, [0.0, 0.0, 0.0])
            t[0] += nblk * three
            t[1] += nblk * best
            if not lvl0:
                t[2] += nblk * (med["grouped"] + med["reduce"])
    for fmt, (a, b, gr) in total.items():
        print(f"{fmt}: the 14 stride-1 bottlenecks of a frame (3 at level 0, 4 at level 1, 7 at level 2): three launches "
              f"{a / 1e3:.3f} ms, with the fused kernels where they apply {b / 1e3:.3f} ms; grouped + reduce of levels 1-2 "
              f"{gr / 1e3:.3f} ms", flush=True)


def run_bench(out_dir):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--no-cpu-baseline", "--no-eager-ref",
                        "--no-secondary"],
                       capture_output=True, text=True, cwd=ROOT)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    if not lines:
        print("bench.py printed no result line; exit", r.returncode, r.stderr[-2000:])
        return
    rec = json.loads(lines[-1])
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "bench_line.json"), "w") as fh:
            fh.write(lines[-1] + "\n")
    print("bench value", rec.get("value"), "latency", json.dumps(rec.get("latency"))[:300])
    for k in (rec.get("roofline") or {}).get("kernels", []):
        if k["name"].startswith("conv"):
            print(f"  {k['name']:28s} {k['ms_per_frame']:7.3f} ms/frame  {k['launches_per_frame']:4.0f} launches")
    roof = rec.get("roofline") or {}
    print("conv families:", roof.get("ms_per_frame"), "ms/frame, share_of_step", roof.get("share_of_step"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--no-bench", action="store_true")
    ap.add_argument("--out", default=None)
    opt = ap.parse_args()
    dev = card()
    print("card:", dev, flush=True)
    records = []
    run_shapes(opt.iters, opt.reps, records)
    if opt.out:
        os.makedirs(opt.out, exist_ok=True)
        with open(os.path.join(opt.out, "bottleneck_experiment.json"), "w") as fh:
            json.dump({"card": dev, "iters": opt.iters, "reps": opt.reps, "shapes": records}, fh, indent=1)
    if not opt.no_bench:
        run_bench(opt.out)


if __name__ == "__main__":
    main()
