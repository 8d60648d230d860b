"""ResNeXt bottleneck (1x1 expand -> grouped 3x3 -> 1x1 reduce + residual) of PyramidFusion at frame size: the three
`ops.conv2d_tc` launches of one bottleneck and, where the library has it, the fused `ops.bottleneck_tc`, timed alternately
with CUDA events.  Prints us, algorithmic bytes and GB/s per shape and activation format, the card's name and power limit,
and (unless --no-bench) the conv families of one `bench.py` run; --out DIR keeps that run's full result line in
DIR/bench_line.json."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# (name, planes, N, H, W): level 0 and level 1 of the C2 frame (5 agents)
SHAPES = [("l0_64_128_64", 64, 5, 256, 256), ("l1_128_256_128", 128, 5, 128, 128)]


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


def run_shapes(iters, reps):
    from heal_b200 import engine, ops
    total = {}
    for fmt in ("split", "bf16"):
        for name, planes, N, H, W in SHAPES:
            fused = hasattr(ops, "bottleneck_tc") and planes == 64     # the fused kernel covers level 0
            blk = make_block(planes, 0)
            pcs = [engine.packed(c, b, True, kind="tc2") for c, b in ((blk.conv1, blk.bn1), (blk.conv2, blk.bn2), (blk.conv3, blk.bn3))]
            x = ops.convert(ops.to_act(torch.randn(N, planes, H, W, device="cuda")), fmt)
            width = 2 * planes
            mid = ops.act_empty(N, H, W, width, fmt, "cuda")
            g = ops.act_empty(N, H, W, width, fmt, "cuda")
            y3 = ops.act_empty(N, H, W, planes, fmt, "cuda")
            y1 = ops.act_empty(N, H, W, planes, fmt, "cuda")

            def three():
                ops.conv2d_tc(x, pcs[0], out=mid)
                ops.conv2d_tc(mid, pcs[1], out=g)
                ops.conv2d_tc(g, pcs[2], residual=x, out=y3)

            def one():
                ops.bottleneck_tc(x, *pcs, out=y1)

            epb = 4 if fmt == "split" else 2
            wbytes = sum((pc.w_diag if pc.w_diag is not None else pc.w).numel() * 2 for pc in pcs)
            px = N * H * W
            b3 = px * epb * (planes + 2 * width + 2 * width + planes + planes) + wbytes   # x, mid w/r, g w/r, y, residual
            b1 = px * epb * (planes + planes) + wbytes
            for _ in range(3):
                three()
                if fused:
                    one()
            torch.cuda.synchronize()
            t3, t1 = [], []
            for _ in range(reps):
                t3.append(time_us(three, iters))
                if fused:
                    t1.append(time_us(one, iters))
            m3 = sorted(t3)[len(t3) // 2]
            line = f"{fmt:5s} {name:16s} N={N} {H}x{W}  three launches {m3:8.1f} us  {b3 / 1e6:7.1f} MB  {b3 / m3 / 1e3:7.1f} GB/s"
            total.setdefault(fmt, [0.0, 0.0])
            nblk = 3 if name.startswith("l0") else 4
            total[fmt][0] += nblk * m3
            m1 = sorted(t1)[len(t1) // 2] if fused else m3
            total[fmt][1] += nblk * m1
            if fused:
                same = torch.equal(y1.t, y3.t)
                line += f" | fused {m1:8.1f} us  {b1 / 1e6:7.1f} MB  {b1 / m1 / 1e3:7.1f} GB/s  x{m3 / m1:4.2f}  equal={same}"
            print(line, flush=True)
    for fmt, (a, b) in total.items():
        print(f"{fmt}: the 7 fusable bottlenecks of a frame (3 at level 0, 4 at level 1): three launches {a / 1e3:.3f} ms"
              + f", with the fused kernel where it applies {b / 1e3:.3f} ms", flush=True)


def run_bench(out_dir):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--no-cpu-baseline", "--no-eager-ref"],
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--no-bench", action="store_true")
    ap.add_argument("--out", default=None)
    opt = ap.parse_args()
    print("card:", card(), flush=True)
    run_shapes(opt.iters, opt.reps)
    if not opt.no_bench:
        run_bench(opt.out)


if __name__ == "__main__":
    main()
