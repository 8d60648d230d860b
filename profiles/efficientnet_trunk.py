"""Times the EfficientNet camera encoder (`CamEncode.heads_nhwc`: csrc/mbconv.cu trunk, `Up` stages on the conv engine, fused heads)
at the camera shapes the yamls use, against the same module's torch / cuDNN path (`heads`) on the same device, and breaks the time
down per kernel.  Needs a GPU; prints the card and its power limit, which belong beside every number taken from the output.

    python profiles/efficientnet_trunk.py [--iters 200] [--out DIR]

Per shape it prints
  * heads_nhwc and eager `heads` time per call (CUDA events around blocks of calls, the two alternating, after warm-up);
  * per kernel family (the ops wrappers' names): calls, time from CUDA events around each call in a separate instrumented pass
    (eager launches, so launch gaps are inside), algorithmic FLOPs and HBM bytes computed from the shapes by the wrappers
    (heal_b200/ops.py), the lower bound max(FLOPs / peak, bytes / 3.35 TB/s) with the bound that applies, and time / bound.
    Peaks are the H100 SXM data-sheet figures: 67 TFLOP/s fp32 for the CUDA-core kernels; 989 / 3 TFLOP/s for the wgmma
    convolutions in the default precision mode (three bf16 MMAs per fp32-equivalent product);
  * per CUDA kernel name, from a torch.profiler pass of its own: calls and mean device time.
"""
import argparse
import collections
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

SHAPES = {"BASELINE camera 4x3x256x704": (4, 3, 256, 704), "HEAL m2 final_dim 4x3x384x512": (4, 3, 384, 512)}
HBM, FP32, TC32 = 3.35e12, 67e12, 989e12 / 3


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()


def timed(fn, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--out", default=None, help="directory for the torch.profiler table (default: print only)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("profiles/efficientnet_trunk.py measures on a GPU; none found")
    import __graft_entry__
    __graft_entry__.build()
    from heal_b200 import engine, ops
    from heal_b200.models.heter_encoders import CamEncode
    from workloads import procedural
    print(f"card: {card()}   precision mode: {engine.PRECISION}   iterations: {args.iters}")
    m = CamEncode(48, 128, 8, [2, 50, 48], "LID", False, False).eval()
    m.load_state_dict(procedural.make_state_dict(procedural.shapes_of(m)), strict=True)
    m = m.cuda()
    for name, shape in SHAPES.items():
        x = torch.randn(*shape, generator=torch.Generator().manual_seed(3)).cuda()
        with torch.no_grad():
            for _ in range(10):
                y = m.heads_nhwc(x)
                dl, ft = m.heads(x)
            torch.cuda.synchronize()
            ref = torch.cat([dl, ft], 1).permute(0, 2, 3, 1)
            err = (y.t - ref).abs().max().item() / max(ref.abs().max().item(), 1.0)
            ours, eager, block = [], [], 20
            for _ in range(max(args.iters // block, 1)):
                ours.append(timed(lambda: m.heads_nhwc(x), block))
                eager.append(timed(lambda: m.heads(x), block))
            print(f"\n== {name}: heads_nhwc {sum(ours) / len(ours):.3f} ms/call (blocks min {min(ours):.3f} max {max(ours):.3f}) | "
                  f"eager torch heads {sum(eager) / len(eager):.3f} ms/call (min {min(eager):.3f} max {max(eager):.3f}) | "
                  f"max|diff| / max|ref| = {err:.2e}")
            ops.PROFILE = []
            m.heads_nhwc(x)
            torch.cuda.synchronize()
            rows = collections.OrderedDict()
            for fam, work, a, b, nbytes, launches in ops.PROFILE:
                r = rows.setdefault(fam, [0, 0.0, 0.0, 0.0])
                r[0] += 1; r[1] += a.elapsed_time(b); r[2] += float(work); r[3] += float(nbytes)
            ops.PROFILE = None
            print(f"{'kernel family':<22}{'calls':>6}{'ms':>9}{'GFLOP':>9}{'MB':>9}{'bound us':>10}  bound   time/bound")
            total = 0.0
            for fam, (calls, ms, fl, by) in rows.items():
                peak = TC32 if fam.startswith("conv_tc") else FP32
                tf, tb = fl / peak, by / HBM
                lo = max(tf, tb)
                total += ms
                print(f"{fam:<22}{calls:>6}{ms:>9.3f}{fl / 1e9:>9.2f}{by / 1e6:>9.1f}{lo * 1e6:>10.1f}  {'FLOPs' if tf > tb else 'HBM':<7}"
                      f"{ms * 1e-3 / lo if lo else float('nan'):>8.1f}x")
            print(f"{'sum of per-call events':<22}{'':>6}{total:>9.3f}")
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA, torch.profiler.ProfilerActivity.CPU]) as prof:
                for _ in range(5):
                    m.heads_nhwc(x)
                torch.cuda.synchronize()
            ks = [(e.key, e.count // 5, e.device_time_total / 5) for e in prof.key_averages() if e.device_time_total > 0 and e.device_type == torch.autograd.DeviceType.CUDA]
            ks.sort(key=lambda r: -r[2])
            lines = [f"{k[:90]:<92}{c:>5}{t:>10.1f}" for k, c, t in ks]
            print(f"{'CUDA kernel (torch.profiler, per call of heads_nhwc)':<92}{'n':>5}{'us':>10}")
            print("\n".join(lines))
            print(f"{'device time, all kernels':<92}{'':>5}{sum(t for _, _, t in ks):>10.1f}")
            if args.out:
                os.makedirs(args.out, exist_ok=True)
                with open(os.path.join(args.out, f"efficientnet_trunk_{shape[2]}x{shape[3]}.txt"), "w") as fh:
                    fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
