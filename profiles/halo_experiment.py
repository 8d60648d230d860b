"""Halo loads and the A-row ring on or off (HEAL_TC_HALO, read once per process): microseconds per launch of the level-2 grouped 3x3 conv of
PyramidFusion and of the two shrink-header 3x3 convs, in tc32 (split activations), one child process per setting, alternating.

    python profiles/halo_experiment.py [--rounds 3] [--iters 50]

Prints one line per (round, setting, shape) and a summary with the card name and its power limit."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

# name, N, Cin, Cout, H = W, groups, residual
SHAPES = [("l2_grouped_512_n5_64px", 5, 512, 512, 64, 32, False),
          ("shrink_384_256_n1_256px", 1, 384, 256, 256, 1, False),
          ("shrink_256_256_n1_256px", 1, 256, 256, 256, 1, False)]


def child(iters):
    from heal_b200 import ops
    torch.manual_seed(0)
    out = {}
    for name, N, cin, cout, hw, groups, res in SHAPES:
        conv = torch.nn.Conv2d(cin, cout, 3, padding=1, groups=groups, bias=False)
        pc = ops.pack_conv_tc(conv, torch.nn.BatchNorm2d(cout).eval(), True, planes=2).to("cuda")
        x = ops.convert(ops.to_act(torch.randn(N, cin, hw, hw, device="cuda")), "split")
        y = ops.act_empty(N, hw, hw, cout, "split", "cuda")
        r = ops.convert(ops.to_act(torch.randn(N, cout, hw, hw, device="cuda")), "split") if res else None
        for _ in range(5):
            ops.conv2d_tc(x, pc, out=y, residual=r)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            ops.conv2d_tc(x, pc, out=y, residual=r)
        b.record()
        torch.cuda.synchronize()
        out[name] = a.elapsed_time(b) / iters * 1e3
    print("RESULT " + json.dumps(out))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE,
                           stderr=subprocess.DEVNULL, text=True, timeout=60).stdout.strip().splitlines()
        return q[0] if q else torch.cuda.get_device_name(0)
    except (OSError, subprocess.TimeoutExpired):
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--child", action="store_true")
    opt = ap.parse_args()
    if opt.child:
        child(opt.iters)
        return
    runs = {"0": [], "1": []}
    for rnd in range(opt.rounds):
        for halo in ("0", "1"):
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "--iters", str(opt.iters)],
                               stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env={**os.environ, "HEAL_TC_HALO": halo})
            lines = [ln for ln in r.stdout.splitlines() if ln.startswith("RESULT ")]
            if r.returncode != 0 or not lines:
                sys.exit(f"HEAL_TC_HALO={halo} failed:\n{r.stdout[-4000:]}")
            res = json.loads(lines[-1][len("RESULT "):])
            runs[halo].append(res)
            for name, us in res.items():
                print(f"round {rnd} HEAL_TC_HALO={halo} {name}: {us:8.1f} us")
    print(f"card: {card()}")
    for name, *_ in SHAPES:
        old, new = [r[name] for r in runs["0"]], [r[name] for r in runs["1"]]
        print(f"{name}: halo off {min(old):7.1f}-{max(old):7.1f} us, on {min(new):7.1f}-{max(new):7.1f} us "
              f"({min(old) / min(new):.2f}x, best of {opt.rounds})")


if __name__ == "__main__":
    main()
