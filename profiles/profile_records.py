"""The `ops.PROFILE` record sequence of eager frames, one JSON file per workload: (name, work, nbytes, launches) per C-ABI
record, callables evaluated.  Two builds that should launch the same work (a refactor of the host wrappers) write identical
files; `--compare A B` diffs two output directories.

    python profiles/profile_records.py --out DIR [--workloads c1 c2 c3 c4] [--frames 2]
    python profiles/profile_records.py --compare DIR_A DIR_B
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def records(workload, frames):
    import torch
    import bench
    from heal_b200 import ops
    wl = bench.GpuWorkload(workload, "bf16" if workload == "c4" else "tc32", torch.device("cuda", 0))
    with torch.no_grad():
        for i in range(2):
            wl.eager(i)
        torch.cuda.synchronize()
        ops.PROFILE = []
        for i in range(frames):
            wl.eager(i)
        torch.cuda.synchronize()
        recs, ops.PROFILE = ops.PROFILE, None
    ev = lambda v: float(v() if callable(v) else v)
    return [[name, ev(work), ev(nbytes), launches] for name, work, _, _, nbytes, launches in recs]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    ap.add_argument("--workloads", nargs="+", default=["c1", "c2", "c3", "c4"])
    ap.add_argument("--frames", type=int, default=2)
    ap.add_argument("--compare", nargs=2, metavar="DIR")
    opt = ap.parse_args()
    if opt.compare:
        a, b = opt.compare
        same = True
        for f in sorted(os.listdir(a)):
            ra, rb = json.load(open(os.path.join(a, f))), json.load(open(os.path.join(b, f)))
            diff = next((i for i, (x, y) in enumerate(zip(ra, rb)) if x != y), None if len(ra) == len(rb) else min(len(ra), len(rb)))
            ok = diff is None
            same &= ok
            print(f"{f}: {len(ra)} / {len(rb)} records, " + ("identical" if ok else f"first difference at {diff}"))
        sys.exit(0 if same else 1)
    os.makedirs(opt.out, exist_ok=True)
    for w in opt.workloads:
        recs = records(w, opt.frames)
        json.dump(recs, open(os.path.join(opt.out, f"{w}.json"), "w"))
        print(f"{w}: {len(recs)} records, {sum(r[3] for r in recs)} launches in {opt.frames} frames")


if __name__ == "__main__":
    main()
