"""Regenerate profiles/sass_counts_r2.txt: per-kernel counts of the SASS mnemonics that prove which hardware paths the in-tree
library uses (python profiles/sass_counts.py; needs cuobjdump, no GPU)."""
import collections
import os
import re
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "..", "heal_b200", "libheal_b200.so")
OPS = ["HGMMA", "UTMALDG", "UTMASTG", "LDGSTS", "HMMA"]


def main():
    sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    names = subprocess.run(["cu++filt"], input="\n".join(re.findall(r"Function : (\S+)", sass)), capture_output=True, text=True).stdout.split("\n")
    per, total, cur, i = collections.OrderedDict(), collections.Counter(), None, 0
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = names[i] if i < len(names) else m.group(1)
            i += 1
            per[cur] = collections.Counter()
            continue
        if cur is None:
            continue
        m = re.search(r"\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
        if m:
            op = m.group(1).split(".")[0]
            if op in OPS:
                per[cur][op] += 1
                total[op] += 1
    out = ["# SASS instruction counts of heal_b200/libheal_b200.so (cuobjdump -sass, sm_90a), kernels that use the tensor-core / TMA / async-copy paths",
           "# HGMMA = wgmma.mma_async, UTMALDG / UTMASTG = TMA tensor load / store, LDGSTS = cp.async, HMMA = mma.sync",
           "total: " + ", ".join(f"{k}={total[k]}" for k in sorted(OPS))]
    for name, c in per.items():
        if c:
            out.append(f"{name[:110]}: " + ", ".join(f"{k}={c[k]}" for k in OPS if c[k]))
    with open(os.path.join(HERE, "sass_counts_r2.txt"), "w") as fh:
        fh.write("\n".join(out) + "\n")
    print(out[2])


if __name__ == "__main__":
    main()
