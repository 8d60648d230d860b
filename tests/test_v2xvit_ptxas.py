"""The V2X-ViT kernels (v2xvit.cu) compile for sm_90a without register spills: every window-attention instantiation keeps its
q fragments, the output accumulator and a key chunk of scores in registers, and a spill would be a silent loss no numerical
test sees.  Compiles with the library's own nvcc flags; needs no GPU."""
import os
import re
import shutil
import subprocess
import tempfile

import pytest

from heal_b200 import build as hb

KERNELS = ["k_window_attention", "k_cav_attention", "k_split_pool", "k_split_gate", "k_split_combine", "k_sttf_resample"]


def test_v2xvit_kernels_compile_without_spills():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not (os.path.exists(nvcc) or shutil.which(nvcc)):
        pytest.skip("nvcc not available")
    with tempfile.TemporaryDirectory() as tmp:
        cmd = [nvcc] + hb.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(hb.CSRC, "v2xvit.cu"), "-o", os.path.join(tmp, "k.o")]
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    current, reports = None, {}
    for line in r.stdout.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            current = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and current:
            reports[current] = m.groups()
    for k in KERNELS:
        found = {name: g for name, g in reports.items() if k in name}
        assert found, f"no {k} entry in the ptxas report:\n{r.stdout}"
        assert all(g == ("0", "0", "0") for g in found.values()), found
    # 3 window sizes x 3 head widths x (bf16, split-bf16)
    assert len([n for n in reports if "k_window_attention" in n]) == 18
