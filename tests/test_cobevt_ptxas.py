"""The CoBEVT kernels (k_swap_attention, k_mean_layernorm) compile for sm_90a without register spills: the attention kernel keeps
a 32-wide q row and output row per thread in registers, and a spill would be a silent loss no numerical test sees.  Compiles
with the library's own nvcc flags; needs no GPU."""
import os
import re
import shutil
import subprocess
import tempfile

import pytest

from heal_b200 import build as hb


@pytest.mark.parametrize("src,kernel", [("swap_attn.cu", "k_swap_attention"), ("convnext.cu", "k_mean_layernorm")])
def test_cobevt_kernels_compile_without_spills(src, kernel):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not (os.path.exists(nvcc) or shutil.which(nvcc)):
        pytest.skip("nvcc not available")
    with tempfile.TemporaryDirectory() as tmp:
        cmd = [nvcc] + hb.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(hb.CSRC, src), "-o", os.path.join(tmp, "k.o")]
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    current, reports = None, []
    for line in r.stdout.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            current = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and current and kernel in current:
            reports.append(m.groups())
    assert reports, f"no {kernel} entry in the ptxas report:\n{r.stdout}"
    assert all(g == ("0", "0", "0") for g in reports), reports
