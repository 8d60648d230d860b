"""The EfficientNet trunk kernels (csrc/mbconv.cu) compile for sm_90a without register spills or local memory: the pointwise GEMM
keeps a 4 x 4 accumulator tile per thread, and a spill would be a silent loss no numerical test sees.  Compiles with the library's
own nvcc flags; needs no GPU."""
import os
import re
import shutil
import subprocess
import tempfile

import pytest

from heal_b200 import build as hb

KERNELS = ("k_stem_conv_swish", "k_dwconv_bn_swish", "k_dwconv_sum_finish", "k_se_gate", "k_pwconv", "k_upsample2x_concat")


def test_mbconv_kernels_compile_without_spills():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not (os.path.exists(nvcc) or shutil.which(nvcc)):
        pytest.skip("nvcc not available")
    with tempfile.TemporaryDirectory() as tmp:
        cmd = [nvcc] + hb.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(hb.CSRC, "mbconv.cu"), "-o", os.path.join(tmp, "k.o")]
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
            for k in KERNELS:
                if k in current:
                    reports[k] = m.groups()
    assert set(reports) == set(KERNELS), f"ptxas report lacks {set(KERNELS) - set(reports)}:\n{r.stdout}"
    assert all(g == ("0", "0", "0") for g in reports.values()), reports
