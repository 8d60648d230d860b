"""The C = 64 attention-fusion kernel (k_att_fuse_g8<NA, FMT>) compiles for sm_90a with a 0-byte stack frame and no register
spills in every instantiation: it keeps NA agents' warped 8-channel slices in registers, and a spill would be a silent loss no
numerical test sees.  Compiles fuse.cu with the library's own nvcc flags; needs no GPU."""
import os
import re
import shutil
import subprocess
import tempfile

import pytest

from heal_b200 import build as hb

# (agents the register file is sized for, input format: 0 f32, 1 bf16, 2 split-bf16)
INSTANTIATIONS = [(na, fmt) for na in (5, 8) for fmt in (0, 1, 2)]


def test_att_fuse_c64_kernels_compile_without_spills():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not (os.path.exists(nvcc) or shutil.which(nvcc)):
        pytest.skip("nvcc not available")
    with tempfile.TemporaryDirectory() as tmp:
        cmd = [nvcc] + hb.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(hb.CSRC, "fuse.cu"), "-o", os.path.join(tmp, "k.o")]
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    current, reports = None, {}
    for line in r.stdout.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            current = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        k = re.search(r"k_att_fuse_g8ILi(\d+)ELi(\d+)E", current or "")
        if m and k:
            reports[(int(k.group(1)), int(k.group(2)))] = m.groups()
    assert sorted(reports) == sorted(INSTANTIATIONS), f"ptxas reported {sorted(reports)}:\n{r.stdout}"
    assert all(g == ("0", "0", "0") for g in reports.values()), reports
