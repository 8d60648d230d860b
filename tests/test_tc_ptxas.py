"""The wgmma convolution kernels compile without serialised wgmma chains (ptxas C7511) and without register spills.

Both are silent performance losses that no numerical test sees: ptxas falls back to waiting for every wgmma before issuing the
next, or moves accumulator registers through local memory.  Compiles with the library's own nvcc flags; needs no GPU."""
import os
import re
import shutil
import subprocess
import tempfile

import pytest

from heal_b200 import build as hb

KERNELS = {"conv2d_tc.cu": "k_conv2d_tc", "conv3x3_ring.cu": "k_gconv3x3_ring"}


def _nvcc():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not (os.path.exists(nvcc) or shutil.which(nvcc)):
        pytest.skip("nvcc not available")
    return nvcc


def _ptxas_report(nvcc, src, out_dir):
    cmd = [nvcc] + hb.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(hb.CSRC, src), "-o", os.path.join(out_dir, src + ".o")]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    return r.stdout


@pytest.mark.parametrize("src", sorted(KERNELS))
def test_tc_kernels_compile_without_wgmma_serialisation_or_spills(src):
    nvcc = _nvcc()
    with tempfile.TemporaryDirectory() as tmp:
        log = _ptxas_report(nvcc, src, tmp)
    serialised = [l for l in log.splitlines() if "C7511" in l]
    assert not serialised, "\n".join(serialised)
    spills, current, seen = [], None, 0
    for line in log.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            current = m.group(1)
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and current and KERNELS[src] in current:
            seen += 1
            if m.group(1) != "0" or m.group(2) != "0":
                spills.append(f"{current}: {line.strip()}")
    assert seen > 0, f"no {KERNELS[src]} entry in the ptxas report:\n{log}"
    assert not spills, "\n".join(spills)
