"""The fused grouped 3x3 + reduce kernel (k_gconv_reduce_tc) compiles without a serialised wgmma chain (ptxas C7511) and
without register spills: it keeps the reduce accumulators live while the grouped conv runs, so either would be a silent loss
that no numerical test sees.  Compiles with the library's own nvcc flags; needs no GPU."""
import os
import re
import shutil
import subprocess
import tempfile

import pytest

from heal_b200 import build as hb


def test_gconv_reduce_kernel_compiles_without_wgmma_serialisation_or_spills():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not (os.path.exists(nvcc) or shutil.which(nvcc)):
        pytest.skip("nvcc not available")
    with tempfile.TemporaryDirectory() as tmp:
        cmd = [nvcc] + hb.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(hb.CSRC, "gconv_reduce_tc.cu"),
                                        "-o", os.path.join(tmp, "gconv_reduce_tc.o")]
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    log = r.stdout
    serialised = [l for l in log.splitlines() if re.search(r"C75(1[1-8]|20)", l)]
    assert not serialised, "\n".join(serialised)
    current, reports = None, []
    for line in log.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            current = m.group(1)
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and current and "k_gconv_reduce_tc" in current:
            reports.append((m.group(1), m.group(2)))
    assert reports, f"no k_gconv_reduce_tc entry in the ptxas report:\n{log}"
    assert all(s == "0" and l == "0" for s, l in reports), reports
