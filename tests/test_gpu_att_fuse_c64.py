"""heal_att_fuse at C = 64 (the first fusion level of HeterModelBaselineMs): the k_att_fuse_g8<NA, FMT> instantiations against the
float64 reference of tests/test_gpu_fuse_kernels.py.

One case per (input format, register-file size): split-bf16, bf16 and fp32 input, NA = 5 (n <= 5) and NA = 8, plus n = 1, an
agent warped entirely out of view, exact-edge poses (whole-pixel shifts and quarter / half turns) and input / output slices of
wider buffers with sentinels around them.  Every case runs the kernel twice, with fp32 output (run A) and with the input's
format (run B), and checks, exactly as test_gpu_fuse_kernels.py does:
  - A is within the first-order bound of the float64 reference (fp32 taps from F.affine_grid on the fp64 theta, bilinear zeros
    padding and the softmax attention in float64) on the exact input the kernel read;
  - B is bit for bit the rounding of A (bf16(A); split: hi = bf16(A), lo = bf16(A - hi));
  - the channels around an input or output slice keep their sentinel.
torch.profiler shows that each case launches exactly its named instantiation and that together the cases launch all six.  Views
the 16-byte loads and stores cannot use (a bf16 / split view at channel 4, an fp32 view at channel 2) are refused with
HEAL_ERR_UNSUPPORTED and launch nothing."""
import json
import math
import os
import re
import subprocess
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_gpu_fuse_kernels as fk  # noqa: E402  (the float64 reference, inputs and buffers of the fuse.cu kernel tests)

Case = fk.Case
CASES = [
    Case("att64_split_n5", "att", "split", 5, 64, 33, 47, ("k_att_fuse_g8<5,2>",), out_of_view=(4,)),
    Case("att64_split_n8_out_slice", "att", "split", 8, 64, 15, 21, ("k_att_fuse_g8<8,2>",), out_slice=(128, 32)),
    Case("att64_split_n1", "att", "split", 1, 64, 9, 13, ("k_att_fuse_g8<5,2>",)),
    Case("att64_split_edges", "att", "split", 4, 64, 16, 32, ("k_att_fuse_g8<5,2>",), edges=True),
    Case("att64_split_slice8", "att", "split", 3, 64, 13, 19, ("k_att_fuse_g8<5,2>",), in_slice=(80, 8), out_slice=(72, 8)),
    Case("att64_bf16_n4_slice8", "att", "bf16", 4, 64, 21, 27, ("k_att_fuse_g8<5,1>",), in_slice=(80, 8)),
    Case("att64_bf16_n7", "att", "bf16", 7, 64, 13, 17, ("k_att_fuse_g8<8,1>",), out_of_view=(6,)),
    Case("att64_bf16_edges", "att", "bf16", 3, 64, 16, 16, ("k_att_fuse_g8<5,1>",), edges=True, out_slice=(80, 16)),
    Case("att64_f32_n3_slice4", "att", "f32", 3, 64, 19, 23, ("k_att_fuse_g8<5,0>",), in_slice=(72, 4)),
    Case("att64_f32_n6_out_slice", "att", "f32", 6, 64, 11, 13, ("k_att_fuse_g8<8,0>",), out_slice=(96, 12), out_of_view=(2,)),
    Case("att64_f32_n1", "att", "f32", 1, 64, 7, 9, ("k_att_fuse_g8<5,0>",)),
    Case("att64_f32_edges", "att", "f32", 4, 64, 8, 16, ("k_att_fuse_g8<5,0>",), edges=True),
]
CASE = {c.name: c for c in CASES}
REACHABLE = {f"k_att_fuse_g8<{na},{fmt}>" for na in (5, 8) for fmt in (0, 1, 2)}


@pytest.mark.parametrize("name", list(CASE))
def test_bound_rejects_plausible_kernel_bugs(name):
    """CPU: on a shrunken case the bound rejects a dropped lo plane, swapped nw / ne taps and a 1/C attention scale, and the
    tap-geometry rule holds."""
    case = CASE[name]
    H, W = fk._shrunk(case)
    inp = fk._inputs(case, H, W)
    st = {"feat": fk._store(inp["feat"], case.fmt)}
    vals = {"feat": fk._value(st["feat"], case.fmt)}
    y, bound, _ = fk._reference(case, inp, vals, H, W)
    assert bool(torch.isfinite(y).all())
    for fault in fk._faults(case):
        v = {"feat": fk._value(st["feat"], case.fmt, drop_lo=True)} if fault == "lo" else vals
        d = (fk._reference(case, inp, v, H, W, fault)[0] - y).abs()
        ratio = torch.where(d == 0, 0.0, d / bound).max().item()
        assert ratio > 1, f"{name}: the bound does not reject '{fault}' (max err / bound {ratio:.3f})"


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASE))
def test_att_fuse_c64(name):
    case = CASE[name]
    r = fk._launch(case)
    torch.cuda.synchronize()
    H, W, oco, cout = case.H, case.W, r["oco"], r["cout"]
    # the input as the kernel read it, and the sentinels around an input slice
    b = r["bufs"]["feat"].cpu()
    width, coff = case.in_slice or (b.shape[-1], 0)
    vals = {"feat": fk._value(b[..., coff:coff + case.C], case.fmt)}
    if width != case.C:
        whole = fk._value(b, case.fmt)
        around = torch.cat([whole[..., :coff].flatten(), whole[..., coff + case.C:].flatten()])
        assert bool((around == fk.SENTINEL).all()), f"{name}: the input buffer around the slice changed"
    # run A against float64
    y, bound, _ = fk._reference(case, r["inp"], vals, H, W)
    y, bound = y.reshape(1, H, W, cout), bound.reshape(1, H, W, cout)
    a_full = r["outs"]["A"].cpu()
    a = a_full[..., oco:oco + cout]
    err = (a.double() - y).abs()
    ok = err <= bound
    ratio = torch.where(err == 0, 0.0, err / bound).max().item()
    print(f"{name}: max err / bound {ratio:.4f}  (max err {err.max().item():.3e}, max|y| {y.abs().max().item():.3f}, "
          f"ALPHA 2^{math.log2(fk.ALPHA):.0f})")
    assert bool(ok.all()), f"{name}: {int((~ok).sum())} elements outside the bound, max err / bound {ratio:.3f}"
    # run B is the rounding of run A
    b_full = r["outs"]["B"].cpu()
    bo = b_full[..., oco:oco + cout]
    if case.fmt == "f32":
        assert torch.equal(fk._bits(bo), fk._bits(a)), f"{name}: the two fp32 runs differ"
    else:
        hi = a.to(torch.bfloat16)
        assert torch.equal(fk._bits(bo[0]), fk._bits(hi)), f"{name}: hi plane != bf16(fp32 output)"
        if case.fmt == "split":
            assert torch.equal(fk._bits(bo[1]), fk._bits((a - hi.float()).to(torch.bfloat16))), f"{name}: lo plane != bf16(fp32 - hi)"
    # the channels around an output slice keep their sentinel
    if case.out_slice:
        for run, t in (("A", a_full), ("B", b_full)):
            v = t.double() if t.dtype == torch.float32 else t[0].double()
            around = torch.cat([v[..., :oco].flatten(), v[..., oco + cout:].flatten()])
            assert bool((around == fk.SENTINEL).all()), f"{name} run {run}: a write spilled out of channels [{oco}, {oco + cout})"
            if case.fmt == "split" and run == "B":
                lo = torch.cat([t[1][..., :oco].flatten(), t[1][..., oco + cout:].flatten()])
                assert bool((lo == 0).all()), f"{name}: a lo-plane write spilled out of the slice"


_KERNEL = re.compile(r"\b(k_[a-z0-9_]+)\b(?:<\s*(?:\(int\))?\s*(\d+)\s*(?:,\s*(?:\(int\))?\s*(\d+)\s*)?>)?")


def _kernel_name(key):
    """`k_name<a,b>` for a heal_b200 kernel's profiler name, None for any other kernel (torch's fills and copies)."""
    m = _KERNEL.search(key)
    if not m:
        return None
    return m.group(1) + (f"<{m.group(2)}" + (f",{m.group(3)}" if m.group(3) else "") + ">" if m.group(2) else "")


def _profiled_kernels():
    """Runs every case under one torch.profiler session and returns the heal_b200 kernels it recorded, in launch order (each case
    is two library launches, runs A and B, so the list holds the cases' pairs in case order).  A session that recorded none of
    the launches the library counted is repeated once (a wrong kernel never is)."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    from heal_b200._lib import lib
    for _ in range(2):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for case in CASES:
                before = lib.heal_launch_count()
                fk._launch(case)
                torch.cuda.synchronize()
                assert lib.heal_launch_count() - before == 2, f"{case.name}: runs A and B are one launch each"
        ours = sorted((e.time_range.start, _kernel_name(e.name)) for e in prof.events()
                      if e.device_type == DeviceType.CUDA and _kernel_name(e.name))
        if ours:
            break
    return [n for _, n in ours]


@pytest.mark.gpu
def test_cases_reach_every_instantiation():
    """Each case runs the instantiation its row names (kernel names from torch.profiler), and together the cases run all six.

    The profiler session runs in a child process.  torch.profiler's CUDA records travel through activity buffers that live for
    the whole process, so sessions in one process are not independent: a session opened here, before the test files that
    follow it have run, moves where in their sessions a buffer changes hands, and a session in which that happens can come back
    without any kernel record.  In its own process this session leaves the rest of the suite's profiler state as it was."""
    tests_dir = os.path.dirname(os.path.abspath(__file__))
    code = ("import json, sys; sys.path[:0] = [%r, %r]; import test_gpu_att_fuse_c64 as t; "
            "print('KERNELS ' + json.dumps(t._profiled_kernels()))" % (tests_dir, os.path.dirname(tests_dir)))
    r = subprocess.run([sys.executable, "-s", "-c", code], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stdout[-4000:]
    names = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("KERNELS ")][-1][len("KERNELS "):])
    assert len(names) == 2 * len(CASES), f"the session recorded {len(names)} heal_b200 kernels for {2 * len(CASES)} launches"
    for i, case in enumerate(CASES):
        assert set(names[2 * i:2 * i + 2]) == set(case.reaches), \
            f"{case.name}: ran {names[2 * i:2 * i + 2]}, expected {sorted(case.reaches)}"
    assert set(names) == REACHABLE


@pytest.mark.gpu
@pytest.mark.parametrize("fmt,coff", [("f32", 2), ("bf16", 4), ("split", 4)])
@pytest.mark.parametrize("where", ["in", "out"])
def test_misaligned_view_is_refused(fmt, coff, where):
    """A view at channel `coff` of a wider buffer: 8-byte aligned in bf16 / split (enough for 4-channel loads, not for 16-byte
    ones) and 8-byte aligned in fp32.  Refused with HEAL_ERR_UNSUPPORTED -> RuntimeError; nothing is launched (the library's
    launch counter does not move)."""
    from heal_b200 import ops
    from heal_b200._lib import lib
    H, W, C, n = 5, 7, 64, 3
    th = fk._thetas(CASE["att64_split_n5"], H, W, n).cuda()

    def act(N, bad):
        t = torch.zeros((N, H, W, C + 8)) if fmt == "f32" else \
            torch.zeros((2 if fmt == "split" else 1, N, H, W, C + 8), dtype=torch.bfloat16)
        t = t.cuda()
        return ops.Act(t[..., coff:coff + C] if bad else t[..., :C], fmt)

    feat, out = act(n, where == "in"), act(1, where == "out")
    torch.cuda.synchronize()
    before = lib.heal_launch_count()
    with pytest.raises(RuntimeError, match="HEAL_ERR_UNSUPPORTED"):
        ops.att_fuse(feat, th, out=out)
    torch.cuda.synchronize()
    assert lib.heal_launch_count() == before


@pytest.mark.gpu
def test_more_than_eight_agents_is_refused():
    from heal_b200 import ops
    x = ops.act_empty(9, 4, 4, 64, "split", "cuda")
    th = torch.eye(2, 3, dtype=torch.float64).expand(9, 2, 3).contiguous().cuda()
    with pytest.raises(RuntimeError, match="HEAL_ERR_UNSUPPORTED"):
        ops.att_fuse(x, th)
