"""heal_conv2d_tc's row-reuse loads for 3x3 stride-1 convs.  Halo loads on two-row tiles (maps 64 to 127 pixels wide): the
grouped 3x3 convs of PyramidFusion level 2 load one activation box of 2 rows x (TW + 2) pixels per kernel row instead of one box
per tap.  The A-row ring of the 128-wide dense convs (the shrink header, maps >= 128 wide): one input row of TW + 2 pixels per
(channel block, kernel row) serves the three kernel columns' k-blocks.

Each case runs the product call (split / bf16 output through the staging epilogue) and a call that also writes f32 (the
direct-store epilogue), in tc32 (split activations) and the 'bf16' mode, and checks:
  - the f32 output is within the float64 bound of tests/test_gpu_conv_epilogue.py, on the exact input the kernel read;
  - the split / bf16 output is exactly the rounding of the f32 output;
  - grouped cases: both outputs equal, bit for bit, those of the same calls with the halo loads switched off (HEAL_TC_HALO=0,
    read once per process, so that run is a child process): a grouped conv visits its taps in the same order either way.  The
    A-row ring sums K in another order (channel block, kernel row, kernel column), so those cases are held to the bound only.
The dense 64-wide case keeps its per-tap loads; it is here so that the two-row dispatch is covered on both sides."""
import os
import subprocess
import sys
import tempfile
import zlib

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_gpu_conv_epilogue as ep  # noqa: E402  (Stage, the nn modules, the float64 reference and its bound)

Stage = ep.Stage
MODES = ep.MODES

# name, (N, H, W), stage
CASES = [
    # PyramidFusion level 2: 5 agents at 64 x 64, 512 channels in 32 groups (16 per group), 1280 tiles
    ("l2_grouped", (5, 64, 64), Stage(512, 512, 3, groups=32)),
    # 8 channels per group; H and W not multiples of the 2 x 64 tile (a ragged tile column and a half-empty tile row)
    ("g32_cg8_ragged", (2, 37, 100), Stage(256, 256, 3, groups=32)),
    # a split / bf16 residual, TMA-loaded into the staging buffers
    ("g32_res", (1, 18, 64), Stage(128, 128, 3, groups=32, res="act")),
    # no ReLU, no BN
    ("g32_linear", (1, 10, 127), Stage(128, 128, 3, groups=32, bn=False, act=0)),
    # dense N = 64 on a 64-wide map: per-tap loads (a dense halo stage would leave room for two stages only)
    ("dense_n64_w64", (2, 24, 64), Stage(64, 64, 3)),
    # the shrink header's convs on fewer rows: A-row ring, two n-tiles per pixel tile
    ("shrink_384_256", (1, 12, 256), Stage(384, 256, 3)),
    ("shrink_256_256", (1, 12, 256), Stage(256, 256, 3)),
    # an f32 residual read by the staging epilogue
    ("shrink_256_256_res_f32", (1, 12, 256), Stage(256, 256, 3, res="f32")),
    # ragged: a 128-pixel tile and a 22-pixel one, an odd number of rows, 128 output channels
    ("ring_ragged", (2, 7, 150), Stage(256, 128, 3)),
]
CASE = {c[0]: c for c in CASES}


def _outputs(name, mode):
    """(input, residual, product output, f32 output, split / bf16 output of the f32 call) of one case, all on the CPU."""
    from heal_b200 import ops
    fmt, planes = MODES[mode]
    _, (N, H, W), st = CASE[name]
    gen = torch.Generator().manual_seed(zlib.crc32(f"halo/{name}".encode()))
    conv, bn = ep._modules(name, 0, st)
    pc = ops.pack_conv_tc(conv, bn, st.act, planes=2).to("cuda")
    x = ops.convert(ops.to_act(torch.randn(N, st.cin, H, W, generator=gen).cuda()), fmt)
    res = None
    if st.res:
        res = ops.to_act(torch.randn(N, st.cout, H, W, generator=gen).cuda())
        res = ops.convert(res, fmt) if st.res == "act" else res
    nan = float("nan")
    a = torch.full((planes, N, H, W, st.cout), nan, dtype=torch.bfloat16, device="cuda")
    ops.conv2d_tc(x, pc, residual=res, out=ops.Act(a, fmt))
    ob = torch.full_like(a, nan)
    of = torch.full((N, H, W, st.cout), nan, dtype=torch.float32, device="cuda")
    ops.conv2d_tc(x, pc, residual=res, out=ops.Act(ob, fmt), out_f32=ops.Act(of, "f32"), want_f32=True)
    torch.cuda.synchronize()
    return dict(x=x.t.cpu(), res=None if res is None else res.t.cpu(), a=a.cpu(), of=of.cpu(), ob=ob.cpu())


def _child_outputs(path):
    torch.save({(n, m): {k: v for k, v in _outputs(n, m).items() if k in ("a", "of", "ob")} for n in CASE for m in MODES}, path)


@pytest.fixture(scope="module")
def halo_off():
    """Every case's outputs with the halo loads switched off, computed in a child process."""
    tests_dir = os.path.dirname(os.path.abspath(__file__))
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "halo_off.pt")
        code = ("import sys; sys.path[:0] = [%r, %r]; import test_gpu_conv_halo as t; t._child_outputs(%r)"
                % (tests_dir, os.path.dirname(tests_dir), path))
        r = subprocess.run([sys.executable, "-s", "-c", code], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                           timeout=900, env={**os.environ, "HEAL_TC_HALO": "0"})
        assert r.returncode == 0, r.stdout[-4000:]
        return torch.load(path)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("name", list(CASE))
def test_conv_halo(name, mode, halo_off):
    planes = MODES[mode][1]
    _, _, st = CASE[name]
    tag = f"{name} [{mode}]"
    o = _outputs(name, mode)
    # 1. the grouped halo loads change no bit of either epilogue's output
    for k in (("a", "of", "ob") if st.groups > 1 else ()):
        assert torch.equal(ep._bits(o[k]), ep._bits(halo_off[(name, mode)][k])), f"{tag}: output '{k}' differs from HEAL_TC_HALO=0"
    # 2. the f32 output against float64
    x64 = o["x"].double().sum(0).permute(0, 3, 1, 2)
    r64 = None if o["res"] is None else (ep._nchw64(o["res"]) if st.res == "f32" else o["res"].double().sum(0).permute(0, 3, 1, 2))
    w, b = ep._folded(*ep._modules(name, 0, st))
    y = ep._reference(st, w, b, x64, r64)
    bound = ep._bound(st, w, x64, y)
    err = (ep._nchw64(o["of"]) - y).abs()
    ratio = (err / bound).max().item()
    print(f"{tag}: max err / bound {ratio:.4f}  (max err {err.max().item():.3e}, max|y| {y.abs().max().item():.3f})")
    assert bool((err <= bound).all()), f"{tag}: {int((~(err <= bound)).sum())} elements outside the bound, max err / bound {ratio:.3f}"
    # 3. the product output and the f32 call's split / bf16 output are the rounding of the f32 output
    hi = o["of"].to(torch.bfloat16)
    for k in ("a", "ob"):
        assert torch.equal(ep._bits(o[k][0]), ep._bits(hi)), f"{tag}: '{k}' hi plane != bf16(f32 output)"
        if planes == 2:
            assert torch.equal(ep._bits(o[k][1]), ep._bits((o["of"] - hi.float()).to(torch.bfloat16))), f"{tag}: '{k}' lo plane"
