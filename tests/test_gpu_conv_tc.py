"""wgmma implicit-GEMM conv (heal_conv2d_tc) vs PyTorch CPU fp32, ordered from a bare GEMM tile to full features.
fp32-equivalent (split-bf16, planes=2) must meet 1e-3 (typically ~2e-5); bf16 (planes=1) must meet 1e-2 relative to scale."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

CASES = [
    # name, N, Cin, H, W, Cout, k, pad, bias, bn, relu, res ('none'|'split'|'f32')
    ("gemm_1tile", 1, 64, 1, 128, 64, 1, 0, False, False, False, "none"),
    ("gemm_k128", 1, 128, 1, 128, 64, 1, 0, False, False, False, "none"),
    ("gemm_2rows", 1, 64, 2, 128, 64, 1, 0, False, False, False, "none"),
    ("gemm_n128", 1, 64, 4, 128, 128, 1, 0, False, False, False, "none"),
    ("gemm_n256_persist", 2, 128, 64, 128, 256, 1, 0, True, False, True, "none"),
    ("conv3x3_basic", 1, 64, 8, 128, 64, 3, 1, False, False, False, "none"),
    ("conv3x3_w64", 2, 64, 16, 64, 64, 3, 1, False, True, True, "split"),
    ("conv3x3_w16", 1, 128, 16, 16, 128, 3, 1, True, False, True, "f32"),
    ("conv3x3_shrink", 1, 384, 32, 32, 256, 3, 1, True, False, True, "none"),
    ("conv3x3_ragged", 1, 64, 19, 40, 64, 3, 1, False, True, True, "split"),
    ("conv1x1_n16", 1, 64, 8, 64, 1, 1, 0, True, False, False, "none"),
    ("conv1x1_n32", 1, 256, 8, 64, 20, 1, 0, True, False, False, "none"),
    ("conv1x1_big", 5, 64, 64, 128, 128, 1, 0, False, True, True, "none"),
]


def _mk(case):
    name, N, Cin, H, W, Cout, k, pad, bias, bn, relu, res = case
    gen = torch.Generator().manual_seed(abs(hash(name)) % 10000)
    conv = torch.nn.Conv2d(Cin, Cout, k, padding=pad, bias=bias)
    bnm = torch.nn.BatchNorm2d(Cout, eps=1e-3).eval() if bn else None
    with torch.no_grad():
        conv.weight.copy_(torch.randn(conv.weight.shape, generator=gen) * (1.0 / (Cin * k * k)) ** 0.5)
        if bias:
            conv.bias.copy_(torch.randn(Cout, generator=gen) * 0.1)
        if bn:
            bnm.weight.copy_(torch.rand(Cout, generator=gen) + 0.5)
            bnm.bias.copy_(torch.randn(Cout, generator=gen) * 0.1)
            bnm.running_mean.copy_(torch.randn(Cout, generator=gen) * 0.1)
            bnm.running_var.copy_(torch.rand(Cout, generator=gen) + 0.5)
    x = torch.randn(N, Cin, H, W, generator=gen)
    with torch.no_grad():
        y = conv(x)
        if bn:
            y = bnm(y)
        r = torch.randn(y.shape, generator=gen) if res != "none" else None
        if r is not None:
            y = y + r
        if relu:
            y = F.relu(y)
    return conv, bnm, x, r, y


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
@pytest.mark.parametrize("planes,wplanes", [(2, 2), (1, 2), (1, 1)], ids=["tc32", "bf16act_splitw", "bf16"])
def test_conv_tc(case, planes, wplanes):
    """(activation planes, weight planes): (2,2) fp32-equivalent; (1,2) the engine's 'bf16' mode; (1,1) plain bf16 x bf16."""
    from heal_b200 import ops
    name, N, Cin, H, W, Cout, k, pad, bias, bn, relu, res = case
    conv, bnm, x, r, y = _mk(case)
    pc = ops.pack_conv_tc(conv, bnm, relu, planes=wplanes).to("cuda")
    fmt = "split" if planes == 2 else "bf16"
    xs = ops.convert(ops.to_act(x.cuda()), fmt)
    rr = None
    if res == "split":
        rr = ops.convert(ops.to_act(r.cuda()), fmt)
    elif res == "f32":
        rr = ops.to_act(r.cuda())
    o_split, o_f32 = ops.conv2d_tc(xs, pc, residual=rr, want_split=True, want_f32=True)
    torch.cuda.synchronize()
    got32 = ops.act_to_nchw(o_f32).cpu()
    gots = ops.act_to_nchw(o_split).cpu()
    scale = y.abs().max().item()
    e32 = (got32 - y).abs().max().item()
    es = (gots - y).abs().max().item()
    print(f"{name} planes={planes}/{wplanes}: max|y|={scale:.3f} err_f32out={e32:.3e} err_splitout={es:.3e}")
    if planes == 2:
        assert e32 < 1e-3 and es < 1e-3
    else:       # bf16 activations: north_star's 1e-2 (relative to the tensor scale) for one layer; the bf16 OUTPUT adds its own rounding
        tol = (1e-2 if wplanes == 2 else 1.5e-2) * max(scale, 1.0)
        assert e32 < tol and es < tol + 4e-3 * max(scale, 1.0)


@pytest.mark.parametrize("up", [1, 2, 4])
def test_deconv_tc(up):
    from heal_b200 import ops
    gen = torch.Generator().manual_seed(up)
    cin = {1: 64, 2: 128, 4: 256}[up]
    de = torch.nn.ConvTranspose2d(cin, 128, up, stride=up, bias=False)
    bnm = torch.nn.BatchNorm2d(128, eps=1e-3).eval()
    with torch.no_grad():
        de.weight.copy_(torch.randn(de.weight.shape, generator=gen) * (1.0 / cin) ** 0.5)
        bnm.running_mean.copy_(torch.randn(128, generator=gen) * 0.1)
        bnm.running_var.copy_(torch.rand(128, generator=gen) + 0.5)
    x = torch.randn(2, cin, 16, 32, generator=gen)
    with torch.no_grad():
        y = F.relu(bnm(de(x)))
    pc = ops.pack_conv_tc(de, bnm, True, planes=2).to("cuda")
    xs = ops.convert(ops.to_act(x.cuda()), "split")
    buf = torch.zeros((2, 2, 16 * up, 32 * up, 384), dtype=torch.bfloat16, device="cuda")
    ops.conv2d_tc(xs, pc, out=ops.Act(buf, "split"), out_coffset=128)
    got = ops.merge_bf16(buf)[..., 128:256].permute(0, 3, 1, 2).cpu()
    err = (got - y).abs().max().item()
    print(f"deconv up={up}: err={err:.3e}")
    assert err < 1e-3
    assert torch.all(buf[..., :128] == 0) and torch.all(buf[..., 256:] == 0)


STRIDE_GROUP_CASES = [
    # name, N, C, H, W, Cout, k, stride, pad, groups
    ("s2_3x3_64", 2, 64, 32, 64, 64, 3, 2, 1, 1),
    ("s2_3x3_canvas", 1, 64, 64, 256, 64, 3, 2, 1, 1),
    ("s2_1x1_128_256", 1, 128, 32, 32, 256, 1, 2, 0, 1),
    ("s2_3x3_odd", 1, 64, 31, 45, 64, 3, 2, 1, 1),
    ("g32_cg4_s1", 2, 128, 24, 40, 128, 3, 1, 1, 32),
    ("g32_cg8_s2", 1, 256, 32, 64, 256, 3, 2, 1, 32),
    ("g32_cg16_s1", 1, 512, 16, 16, 512, 3, 1, 1, 32),
    ("g32_cg16_s2", 1, 512, 17, 23, 512, 3, 2, 1, 32),
    # one-row tiles (W >= 128): halo loads (one activation box per kernel row, base-offset descriptors)
    ("halo_res_w256", 2, 64, 5, 256, 64, 3, 1, 1, 1),
    ("halo_res_cin128_w128", 1, 128, 7, 128, 64, 3, 1, 1, 1),
    ("halo_ragged_w150", 1, 64, 4, 150, 64, 3, 1, 1, 1),
    ("halo_g32_cg4_w128", 1, 128, 6, 128, 128, 3, 1, 1, 32),
    ("halo_g32_cg8_w256", 1, 256, 3, 256, 256, 3, 1, 1, 32),
]


@pytest.mark.parametrize("case", STRIDE_GROUP_CASES, ids=[c[0] for c in STRIDE_GROUP_CASES])
def test_conv_tc_stride_grouped(case):
    from heal_b200 import ops
    name, N, C, H, W, Cout, k, stride, pad, groups = case
    gen = torch.Generator().manual_seed(abs(hash(name)) % 10000)
    conv = torch.nn.Conv2d(C, Cout, k, stride=stride, padding=pad, groups=groups, bias=False)
    bnm = torch.nn.BatchNorm2d(Cout, eps=1e-5).eval()
    with torch.no_grad():
        conv.weight.copy_(torch.randn(conv.weight.shape, generator=gen) * (1.0 / (C // groups * k * k)) ** 0.5)
        bnm.weight.copy_(torch.rand(Cout, generator=gen) + 0.5)
        bnm.bias.copy_(torch.randn(Cout, generator=gen) * 0.1)
        bnm.running_mean.copy_(torch.randn(Cout, generator=gen) * 0.1)
        bnm.running_var.copy_(torch.rand(Cout, generator=gen) + 0.5)
    x = torch.randn(N, C, H, W, generator=gen)
    with torch.no_grad():
        y = F.relu(bnm(conv(x)))
    assert ops.tc_eligible(conv)
    pc = ops.pack_conv_tc(conv, bnm, True, planes=2).to("cuda")
    o, _ = ops.conv2d_tc(ops.convert(ops.to_act(x.cuda()), "split"), pc)
    torch.cuda.synchronize()
    got = ops.act_to_nchw(o).cpu()
    assert got.shape == y.shape
    err = (got - y).abs().max().item()
    print(f"{name}: max|y|={y.abs().max().item():.3f} err={err:.3e}")
    assert err < 1e-3


RING_CASES = [
    # name, N, C, H, W, groups  -> strips x row segments (conv3x3_ring.cu): multi-segment, ragged last segment, one-row segments
    ("ring_cg4_w256_h37", 3, 128, 37, 256, 32),       # 12 strips x 8 segments of 5 rows (last: 2)
    ("ring_cg8_w128_h64", 5, 256, 64, 128, 32),       # 20 strips x 7 segments of 10 rows (last: 4)
    ("ring_cg4_w128_h5", 1, 128, 5, 128, 32),         # 2 strips, 1 segment: fewer rows than ring slots + 1
    ("ring_cg16_w128_h130", 1, 512, 130, 128, 32),    # 8 strips x 18 segments
]


@pytest.mark.parametrize("case", RING_CASES, ids=[c[0] for c in RING_CASES])
@pytest.mark.parametrize("planes", [2, 1], ids=["tc32", "bf16"])
def test_grouped_conv_row_ring(case, planes):
    """Grouped 3x3 on maps >= 128 wide runs the row-ring kernel: vs fp32 PyTorch on the CPU, and written into a channel slice of a
    wider buffer (the neighbours must stay untouched)."""
    from heal_b200 import ops
    name, N, C, H, W, groups = case
    gen = torch.Generator().manual_seed(abs(hash(name)) % 10000)
    conv = torch.nn.Conv2d(C, C, 3, padding=1, groups=groups, bias=False)
    bnm = torch.nn.BatchNorm2d(C, eps=1e-5).eval()
    with torch.no_grad():
        conv.weight.copy_(torch.randn(conv.weight.shape, generator=gen) * (1.0 / (C // groups * 9)) ** 0.5)
        bnm.weight.copy_(torch.rand(C, generator=gen) + 0.5)
        bnm.bias.copy_(torch.randn(C, generator=gen) * 0.1)
        bnm.running_mean.copy_(torch.randn(C, generator=gen) * 0.1)
        bnm.running_var.copy_(torch.rand(C, generator=gen) + 0.5)
    x = torch.randn(N, C, H, W, generator=gen)
    with torch.no_grad():
        y = F.relu(bnm(conv(x)))
    fmt = "split" if planes == 2 else "bf16"
    pc = ops.pack_conv_tc(conv, bnm, True, planes=2).to("cuda")
    xs = ops.convert(ops.to_act(x.cuda()), fmt)
    o, _ = ops.conv2d_tc(xs, pc)
    buf = torch.zeros((planes, N, H, W, C + 128), dtype=torch.bfloat16, device="cuda")
    ops.conv2d_tc(xs, pc, out=ops.Act(buf, fmt), out_coffset=64)
    torch.cuda.synchronize()
    got = ops.act_to_nchw(o).cpu()
    scale = max(y.abs().max().item(), 1.0)
    err = (got - y).abs().max().item()
    print(f"{name} planes={planes}: max|y|={scale:.3f} err={err:.3e}")
    assert err < (1e-3 if planes == 2 else 1.4e-2 * scale)
    assert torch.equal(buf[..., 64:64 + C], o.t) and torch.all(buf[..., :64] == 0) and torch.all(buf[..., 64 + C:] == 0)


def test_grouped_conv_row_ring_equals_tile_kernel(monkeypatch):
    """Same MMAs in the same order per output element: the ring kernel and the tile-per-CTA kernel agree bit for bit
    (HEAL_TC_RING is read once per process, so the tile kernel runs in a child process)."""
    import os, subprocess, sys, tempfile
    from heal_b200 import ops
    code = (
        "import sys, torch\n"
        "from heal_b200 import ops\n"
        "g = torch.Generator().manual_seed(5)\n"
        "conv = torch.nn.Conv2d(128, 128, 3, padding=1, groups=32, bias=False)\n"
        "conv.weight.data.copy_(torch.randn(conv.weight.shape, generator=g) / 6)\n"
        "x = torch.randn(2, 128, 21, 256, generator=g)\n"
        "pc = ops.pack_conv_tc(conv, None, True, planes=2).to('cuda')\n"
        "o, _ = ops.conv2d_tc(ops.convert(ops.to_act(x.cuda()), 'split'), pc)\n"
        "torch.cuda.synchronize()\n"
        "torch.save(o.t.cpu(), sys.argv[1])\n")
    outs = []
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with tempfile.TemporaryDirectory() as td:
        for ring in ("1", "0"):
            path = os.path.join(td, f"o{ring}.pt")
            env = dict(os.environ, HEAL_TC_RING=ring, PYTHONPATH=root)
            subprocess.run([sys.executable, "-c", code, path], check=True, env=env, timeout=300, cwd=root)
            outs.append(torch.load(path))
    assert torch.equal(outs[0], outs[1])
