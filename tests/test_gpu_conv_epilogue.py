"""heal_conv2d_tc against a float64 reference, one case per kernel configuration its dispatch can reach.

Every case runs each conv twice: the product call (A: split/bf16 output only, which drains through the staging tile and a TMA
store wherever that epilogue is eligible, or the f32 output a head asks for) and a call that also asks for f32 (B: the
direct-store epilogue).  The checks, in tc32 (split activations, planes 2/2) and the 'bf16' mode (planes 1/2):
  - A and B agree bit for bit: both epilogues add bias, residual hi, residual lo in that order and round the same way;
  - B's f32 output is within a per-element bound of float64 computed from the nn modules themselves (so the BN fold and the
    packing are covered), on the exact input the kernel read;
  - B's split/bf16 output is exactly the rounding of its f32 output;
  - channels around a slice that is written, or read, still hold their sentinel.

The bound is |got - y64| <= ALPHA * (|W| (*) |x|) + 2^-22 |y64|, where |W| (*) |x| is the same convolution on absolute
values; for GELU the first term is multiplied by max |GELU'|.  test_bound_rejects_plausible_kernel_bugs (no GPU) shows that
the bound is sharp enough to reject each plausible epilogue or operand bug on these cases."""
import math
import re
import zlib
from dataclasses import dataclass
from typing import Optional, Tuple

import pytest
import torch
import torch.nn.functional as F

# Split operands carry ~2^-17 relative error, the dropped lo x lo product ~2^-16, and the products accumulate in fp32.
# Calibrated on an H100 80GB HBM3: with ALPHA = 2^-14 the largest err / bound over all cases and both modes was 0.105
# (g32_tile, tc32; 0.054 in the 'bf16' mode), so these kernels need ALPHA >= 2^-17.25.  2^-16 leaves 2.4x of headroom.
# test_conv_epilogue prints err / bound for every case.
ALPHA = 2.0 ** -16
REL = 2.0 ** -22
GELU_SLOPE = 1.13          # max |GELU'(v)| = 1.1289, at v = sqrt(2)
SENTINEL = -1000.0         # finite and exact in bf16: fills the channels around a slice

MODES = {"tc32": ("split", 2), "bf16": ("bf16", 1)}     # activation format and planes; the weights always carry 2 planes


@dataclass(frozen=True)
class Stage:
    cin: int
    cout: int
    k: int = 1
    stride: int = 1
    groups: int = 1
    deconv: bool = False                          # ConvTranspose2d with kernel == stride == k
    bn: bool = True
    act: int = 1                                  # 0 none, 1 ReLU, 2 GELU (erf)
    res: Optional[str] = None                     # None | 'act' (the mode's format) | 'f32' | 'input' (the case's input map)
    out: str = "act"                              # what the product call writes: 'act' (split / bf16) or 'f32'
    out_slice: Optional[Tuple[int, int]] = None   # (buffer width, channel offset) the product call writes into
    in_slice: Optional[Tuple[int, int]] = None    # (buffer width, channel offset) the input is read from

    @property
    def pad(self):
        return 0 if self.deconv else self.k // 2

    @property
    def fan_in(self):
        return self.cin if self.deconv else self.cin // self.groups * self.k * self.k

    def out_hw(self, H, W):
        if self.deconv:
            return H * self.k, W * self.k
        return (H + 2 * self.pad - self.k) // self.stride + 1, (W + 2 * self.pad - self.k) // self.stride + 1


# name, (N, H, W), stages, the k_conv2d_tc<BLOCK_N, STAGES, STG[, gelu][, grouped]> instantiations the A and B runs reach
CASES = [
    # <128,2,2> with the split residual TMA-loaded into the staging buffers: 384 tiles, 2-3 per CTA (cross-tile prefetch)
    ("res_split_1x1_n128", (3, 64, 256), [Stage(64, 128, res="act")], {"128,2,2", "128,3,0"}),
    # <128,2,2> residual TMA, 2 n-tiles per pixel tile, 160 tiles
    ("res_split_3x3_n256", (2, 40, 72), [Stage(128, 256, 3, res="act")], {"128,2,2", "128,3,0"}),
    # <128,3,1>: the single staging buffer is refilled right after bulk_wait_read<0>
    ("nores_3x3_n256", (2, 40, 72), [Stage(128, 256, 3)], {"128,3,1", "128,3,0"}),
    # <128,3,1> with the staged f32 residual; 150 columns = a 128-pixel tile and a ragged 22-pixel one
    ("res_f32_3x3_n128", (2, 33, 150), [Stage(64, 128, 3, res="f32")], {"128,3,1", "128,3,0"}),
    # <128,2,2>, coutp 256: the chunk [192, 256) is staged and clipped by the TMA store; into channels [64, 256) of 320
    ("n192_slice", (2, 24, 40), [Stage(64, 192, out_slice=(320, 64))], {"128,2,2", "128,3,0"}),
    # <128,2,2> residual TMA: the residual box [192, 256) lies past Cout and is zero-filled
    ("n192_res_split", (1, 24, 40), [Stage(768, 192, res="act")], {"128,2,2", "128,3,0"}),
    # <128,3,1> with an f32 residual and a chunk past Cout: neither bias nor residual may be read there
    ("n192_res_f32", (1, 24, 40), [Stage(64, 192, 3, res="f32")], {"128,3,1", "128,3,0"}),
    # <128,2,2>, 3 n-tiles, the last one half past Cout
    ("n320", (1, 24, 40), [Stage(128, 320)], {"128,2,2", "128,3,0"}),
    # <128,2,2,GELU>
    ("gelu_k1", (2, 24, 40), [Stage(64, 256, bn=False, act=2)], {"128,2,2,gelu", "128,3,0,gelu"}),
    ("gelu_n192", (2, 24, 40), [Stage(64, 192, bn=False, act=2)], {"128,2,2,gelu", "128,3,0,gelu"}),
    # <128,3,1,GELU>: 6 k-blocks
    ("gelu_k6", (1, 24, 40), [Stage(384, 512, bn=False, act=2)], {"128,3,1,gelu", "128,3,0,gelu"}),
    # <128,3,0,GELU>
    ("gelu_f32", (1, 24, 40), [Stage(64, 256, bn=False, act=2, out="f32")], {"128,3,0,gelu"}),
    # halo <64,2,2> residual TMA (the lidar ResNet level-0 BasicBlock), 320 tiles
    ("halo_res", (2, 80, 256), [Stage(64, 64, 3, res="act")], {"64,2,2", "64,2,0"}),
    # halo <64,2,0>
    ("halo_f32", (1, 8, 256), [Stage(64, 64, 3, out="f32")], {"64,2,0"}),
    # <64,3,2> residual TMA; the f32 run is <64,4,0>
    ("n64_res", (2, 24, 96), [Stage(64, 64, 3, res="act")], {"64,3,2", "64,4,0"}),
    # <64,4,0>: an odd channel offset takes the scalar-store branch
    ("n48_odd_slice", (1, 17, 23), [Stage(64, 48, out_slice=(56, 3))], {"64,4,0"}),
    # <16,4,0>: f32 into column 1 of a 3-wide map (scalar f32 stores)
    ("n1_head", (2, 24, 40), [Stage(64, 1, bn=False, act=0, out="f32", out_slice=(3, 1))], {"16,4,0"}),
    # <32,4,0>
    ("n20_head", (2, 24, 40), [Stage(256, 20, bn=False, act=0)], {"32,4,0"}),
    # grouped, two-row tiles: <64,3,2,G>; the f32 run is <64,4,0,G>
    ("g32_tile", (1, 24, 96), [Stage(128, 128, 3, groups=32)], {"64,3,2,grouped", "64,4,0,grouped"}),
    # grouped halo with the packed diagonal weights: <64,3,2,G> / <64,4,0,G> (W % 128 != 0 keeps it off the row-ring kernel)
    ("g32_halo", (1, 6, 150), [Stage(128, 128, 3, groups=32)], {"64,3,2,grouped", "64,4,0,grouped"}),
    # <128,3,1>: stride 2 through TMA element strides
    ("s2_3x3", (1, 41, 57), [Stage(64, 128, 3, stride=2)], {"128,3,1", "128,3,0"}),
    # <128,3,0>
    ("s2_1x1_f32", (1, 41, 57), [Stage(64, 128, 1, stride=2, act=0, out="f32")], {"128,3,0"}),
    # direct stores, 2x2 sub-positions as n-tiles; into channels [128, 256) of 384
    ("deconv_up2_slice", (2, 12, 20), [Stage(128, 128, 2, deconv=True, out_slice=(384, 128))], {"128,3,0"}),
    # TW 8 / TH 16 tiles, most of each tile out of range: <128,2,2> residual TMA
    ("tiny_5x7", (1, 5, 7), [Stage(64, 128, 3, res="act")], {"128,2,2", "128,3,0"}),
    ("tiny_s2_3x3", (1, 3, 3), [Stage(64, 128, 3, stride=2, res="act")], {"128,2,2", "128,3,0"}),
    ("tiny_1x1", (1, 1, 1), [Stage(64, 128, 3, res="act")], {"128,2,2", "128,3,0"}),
    # an activation tensor map with cstride 192 != Cin 64: <64,3,2>
    ("input_slice", (1, 24, 40), [Stage(64, 64, 3, in_slice=(192, 64))], {"64,3,2", "64,4,0"}),
    # three dependent PDL launches, no synchronisation between them: <128,2,2>, <128,3,1>, <64,3,2> + the case's input
    ("pdl_chain", (1, 40, 256), [Stage(64, 128), Stage(128, 128, 3), Stage(128, 64, res="input")],
     {"128,2,2", "128,3,1", "64,3,2", "128,3,0", "64,4,0"}),
]
CASE = {c[0]: c for c in CASES}

# every instantiation heal_conv2d_tc can dispatch to from ops.conv2d_tc (which always passes the packed diagonal weights, so
# the grouped <64,2,x,G> forms are unreachable)
REACHABLE = {"16,4,0", "32,4,0", "64,2,0", "64,4,0", "64,2,2", "64,3,2", "128,3,0", "128,2,2", "128,3,1",
             "128,2,2,gelu", "128,3,1,gelu", "128,3,0,gelu", "64,3,2,grouped", "64,4,0,grouped"}


# ------------------------------------------------------------------------------------------------ float64 reference
def _modules(name, i, st):
    gen = torch.Generator().manual_seed(zlib.crc32(f"{name}/{i}".encode()))
    if st.deconv:
        conv = torch.nn.ConvTranspose2d(st.cin, st.cout, st.k, stride=st.k)
    else:
        conv = torch.nn.Conv2d(st.cin, st.cout, st.k, stride=st.stride, padding=st.pad, groups=st.groups)
    bn = torch.nn.BatchNorm2d(st.cout, eps=1e-3).eval() if st.bn else None
    with torch.no_grad():
        # GELU: a small convolution under widely spread biases, so that pre-activations reach |v| ~ 2.7, where the erf and
        # tanh forms differ most, while |W| (*) |x| stays small
        conv.weight.copy_(torch.randn(conv.weight.shape, generator=gen) * ((0.25 if st.act == 2 else 1.0) / math.sqrt(st.fan_in)))
        conv.bias.copy_(torch.rand(st.cout, generator=gen) * 7 - 3.5 if st.act == 2 else torch.randn(st.cout, generator=gen) * 0.1)
        if bn is not None:
            bn.weight.copy_(torch.rand(st.cout, generator=gen) + 0.5)
            bn.bias.copy_(torch.randn(st.cout, generator=gen) * 0.1)
            bn.running_mean.copy_(torch.randn(st.cout, generator=gen) * 0.1)
            bn.running_var.copy_(torch.rand(st.cout, generator=gen) + 0.5)
    return conv, bn


def _folded(conv, bn):
    """Eval BatchNorm folded into the conv's weight and bias, in float64."""
    w, b = conv.weight.detach().double(), conv.bias.detach().double()
    if bn is not None:
        s = bn.weight.detach().double() / torch.sqrt(bn.running_var.detach().double() + bn.eps)
        b = (b - bn.running_mean.detach().double()) * s + bn.bias.detach().double()
        w = w * (s.view(1, -1, 1, 1) if isinstance(conv, torch.nn.ConvTranspose2d) else s.view(-1, 1, 1, 1))
    return w, b


def _conv(st, x, w):
    if st.deconv:
        return F.conv_transpose2d(x, w, stride=st.k)
    return F.conv2d(x, w, stride=st.stride, padding=st.pad, groups=st.groups)


def _gelu(v, tanh=False):
    if tanh:
        return 0.5 * v * (1 + torch.tanh(math.sqrt(2 / math.pi) * (v + 0.044715 * v ** 3)))
    return 0.5 * v * (1 + torch.erf(v / math.sqrt(2)))


def _reference(st, w, b, x, r, fault=None):
    """act(conv(x) + b + r) in float64; `fault` = 'relu_first' / 'tanh_gelu' restates that epilogue bug."""
    v = _conv(st, x, w) + b.view(1, -1, 1, 1)
    if fault == "relu_first":
        v = v.clamp_min(0)
    if r is not None:
        v = v + r
    if st.act == 1 and fault != "relu_first":
        v = v.clamp_min(0)
    elif st.act == 2:
        v = _gelu(v, tanh=fault == "tanh_gelu")
    return v


def _bound(st, w, x, y):
    return ALPHA * (GELU_SLOPE if st.act == 2 else 1.0) * _conv(st, x.abs(), w.abs()) + REL * y.abs()


def _exact(x32, planes):
    """The value a kernel reads when fp32 `x32` is stored as bf16 hi (planes 1) or hi + lo (planes 2), in float64."""
    hi = x32.to(torch.bfloat16)
    if planes == 1:
        return hi.double()
    return hi.double() + (x32 - hi.float()).to(torch.bfloat16).double()


# ------------------------------------------------------------------------------------------------ the bound is sharp (CPU)
def _faults(st, mode):
    f = ["w_lo", "bias_chunk"]
    if mode == "tc32":
        f.append("act_lo")
        if st.res in ("act", "input"):
            f.append("res_lo")
    if st.act == 2:
        f.append("tanh_gelu")
    if st.act == 1 and st.res is not None:
        f.append("relu_first")
    return f


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("name", list(CASE))
def test_bound_rejects_plausible_kernel_bugs(name, mode):
    """Each plausible kernel bug, applied to the float64 computation of a shrunken case, leaves the bound on some element:
    the lo plane of the activations (tc32), of the weights or of a split residual dropped, the bias missing from one
    64-channel chunk, tanh-approximate GELU, ReLU before the residual add."""
    _, (N, H, W), stages, _ = CASE[name]
    planes = MODES[mode][1]
    H, W = min(H, 8), min(W, 16)
    gen = torch.Generator().manual_seed(zlib.crc32(f"cpu/{name}".encode()))
    x = torch.randn(1, stages[0].cin, H, W, generator=gen)
    x_in = x
    for i, st in enumerate(stages):
        w, b = _folded(*_modules(name, i, st))
        Ho, Wo = st.out_hw(H, W)
        r32 = x_in if st.res == "input" else torch.randn(1, st.cout, Ho, Wo, generator=gen) if st.res else None
        xe = _exact(x, planes)
        re_ = None if r32 is None else (r32.double() if st.res == "f32" else _exact(r32, planes))
        y = _reference(st, w, b, xe, re_)
        bound = _bound(st, w, xe, y)
        for fault in _faults(st, mode):
            xf, wf, bf, rf = xe, w, b, re_
            if fault == "act_lo":
                xf = _exact(x, 1)
            elif fault == "w_lo":
                wf = w.float().to(torch.bfloat16).double()
            elif fault == "res_lo":
                rf = _exact(r32, 1)
            elif fault == "bias_chunk":
                bf = b.clone()
                bf[64 * ((st.cout - 1) // 64):] = 0
            ratio = ((_reference(st, wf, bf, xf, rf, fault) - y).abs() / bound).max().item()
            assert ratio > 1, f"{name} [{mode}] stage {i}: the bound does not reject '{fault}' (max err / bound {ratio:.3f})"
        x, H, W = y.float(), Ho, Wo


# ------------------------------------------------------------------------------------------------ the kernels (GPU)
def _launch(name, mode):
    """The case's product calls (A) back to back with no synchronisation, then one call per stage that also writes f32 (B).
    Returns one record per stage."""
    from heal_b200 import ops
    fmt, planes = MODES[mode]
    _, (N, H, W), stages, _ = CASE[name]
    gen = torch.Generator().manual_seed(zlib.crc32(name.encode()))
    nan = float("nan")
    runs, prev, x_in = [], None, None
    for i, st in enumerate(stages):
        conv, bn = _modules(name, i, st)
        pc = ops.pack_conv_tc(conv, bn, st.act, planes=2).to("cuda")
        Ho, Wo = st.out_hw(H, W)
        if prev is None:
            width, coff = st.in_slice or (st.cin, 0)
            x32 = torch.full((N, width, H, W), SENTINEL)
            x32[:, coff:coff + st.cin] = torch.randn(N, st.cin, H, W, generator=gen)
            x = x_in = ops.convert(ops.to_act(x32.cuda()), fmt)
        else:
            x, coff = prev, 0
        res = None
        if st.res == "act":
            res = ops.convert(ops.to_act(torch.randn(N, st.cout, Ho, Wo, generator=gen).cuda()), fmt)
        elif st.res == "f32":
            res = ops.to_act(torch.randn(N, st.cout, Ho, Wo, generator=gen).cuda())
        elif st.res == "input":
            res = x_in
        width, oco = st.out_slice or (st.cout, 0)
        fill = SENTINEL if st.out_slice else nan
        if st.out == "act":
            a = torch.full((planes, N, Ho, Wo, width), fill, dtype=torch.bfloat16, device="cuda")
            ops.conv2d_tc(x, pc, residual=res, out=ops.Act(a, fmt), out_coffset=oco, in_coffset=coff)
            prev = ops.Act(a, fmt)
        else:
            a = torch.full((N, Ho, Wo, width), fill, dtype=torch.float32, device="cuda")
            ops.conv2d_tc(x, pc, residual=res, want_split=False, out_f32=ops.Act(a, "f32"), want_f32=True, out32_coffset=oco,
                          in_coffset=coff)
            prev = None
        runs.append(dict(st=st, conv=conv, bn=bn, pc=pc, x=x, coff=coff, res=res, a=a, oco=oco))
        H, W = Ho, Wo
    for run in runs:
        st, a = run["st"], run["a"]
        N_, Ho, Wo = a.shape[-4:-1]
        run["ob"] = torch.full((planes, N_, Ho, Wo, st.cout), nan, dtype=torch.bfloat16, device="cuda")
        run["of"] = torch.full((N_, Ho, Wo, st.cout), nan, dtype=torch.float32, device="cuda")
        ops.conv2d_tc(run["x"], run["pc"], residual=run["res"], out=ops.Act(run["ob"], fmt), out_f32=ops.Act(run["of"], "f32"),
                      want_f32=True, in_coffset=run["coff"])
    return runs


def _bits(t):
    t = t.contiguous()
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


def _nchw64(t_nhwc):
    return t_nhwc.double().permute(0, 3, 1, 2)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("name", list(CASE))
def test_conv_epilogue(name, mode):
    planes = MODES[mode][1]
    runs = _launch(name, mode)
    torch.cuda.synchronize()
    for i, run in enumerate(runs):
        st, cout, oco = run["st"], run["st"].cout, run["oco"]
        tag = f"{name} [{mode}] stage {i}"
        a, ob, of = run["a"].cpu(), run["ob"].cpu(), run["of"].cpu()
        # 1. the product call and the direct-store call agree bit for bit
        if st.out == "act":
            assert torch.equal(_bits(a[..., oco:oco + cout]), _bits(ob)), f"{tag}: staging and direct-store epilogues differ"
        else:
            assert torch.equal(_bits(a[..., oco:oco + cout]), _bits(of)), f"{tag}: f32-only and split + f32 outputs differ"
        # 2. the f32 output against float64, element by element
        x = run["x"].t[..., run["coff"]:run["coff"] + st.cin].cpu()
        x64 = x.double().sum(0).permute(0, 3, 1, 2)
        r64 = None
        if run["res"] is not None:
            rt = run["res"].t.cpu()
            r64 = _nchw64(rt) if run["res"].fmt == "f32" else rt.double().sum(0).permute(0, 3, 1, 2)
        w, b = _folded(run["conv"], run["bn"])
        y = _reference(st, w, b, x64, r64)
        bound = _bound(st, w, x64, y)
        err = (_nchw64(of) - y).abs()
        ratio = (err / bound).max().item()
        print(f"{tag}: max err / bound {ratio:.4f}  (max err {err.max().item():.3e}, max|y| {y.abs().max().item():.3f}, ALPHA 2^{math.log2(ALPHA):.0f})")
        assert bool((err <= bound).all()), f"{tag}: {int((~(err <= bound)).sum())} elements outside the bound, max err / bound {ratio:.3f}"
        # 3. the split / bf16 output is the rounding of the f32 output
        hi = of.to(torch.bfloat16)
        assert torch.equal(_bits(ob[0]), _bits(hi)), f"{tag}: hi plane != bf16(f32 output)"
        if planes == 2:
            assert torch.equal(_bits(ob[1]), _bits((of - hi.float()).to(torch.bfloat16))), f"{tag}: lo plane != bf16(f32 - hi)"
        # 4. the channels around a slice keep their sentinel
        if st.out_slice:
            around = torch.cat([a[..., :oco].flatten(), a[..., oco + cout:].flatten()]).float()
            assert bool((around == SENTINEL).all()), f"{tag}: a write spilled out of channels [{oco}, {oco + cout})"
        if st.in_slice:
            xb = run["x"].t.cpu().double().sum(0)
            coff = run["coff"]
            around = torch.cat([xb[..., :coff].flatten(), xb[..., coff + st.cin:].flatten()])
            assert bool((around == SENTINEL).all()), f"{tag}: the input buffer around the slice changed"


_KERNEL = re.compile(r"k_conv2d_tc<\s*(?:\(int\))?(\d+),\s*(?:\(int\))?(\d+),\s*(?:\(int\))?(\d+),\s*(true|false|\(bool\)[01]),"
                     r"\s*(true|false|\(bool\)[01])\s*>")


def _config(m):
    on = lambda s: s in ("true", "(bool)1")
    return ",".join(m.group(1, 2, 3)) + (",gelu" if on(m.group(4)) else "") + (",grouped" if on(m.group(5)) else "")


@pytest.mark.gpu
def test_cases_reach_every_dispatch_configuration():
    """Each case runs the instantiations its row names (kernel names from torch.profiler), and together the cases run every
    instantiation the dispatch can reach: a change to the dispatch cannot quietly move a case off what it exists to test."""
    from torch.profiler import ProfilerActivity, profile
    seen_all = set()
    for name, _, _, reaches in CASES:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            _launch(name, "tc32")
            torch.cuda.synchronize()
        seen = {_config(m) for e in prof.key_averages() for m in [_KERNEL.search(e.key)] if m}
        assert seen == reaches, f"{name}: ran {sorted(seen)}, expected {sorted(reaches)}"
        seen_all |= seen
    assert seen_all == REACHABLE
