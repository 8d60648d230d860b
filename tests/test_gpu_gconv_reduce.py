"""Fused grouped 3x3 + 1x1 reduce of the stride-1 level-1 and level-2 ResNeXt bottlenecks (heal_gconv_reduce_tc): bit-identical
to the two heal_conv2d_tc launches it replaces, and within the conv engine's tolerances of a float64 bottleneck."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

# (C, N, H, W): level 1 (128 -> 256 -> 128) and level 2 (256 -> 512 -> 256), at frame width and on maps that leave partial
# 16 x 8 tiles (and send the grouped conv of the two-launch path through its row-ring and its halo-tile kernels)
SHAPES = [(128, 1, 128, 128), (128, 5, 72, 72), (128, 2, 40, 136), (256, 1, 64, 64), (256, 2, 40, 136), (256, 5, 21, 19)]
FMTS = [("split", 2), ("bf16", 1)]


def _block(C, seed):
    """PyramidFusion's bottleneck C -> 2C -> C (32 groups) with random BN statistics and non-zero BN shifts, so that ReLU(bias)
    is not 0 at the padded pixels of either conv's input."""
    g = torch.Generator().manual_seed(seed)
    width = 2 * C
    convs = [torch.nn.Conv2d(C, width, 1, bias=False), torch.nn.Conv2d(width, width, 3, padding=1, groups=32, bias=False),
             torch.nn.Conv2d(width, C, 1, bias=False)]
    bns = [torch.nn.BatchNorm2d(c).eval() for c in (width, width, C)]
    with torch.no_grad():
        for conv in convs:
            fan_in = conv.weight[0].numel()
            conv.weight.copy_(torch.randn(conv.weight.shape, generator=g) * (2.0 / fan_in) ** 0.5)
        for bn in bns:
            c = bn.num_features
            bn.weight.copy_(torch.rand(c, generator=g) + 0.5)
            bn.bias.copy_(torch.randn(c, generator=g) * 0.1 + 0.3)
            bn.running_mean.copy_(torch.randn(c, generator=g) * 0.1)
            bn.running_var.copy_(torch.rand(c, generator=g) + 0.5)
    return convs, bns


def _reference(convs, bns, x):
    """The whole block in float64 on the CPU."""
    import copy
    c64 = [copy.deepcopy(m).double() for m in convs]
    b64 = [copy.deepcopy(m).double() for m in bns]
    with torch.no_grad():
        x = x.double()
        y = F.relu(b64[0](c64[0](x)))
        y = F.relu(b64[1](c64[1](y)))
        return F.relu(b64[2](c64[2](y)) + x)


def _run(C, N, H, W, fmt, seed):
    from heal_b200 import ops
    convs, bns = _block(C, seed)
    x = torch.randn(N, C, H, W, generator=torch.Generator().manual_seed(seed + 1))
    pcs = [ops.pack_conv_tc(c, b, True, planes=2).to("cuda") for c, b in zip(convs, bns)]
    xa = ops.convert(ops.to_act(x.cuda()), fmt)
    mid, _ = ops.conv2d_tc(xa, pcs[0])
    return convs, bns, x, pcs, xa, mid


def _two_launches(mid, xa, pcs):
    from heal_b200 import ops
    g, _ = ops.conv2d_tc(mid, pcs[1])
    y, _ = ops.conv2d_tc(g, pcs[2], residual=xa)
    return y


@pytest.mark.parametrize("shape", SHAPES, ids=[f"c{c}_n{n}_{h}x{w}" for c, n, h, w in SHAPES])
@pytest.mark.parametrize("fmt,planes", FMTS, ids=[f for f, _ in FMTS])
def test_gconv_reduce_matches_two_launches_and_reference(shape, fmt, planes):
    from heal_b200 import ops
    C, N, H, W = shape
    convs, bns, x, pcs, xa, mid = _run(C, N, H, W, fmt, C + H * W + N)
    fused = ops.gconv_reduce_tc(mid, pcs[1], pcs[2], xa)
    two = _two_launches(mid, xa, pcs)
    torch.cuda.synchronize()
    assert torch.equal(fused.t, two.t)
    ref = _reference(convs, bns, x)
    got = ops.act_to_nchw(fused).cpu().double()
    scale = ref.abs().max().item()
    err = (got - ref).abs().max().item()
    tol = 1e-3 * max(scale, 1.0) if planes == 2 else (1e-2 + 4e-3) * max(scale, 1.0)
    assert err < tol, (err, tol, scale)


@pytest.mark.parametrize("fmt", ["split", "bf16"])
def test_gconv_reduce_writes_a_channel_slice_and_replays_in_a_graph(fmt):
    from heal_b200 import ops
    C, N, H, W = 128, 2, 24, 40
    _, _, _, pcs, xa, mid = _run(C, N, H, W, fmt, 11)
    ref = ops.gconv_reduce_tc(mid, pcs[1], pcs[2], xa)
    P = 2 if fmt == "split" else 1
    buf = torch.full((P, N, H, W, 3 * C), 3.0, dtype=torch.bfloat16, device="cuda")
    ops.gconv_reduce_tc(mid, pcs[1], pcs[2], xa, out=ops.Act(buf, fmt), out_coffset=C)
    torch.cuda.synchronize()
    assert torch.equal(buf[..., C:2 * C], ref.t)
    assert torch.all(buf[..., :C] == 3.0) and torch.all(buf[..., 2 * C:] == 3.0)

    out = ops.act_empty(N, H, W, C, fmt, "cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        ops.gconv_reduce_tc(mid, pcs[1], pcs[2], xa, out=out)
    torch.cuda.current_stream().wait_stream(side)
    out.t.zero_()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.gconv_reduce_tc(mid, pcs[1], pcs[2], xa, out=out)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out.t, ref.t)
