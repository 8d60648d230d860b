"""Fused ResNeXt bottleneck (heal_bottleneck_tc): bit-identical to the three heal_conv2d_tc launches it replaces, and within
the conv engine's tolerances of a PyTorch CPU fp32 bottleneck."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

SHAPES = [(2, 19, 40), (1, 37, 256), (1, 5, 7), (3, 33, 24)]
FMTS = [("split", 2), ("bf16", 1)]


def _block(seed, bn1_shift=0.0):
    """PyramidFusion's level-0 bottleneck (64 -> 128 -> 64, 32 groups) with random BN statistics."""
    g = torch.Generator().manual_seed(seed)
    convs = [torch.nn.Conv2d(64, 128, 1, bias=False), torch.nn.Conv2d(128, 128, 3, padding=1, groups=32, bias=False),
             torch.nn.Conv2d(128, 64, 1, bias=False)]
    bns = [torch.nn.BatchNorm2d(c).eval() for c in (128, 128, 64)]
    with torch.no_grad():
        for conv in convs:
            fan_in = conv.weight[0].numel()
            conv.weight.copy_(torch.randn(conv.weight.shape, generator=g) * (2.0 / fan_in) ** 0.5)
        for bn in bns:
            c = bn.num_features
            bn.weight.copy_(torch.rand(c, generator=g) + 0.5)
            bn.bias.copy_(torch.randn(c, generator=g) * 0.1)
            bn.running_mean.copy_(torch.randn(c, generator=g) * 0.1)
            bn.running_var.copy_(torch.rand(c, generator=g) + 0.5)
        bns[0].bias.add_(bn1_shift)
    return convs, bns


def _reference(convs, bns, x):
    with torch.no_grad():
        y = F.relu(bns[0](convs[0](x)))
        y = F.relu(bns[1](convs[1](y)))
        return F.relu(bns[2](convs[2](y)) + x)


def _packed(convs, bns):
    from heal_b200 import ops
    return [ops.pack_conv_tc(c, b, True, planes=2).to("cuda") for c, b in zip(convs, bns)]


def _three_launches(x, pcs):
    from heal_b200 import ops
    mid, _ = ops.conv2d_tc(x, pcs[0])
    g, _ = ops.conv2d_tc(mid, pcs[1])
    y, _ = ops.conv2d_tc(g, pcs[2], residual=x)
    return y


def _check_reference(got, ref, planes):
    scale = ref.abs().max().item()
    err = (got - ref).abs().max().item()
    tol = 1e-3 if planes == 2 else (1e-2 + 4e-3) * max(scale, 1.0)
    assert err < tol, (err, tol, scale)


@pytest.mark.parametrize("shape", SHAPES, ids=[f"n{n}_{h}x{w}" for n, h, w in SHAPES])
@pytest.mark.parametrize("fmt,planes", FMTS, ids=[f for f, _ in FMTS])
def test_bottleneck_matches_three_launches_and_reference(shape, fmt, planes):
    from heal_b200 import ops
    N, H, W = shape
    convs, bns = _block(H * W + N)
    x = torch.randn(N, 64, H, W, generator=torch.Generator().manual_seed(N + H + W))
    pcs = _packed(convs, bns)
    xa = ops.convert(ops.to_act(x.cuda()), fmt)
    fused = ops.bottleneck_tc(xa, *pcs)
    three = _three_launches(xa, pcs)
    torch.cuda.synchronize()
    assert torch.equal(fused.t, three.t)
    _check_reference(ops.act_to_nchw(fused).cpu(), _reference(convs, bns, x), planes)


@pytest.mark.parametrize("fmt,planes", FMTS, ids=[f for f, _ in FMTS])
def test_bottleneck_zero_pads_the_mid_map(fmt, planes):
    """A large positive bn1 shift makes ReLU(bias1) large: mid pixels outside the image must still be 0, not ReLU(bias1)."""
    from heal_b200 import ops
    convs, bns = _block(7, bn1_shift=5.0)
    x = torch.randn(2, 64, 21, 19, generator=torch.Generator().manual_seed(7))
    pcs = _packed(convs, bns)
    xa = ops.convert(ops.to_act(x.cuda()), fmt)
    fused = ops.bottleneck_tc(xa, *pcs)
    torch.cuda.synchronize()
    assert torch.equal(fused.t, _three_launches(xa, pcs).t)
    _check_reference(ops.act_to_nchw(fused).cpu(), _reference(convs, bns, x), planes)


def test_bottleneck_writes_a_channel_slice_and_replays_in_a_graph():
    from heal_b200 import ops
    convs, bns = _block(11)
    x = torch.randn(2, 64, 24, 40, generator=torch.Generator().manual_seed(11))
    pcs = _packed(convs, bns)
    xa = ops.convert(ops.to_act(x.cuda()), "split")
    ref = ops.bottleneck_tc(xa, *pcs)
    buf = torch.full((2, 2, 24, 40, 192), 3.0, dtype=torch.bfloat16, device="cuda")
    ops.bottleneck_tc(xa, *pcs, out=ops.Act(buf, "split"), out_coffset=64)
    torch.cuda.synchronize()
    assert torch.equal(buf[..., 64:128], ref.t)
    assert torch.all(buf[..., :64] == 3.0) and torch.all(buf[..., 128:] == 3.0)

    out = ops.act_empty(2, 24, 40, 64, "split", "cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        ops.bottleneck_tc(xa, *pcs, out=out)
    torch.cuda.current_stream().wait_stream(side)
    out.t.zero_()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.bottleneck_tc(xa, *pcs, out=out)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out.t, ref.t)
