"""EfficientNet camera encoder on the GPU: every csrc/mbconv.cu kernel against a float64 torch reference computed here, the whole
encoder (`CamEncode.heads_nhwc`) against its torch path and the golden made from the unmodified reference CamEncode, and
LiftSplatShoot / HeterPyramidCollab with `camera_encoder: EfficientNet` against their reference goldens."""
import copy
import os

import pytest
import torch
import torch.nn.functional as F

from oracle import efficientnet as oe
from oracle import golden

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _restore_precision():
    from heal_b200 import engine
    old = engine.PRECISION
    yield
    engine.set_precision(old)


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _bn(c, g, eps=1e-3):
    bn = torch.nn.BatchNorm2d(c, eps=eps).eval()
    with torch.no_grad():
        bn.weight.copy_(torch.rand(c, generator=g) + 0.5)
        bn.bias.copy_(torch.randn(c, generator=g) * 0.3)
        bn.running_mean.copy_(torch.randn(c, generator=g) * 0.2)
        bn.running_var.copy_(torch.rand(c, generator=g) + 0.5)
    return bn


def _bn64(bn, y):
    s = bn.weight.double() / torch.sqrt(bn.running_var.double() + bn.eps)
    return y * s[None, :, None, None] + (bn.bias.double() - bn.running_mean.double() * s)[None, :, None, None]


def _swish64(y):
    return y * torch.sigmoid(y)


def _close(got, ref, tol, what):
    err = (got.double().cpu() - ref).abs().max().item()
    scale = max(ref.abs().max().item(), 1.0)
    print(f"{what}: max|ref|={scale:.3f} err={err:.3e}")
    assert err <= tol * scale, (what, err, scale)


def _nhwc(a):
    return a.t.permute(0, 3, 1, 2)


@pytest.mark.parametrize("N,Cimg,H,W", [(1, 3, 33, 47), (5, 4, 32, 64), (2, 4, 17, 18)])
def test_stem_conv_swish(N, Cimg, H, W):
    from heal_b200 import ops
    g = _gen(1)
    conv = torch.nn.Conv2d(3, 32, 3, stride=2, bias=False)
    with torch.no_grad():
        conv.weight.copy_(torch.randn(32, 3, 3, 3, generator=g) * 0.3)
    bn = _bn(32, g)
    x = torch.randn(N, Cimg, H, W, generator=g)
    ref = _swish64(_bn64(bn, F.conv2d(F.pad(x[:, :3].double(), (0, 1, 0, 1)), conv.weight.double(), stride=2)))
    w, b = ops.pack_stem_conv(conv, bn)
    y = ops.stem_conv_swish(x.cuda(), w.cuda(), b.cuda())
    assert (y.N, y.H, y.W, y.C) == (N, ref.shape[2], ref.shape[3], 32)
    _close(_nhwc(y), ref, 1e-5, "stem")


@pytest.mark.parametrize("k,stride", [(3, 1), (3, 2), (5, 1), (5, 2)])
@pytest.mark.parametrize("N,C,H,W", [(1, 16, 23, 37), (5, 24, 9, 14), (1, 40, 32, 31), (5, 96, 17, 12), (1, 144, 8, 22),
                                     (1, 672, 5, 7), (5, 1152, 3, 4), (2, 32, 64, 88)])
def test_dwconv_bn_swish_and_se_sums(k, stride, N, C, H, W):
    from heal_b200 import ops
    from heal_b200.models.sub_modules.efficientnet_b0 import same_pads
    g = _gen(2 + k + stride)
    conv = torch.nn.Conv2d(C, C, k, stride=stride, groups=C, bias=False)
    with torch.no_grad():
        conv.weight.copy_(torch.randn(C, 1, k, k, generator=g) / k)
    bn = _bn(C, g)
    x = torch.randn(N, C, H, W, generator=g)
    p = (k // 2, k // 2) if stride == 1 else {3: (0, 1), 5: (1, 2)}[k]          # the static "same" pads, written out
    assert same_pads(k, stride) == p
    ref = _swish64(_bn64(bn, F.conv2d(F.pad(x.double(), (p[0], p[1], p[0], p[1])), conv.weight.double(), stride=stride, groups=C)))
    w, b = ops.pack_dwconv(conv, bn)
    xa = ops.to_act(x.cuda())
    y, sums = ops.dwconv_bn_swish(xa, w.cuda(), b.cuda(), k, stride, (p[0], p[1], p[0], p[1]))
    assert (y.N, y.C, y.H, y.W) == tuple(ref.shape)
    _close(_nhwc(y), ref, 1e-5, f"dwconv k{k} s{stride} C{C}")
    rs = ref.sum((2, 3))
    err = (sums.double().cpu() - rs).abs().max().item()
    assert err <= 1e-5 * max(ref.abs().sum((2, 3)).max().item(), 1.0), err
    y2, sums2 = ops.dwconv_bn_swish(xa, w.cuda(), b.cuda(), k, stride, (p[0], p[1], p[0], p[1]))
    assert torch.equal(sums, sums2) and torch.equal(y.t, y2.t)                    # no atomics: the same bits on every run


@pytest.mark.parametrize("N,C,Csq,hw", [(1, 32, 8, 100), (5, 96, 4, 7), (2, 144, 6, 1), (1, 672, 28, 176), (5, 1152, 48, 12)])
def test_se_gate(N, C, Csq, hw):
    from heal_b200 import ops
    g = _gen(5)
    red, exp = torch.nn.Conv2d(C, Csq, 1), torch.nn.Conv2d(Csq, C, 1)
    with torch.no_grad():
        red.weight.copy_(torch.randn(Csq, C, 1, 1, generator=g) / C ** 0.5)
        red.bias.copy_(torch.randn(Csq, generator=g))
        exp.weight.copy_(torch.randn(C, Csq, 1, 1, generator=g))
        exp.bias.copy_(torch.randn(C, generator=g) * 2)
    sums = torch.randn(N, C, generator=g) * hw
    m = sums.double() / hw
    s = _swish64(m @ red.weight.double()[:, :, 0, 0].t() + red.bias.double())
    ref = torch.sigmoid(s @ exp.weight.double()[:, :, 0, 0].t() + exp.bias.double())
    gate = ops.se_gate(sums.cuda(), hw, *[t.cuda() for t in ops.pack_se(red, exp)])
    assert (gate.double().cpu() - ref).abs().max().item() <= 2e-6
    assert ref.std().item() > 0.1                                                    # the gates are spread, not all ~0.5


@pytest.mark.parametrize("N,H,W,Cin,Cout", [(1, 9, 13, 16, 96), (5, 5, 7, 96, 24), (1, 8, 11, 144, 40), (5, 3, 5, 40, 240),
                                            (1, 4, 6, 672, 112), (1, 2, 3, 1152, 320), (5, 2, 3, 192, 1152), (2, 16, 24, 32, 16)])
@pytest.mark.parametrize("gate,res,act", [(False, False, True), (True, False, False), (True, True, False), (False, True, True)])
def test_pwconv(N, H, W, Cin, Cout, gate, res, act):
    from heal_b200 import ops
    g = _gen(7)
    conv = torch.nn.Conv2d(Cin, Cout, 1, bias=False)
    with torch.no_grad():
        conv.weight.copy_(torch.randn(Cout, Cin, 1, 1, generator=g) / Cin ** 0.5)
    bn = _bn(Cout, g)
    x = torch.randn(N, Cin, H, W, generator=g)
    gt = torch.rand(N, Cin, generator=g) if gate else None
    r = torch.randn(N, Cout, H, W, generator=g) if res else None
    xin = x.double() * gt.double()[:, :, None, None] if gate else x.double()
    ref = _bn64(bn, F.conv2d(xin, conv.weight.double()))
    if act:
        ref = _swish64(ref)
    if res:
        ref = ref + r.double()
    w, b = ops.pack_pwconv(conv, bn)
    y = ops.pwconv(ops.to_act(x.cuda()), w.cuda(), b.cuda(), gate=gt.cuda() if gate else None, swish=act,
                   residual=ops.to_act(r.cuda()) if res else None)
    _close(_nhwc(y), ref, 2e-5, f"pwconv {Cin}->{Cout}")


@pytest.mark.parametrize("N,H1,W1,C1,C2", [(1, 2, 3, 320, 112), (5, 4, 6, 512, 40), (2, 1, 5, 64, 8), (1, 3, 1, 8, 64), (1, 1, 1, 4, 4)])
@pytest.mark.parametrize("fmt", ["f32", "split", "bf16"])
def test_upsample2x_concat(N, H1, W1, C1, C2, fmt):
    from heal_b200 import ops
    g = _gen(9)
    x1 = torch.randn(N, C1, H1, W1, generator=g)
    x2 = torch.randn(N, C2, 2 * H1, 2 * W1, generator=g)
    up = F.interpolate(x1.double(), scale_factor=2, mode="bilinear", align_corners=True)
    ref = torch.cat([x2.double(), up], 1)
    def act(x):                       # a freshly allocated (N,H,W,C) buffer: canonical strides also when H or W is 1
        return ops.Act(torch.empty((x.shape[0], x.shape[2], x.shape[3], x.shape[1]), device="cuda").copy_(x.permute(0, 2, 3, 1)), "f32")
    x1a = ops.convert(act(x1), fmt)                                                  # up2 reads the conv engine's output format
    y = ops.upsample2x_concat(x1a, act(x2), fmt)
    Cp = (C1 + C2 + 63) // 64 * 64
    assert (y.fmt, y.N, y.H, y.W, y.C) == (fmt, N, 2 * H1, 2 * W1, Cp)
    got = _nhwc(ops.convert(y, "f32"))
    assert (got[:, C1 + C2:] == 0).all()                                             # the tail the padded conv weights ignore
    _close(got[:, :C1 + C2], ref, {"f32": 1e-5, "split": 3e-5, "bf16": 1.2e-2}[fmt], f"upsample2x_concat {fmt}")


def _cam_encode(ds, g):
    from heal_b200.models.heter_encoders import CamEncode
    m = CamEncode(g["D"], g["C"], ds, g["ddiscr"], "LID", False, False).eval()
    m.load_state_dict(oe.state_dict_of(g["cases"][ds]["shapes"]), strict=True)
    return m


@pytest.mark.parametrize("ds", [8, 16])
def test_cam_encode_heads_nhwc_vs_torch_path_and_reference_golden(golden_dir, ds):
    from heal_b200 import engine
    g = golden.load(os.path.join(golden_dir, "efficientnet_trunk.pt"))
    case = g["cases"][ds]
    m = _cam_encode(ds, g)
    x = oe.trunk_images()
    with torch.no_grad():
        dl, ft = copy.deepcopy(m).double().heads(x.double())                        # the torch path in float64
    ref = torch.cat([dl, ft], 1).permute(0, 2, 3, 1)
    gref = torch.cat([case["depth_logits"], case["feat"]], 1).permute(0, 2, 3, 1).double()
    assert (ref - gref).abs().max().item() <= 1e-5 * max(gref.abs().max().item(), 1.0)
    m = m.cuda()
    for prec, tol in (("tc32", 1e-3), ("fp32", 1e-5), ("bf16", 2.5e-2)):
        engine.set_precision(prec)
        with torch.no_grad():
            y4 = m.heads_nhwc(x.cuda()).t
            y3 = m.heads_nhwc(x[:, :3].contiguous().cuda()).t
        assert torch.equal(y3, y4)                                                   # the fourth image plane is never read
        assert y4.shape == ref.shape
        for name, r in (("torch path (float64)", ref), ("reference golden", gref)):
            err = (y4.cpu().double() - r).abs().max().item()
            scale = max(r.abs().max().item(), 1.0)
            print(f"CamEncode ds={ds} {prec} vs {name}: max|ref|={scale:.3f} err={err:.3e}")
            assert err <= (tol if r is ref else max(tol, 5e-5)) * scale, (prec, name, err, scale)   # the golden itself is fp32
    with torch.no_grad():                                                            # endpoints of the kernels vs the reference's
        engine.set_precision("fp32")
        r3, r4, r5 = m.trunk.endpoints_nhwc(x.cuda())
    for a, k in ((r3, "reduction_3"), (r4, "reduction_4"), (r5, "reduction_5")):
        if k in case["endpoints"]:
            _close(_nhwc(a), case["endpoints"][k].double(), 1e-5, k)


def _lss(g):
    from heal_b200.models.heter_encoders import LiftSplatShoot
    m = LiftSplatShoot(copy.deepcopy(g["cfg"])).eval()
    m.load_state_dict(oe.state_dict_of(g["shapes"]), strict=True)
    return m.cuda()


def _cuda(d):
    return {k: (v.cuda() if torch.is_tensor(v) else _cuda(v) if isinstance(v, dict) else v) for k, v in d.items()}


@pytest.mark.parametrize("prec,tol", [("fp32", 1e-3), ("tc32", 1e-3), ("bf16", 2.5e-2)])
def test_lift_splat_shoot_efficientnet_vs_reference_golden(golden_dir, prec, tol):
    """A frustum point within rounding of a cell boundary may land next door on another device (tests/test_gpu_lss.py), which
    moves one point's mass between two cells: all but a bounded handful of cells must meet the tolerance."""
    from heal_b200 import engine
    engine.set_precision(prec)
    g = golden.load(os.path.join(golden_dir, "lss_efficientnet_small.pt"))
    m = _lss(g)
    with torch.no_grad():
        bev = m({"inputs_m2": _cuda(oe.cam_inputs())}, "m2").cpu()
    assert bev.shape == g["bev"].shape
    scale = max(g["bev"].abs().max().item(), 1.0)
    bad = ((bev - g["bev"]).abs() > tol * scale).any(1).float().mean().item()
    print(f"LSS-EfficientNet {prec}: cells beyond tolerance {bad:.2e}, max err {(bev - g['bev']).abs().max().item():.3e}")
    assert bad < 2e-3


@pytest.mark.parametrize("prec,tol", [("fp32", 1e-3), ("tc32", 1e-3), ("bf16", 2.5e-2)])
def test_heter_pyramid_collab_with_efficientnet_camera_agent_vs_reference_golden(golden_dir, prec, tol):
    from heal_b200 import engine
    from heal_b200.models.heter_pyramid_collab import HeterPyramidCollab
    engine.set_precision(prec)
    g = golden.load(os.path.join(golden_dir, "heter_pyramid_collab_effnet_small.pt"))
    m = HeterPyramidCollab(copy.deepcopy(g["args"])).eval()
    m.load_state_dict(oe.state_dict_of(g["shapes"]), strict=True)
    m = m.cuda()
    data = _cuda(oe.collab_data())
    data["record_len"] = torch.tensor([3])
    with torch.no_grad():
        out = m(data)
    for k in ("cls_preds", "reg_preds", "dir_preds"):
        ref = g["out"][k]
        err = (out[k].cpu() - ref).abs().max().item()
        scale = max(ref.abs().max().item(), 1.0)
        print(f"collab [m1, m2 EfficientNet, m1] {prec}/{k}: max|ref|={scale:.3f} err={err:.3e}")
        assert out[k].shape == ref.shape and err < tol * scale, (k, err, scale)


def test_lss_efficientnet_captures_into_a_cuda_graph(golden_dir):
    g = golden.load(os.path.join(golden_dir, "lss_efficientnet_small.pt"))
    m = _lss(g)
    dd = {"inputs_m2": _cuda(oe.cam_inputs())}
    with torch.no_grad():
        eager = m(dd, "m2").clone()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            m(dd, "m2")
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, capture_error_mode="thread_local"):
            out = m(dd, "m2")
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, eager)
        dd["inputs_m2"]["imgs"].normal_()          # the graph reads the static input buffers: new images, same graph
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, m(dd, "m2")) and not torch.equal(out, eager)
