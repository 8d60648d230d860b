"""Feature compression (`compressor:`) on the GPU: heal_conv3x3_narrow_tc against float64 F.conv2d, the NaiveCompressor mirror
against goldens of the reference module at every ratio, HeterPyramidCollab and HeterModelBaseline with a compressor against
goldens of the reference models (also built through the reference's own create_model), CUDA-graph replay of a compressed frame."""
import copy
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import efficientnet as oe, golden, make_golden, make_golden_compressor as mgc, procedural, ref_shim

pytestmark = pytest.mark.gpu

BF16_TOL = 2.5e-2
PREC = [("fp32", 1e-3), ("tc32", 1e-3), ("bf16", BF16_TOL)]
HEADS = ("cls_preds", "reg_preds", "dir_preds")
SINGLE = ("cls_preds_single", "reg_preds_single", "dir_preds_single")


@pytest.fixture(autouse=True)
def _restore_precision():
    from heal_b200 import engine
    old = engine.PRECISION
    yield
    engine.set_precision(old)


def _tol_check(got, ref, tol, name):
    err = (got.float().cpu() - ref.float().cpu()).abs().max().item()
    scale = max(ref.abs().max().item(), 1.0)
    print(f"{name}: max|ref|={scale:.3f} max_abs_err={err:.3e} err/scale={err / scale:.3e}")
    assert got.shape == ref.shape and err < tol * scale, (name, err, scale)


def _to_cuda(d):
    if torch.is_tensor(d):
        return d.cuda()
    if isinstance(d, dict):
        return {k: _to_cuda(v) for k, v in d.items()}
    return d


# ---------------------------------------------------------------------------------------------------------------------------
# kernel
# ---------------------------------------------------------------------------------------------------------------------------
def _conv_bn(cin, cout, seed):
    g = torch.Generator().manual_seed(seed)
    conv = nn.Conv2d(cin, cout, 3, padding=1)
    bn = nn.BatchNorm2d(cout, eps=1e-3)
    with torch.no_grad():
        conv.weight.copy_(torch.randn(conv.weight.shape, generator=g) / np.sqrt(9 * cin))
        conv.bias.copy_(0.1 * torch.randn(cout, generator=g))
        bn.weight.copy_(1 + 0.2 * torch.randn(cout, generator=g))
        bn.bias.copy_(0.1 * torch.randn(cout, generator=g))
        bn.running_mean.copy_(0.1 * torch.randn(cout, generator=g))
        bn.running_var.copy_(0.5 + torch.rand(cout, generator=g))
    return conv.eval(), bn.eval()


def _ref64(x, conv, bn, relu):
    """float64 F.conv2d + eval BatchNorm (+ ReLU) on the device, NCHW."""
    w, b = conv.weight.double().cuda(), conv.bias.double().cuda()
    y = F.conv2d(x.double(), w, b, padding=1)
    s = bn.weight.double().cuda() / torch.sqrt(bn.running_var.double().cuda() + bn.eps)
    y = (y - bn.running_mean.double().cuda()[:, None, None]) * s[:, None, None] + bn.bias.double().cuda()[:, None, None]
    return torch.relu(y) if relu else y


SHAPES = [(1, 1, 1), (3, 37, 53), (5, 256, 256)]


@pytest.mark.parametrize("N,H,W", SHAPES)
@pytest.mark.parametrize("cout", [64, 256])
@pytest.mark.parametrize("cin", [1, 2, 3, 4, 8, 16, 21, 32, 48, 63])
def test_narrow_kernel_vs_float64(cin, cout, N, H, W):
    """ReLU on and off; the input is a channel slice of a wider map, at an even offset (channel pairs loaded as one word) and at an
    odd one (channel by channel): tc32 from split and from f32 input, to split and to a channel slice of a wide f32 map; bf16
    from bf16 input to bf16."""
    from heal_b200 import ops
    conv, bn = _conv_bn(cin, cout, seed=cin * 1000 + cout)
    g = torch.Generator().manual_seed(cin + 7 * cout + H)
    wide = torch.randn((N, H, W, (cin + 10) // 2 * 2), generator=g).cuda()
    split, bf16 = ops.convert(ops.Act(wide, "f32"), "split"), ops.convert(ops.Act(wide, "f32"), "bf16")
    for relu in (False, True):
        pc = ops.pack_conv3x3_narrow(conv, bn, relu).to("cuda")
        for off in (4, 5):
            ref = _ref64(wide[..., off:off + cin].permute(0, 3, 1, 2), conv, bn, relu).float()
            what = f"cin={cin} cout={cout} relu={relu} offset={off} {N}x{H}x{W}"
            xs = ops.Act(split.t[..., off:off + cin], "split")
            y = ops.conv3x3_narrow_tc(xs, pc, planes=2, out_fmt="split")
            _tol_check(ops.act_to_nchw(y), ref, 1e-3, f"tc32 split->split {what}")
            y = ops.conv3x3_narrow_tc(ops.Act(wide[..., off:off + cin], "f32"), pc, planes=2, out_fmt="split")
            _tol_check(ops.act_to_nchw(y), ref, 1e-3, f"tc32 f32->split {what}")
            o32 = torch.full((N, H, W, cout + 6), 7.0, device="cuda")
            ops.conv3x3_narrow_tc(xs, pc, planes=2, out=ops.Act(o32[..., 2:2 + cout], "f32"))
            _tol_check(o32[..., 2:2 + cout].permute(0, 3, 1, 2), ref, 1e-3, f"tc32 split->f32 slice {what}")
            assert torch.all(o32[..., :2] == 7.0) and torch.all(o32[..., 2 + cout:] == 7.0)
            yb = ops.conv3x3_narrow_tc(ops.Act(bf16.t[..., off:off + cin], "bf16"), pc, planes=1, out_fmt="bf16")
            _tol_check(ops.act_to_nchw(yb), ref, BF16_TOL, f"bf16 {what}")


def test_narrow_kernel_refuses_bad_arguments():
    from heal_b200 import ops
    from heal_b200._lib import lib
    conv, bn = _conv_bn(8, 64, seed=1)
    pc = ops.pack_conv3x3_narrow(conv, bn, True).to("cuda")
    x = ops.act_zeros(1, 8, 8, 8, "split", "cuda")
    out = ops.act_zeros(1, 8, 8, 64, "f32", "cuda")
    stream = ops._stream()
    call = lambda cin, cout, planes, o: lib.heal_conv3x3_narrow_tc(x.view(), 1, 8, 8, cin, ops._p(pc.w), ops._p(pc.bias),
                                                                  cout, planes, 1, o.view(), stream)
    assert call(8, 64, 2, out) == 0
    assert call(64, 64, 2, out) == -1           # Cin > 63
    assert call(8, 72, 2, out) == -1            # Cout not a multiple of 16
    assert call(8, 64, 3, out) == -1            # planes
    odd = ops.Act(torch.zeros((1, 8, 8, 65), device="cuda")[..., 1:65], "f32")
    assert lib.heal_conv3x3_narrow_tc(x.view(), 1, 8, 8, 8, ops._p(pc.w), ops._p(pc.bias), 64, 2, 1, odd.view(), stream) == -4
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------------------------
# module
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("prec,tol", PREC)
@pytest.mark.parametrize("C", [64, 256])
def test_naive_compressor_vs_reference_golden(golden_dir, C, prec, tol):
    from heal_b200 import engine
    from heal_b200.models.sub_modules.naive_compress import NaiveCompressor
    engine.set_precision(prec)
    g = golden.load(os.path.join(golden_dir, f"compressor_c{C}.pt"))
    x = mgc.module_x(C).cuda()
    assert sorted(g["ratios"]) == list(mgc.RATIOS)
    for r, gr in g["ratios"].items():
        m = NaiveCompressor(C, r).eval()
        m.load_state_dict(procedural.make_state_dict(gr["shapes"]), strict=True)
        with torch.no_grad():
            y = m.cuda()(x)
        _tol_check(y[:, ::g["step"]], gr["out_s"], tol, f"NaiveCompressor({C}, {r}) {prec}")


# ---------------------------------------------------------------------------------------------------------------------------
# models
# ---------------------------------------------------------------------------------------------------------------------------
def _collab(g, sd_of=procedural.make_state_dict):
    from heal_b200.models.heter_pyramid_collab import HeterPyramidCollab
    m = HeterPyramidCollab(copy.deepcopy(g["args"])).eval()
    m.load_state_dict(sd_of(g["shapes"]), strict=True)
    return m.cuda()


def _small_data():
    data = _to_cuda(make_golden.small_scene())
    data["record_len"] = torch.tensor([3])
    return data


@pytest.mark.parametrize("prec,tol", PREC)
def test_heter_pyramid_collab_compressed_vs_reference_golden(golden_dir, prec, tol):
    from heal_b200 import engine
    engine.set_precision(prec)
    g = golden.load(os.path.join(golden_dir, "heter_pyramid_collab_compress_small.pt"))
    m = _collab(g)
    assert m.compress and m.compressor.decoder[0].in_channels == 8
    with torch.no_grad():
        out = m(_small_data())
    for k in HEADS:
        _tol_check(out[k], g["out"][k], tol, f"collab compress {prec}/{k}")


@pytest.mark.parametrize("prec,tol", PREC)
def test_heter_pyramid_collab_hetero_compressed_vs_reference_golden(golden_dir, prec, tol):
    """agents [m1 PointPillar, m2 LSS-EfficientNet, m1]: the compressor runs on the torch.cat assembly of both modalities."""
    from heal_b200 import engine
    engine.set_precision(prec)
    g = golden.load(os.path.join(golden_dir, "heter_pyramid_collab_hetero_compress_small.pt"))
    m = _collab(g, oe.state_dict_of)
    data = _to_cuda(oe.collab_data())
    data["record_len"] = torch.tensor([3])
    with torch.no_grad():
        out = m(data)
    for k in HEADS:
        _tol_check(out[k], g["out"][k], tol, f"collab hetero compress {prec}/{k}")


@pytest.mark.parametrize("prec,tol", PREC)
def test_heter_model_baseline_compressed_vs_reference_golden(golden_dir, prec, tol):
    from heal_b200 import engine
    from heal_b200.models.heter_model_baseline import HeterModelBaseline
    engine.set_precision(prec)
    g = golden.load(os.path.join(golden_dir, "heter_model_baseline_compress_small.pt"))
    m = HeterModelBaseline(copy.deepcopy(g["args"])).eval()
    m.load_state_dict(procedural.make_state_dict(g["shapes"]), strict=True)
    assert m.compress and m.compressor.decoder[0].in_channels == 8
    with torch.no_grad():
        out = m.cuda()(_small_data())
    for k in HEADS + SINGLE:
        _tol_check(out[k], g["out"][k], tol, f"baseline compress {prec}/{k}")


@pytest.fixture
def _isolate_opencood_modules():
    before = {k: v for k, v in sys.modules.items() if k.startswith("opencood")}
    yield
    for k in [k for k in sys.modules if k.startswith("opencood")]:
        del sys.modules[k]
    sys.modules.update(before)


@pytest.mark.parametrize("core,name", [("heter_pyramid_collab", "heter_pyramid_collab_compress_small"),
                                       ("heter_model_baseline", "heter_model_baseline_compress_small")])
def test_reference_create_model_builds_the_compressed_mirror(golden_dir, core, name, _isolate_opencood_modules):
    """After install_into_opencood(), the reference's train_utils.create_model builds the mirror with its compressor, a
    reference-keyed checkpoint loads strictly and the frame matches the golden."""
    if not ref_shim.available():
        pytest.skip("oracle/_ref not built")
    from unittest.mock import MagicMock
    from heal_b200 import engine, install
    from heal_b200.models.sub_modules.naive_compress import NaiveCompressor
    ref_shim.install()
    sys.modules.setdefault("opencood.utils.box_overlaps", MagicMock())
    done = install.install_into_opencood()
    assert f"opencood.models.{core}" in done
    from opencood.tools.train_utils import create_model
    g = golden.load(os.path.join(golden_dir, name + ".pt"))
    model = create_model({"model": {"core_method": core, "args": copy.deepcopy(g["args"])}})
    assert type(model).__module__ == f"heal_b200.models.{core}"
    assert isinstance(model.compressor, NaiveCompressor)
    res = model.load_state_dict(procedural.make_state_dict(g["shapes"]), strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    engine.set_precision("tc32")
    with torch.no_grad():
        out = model.cuda().eval()(_small_data())
    for k in g["out"]:
        _tol_check(out[k], g["out"][k], 1e-3, f"create_model/{core}/{k}")


def test_compressed_collab_frame_graph_replay_equals_eager(golden_dir):
    from heal_b200 import engine, synth
    from heal_b200.graph import FrameGraph
    engine.set_precision("tc32")
    g = golden.load(os.path.join(golden_dir, "heter_pyramid_collab_compress_small.pt"))
    m = _collab(g)
    sc = synth.scene(3, n_agents=3, rings=16, azimuth=256)
    pts = torch.from_numpy(np.concatenate(sc["points"]))
    offs = torch.from_numpy(np.concatenate([[0], np.cumsum([p.shape[0] for p in sc["points"]])]).astype(np.int32))
    pw = torch.from_numpy(sc["pairwise_t_matrix"])
    with torch.no_grad():
        eager = m({"inputs_m1": {"points": pts.cuda(), "agent_offsets": offs.cuda()}, "agent_modality_list": ["m1"] * 3,
                   "record_len": torch.tensor([3]), "pairwise_t_matrix": pw.cuda()})
        eager = {k: eager[k].cpu().clone() for k in HEADS}
    fg = FrameGraph(m, 3, pts.shape[0] + 64, tuple(pw.shape))
    fg.load(pts, offs, pw)
    out = fg.replay()
    for k in HEADS:
        assert torch.equal(out[k].cpu(), eager[k]), k
