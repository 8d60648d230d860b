"""MaxFusion (F-Cooper) and V2VNetFusion on the GPU: the new fusion kernels against grid_sample, the mirror modules and
HeterModelBaseline against goldens of the reference's own modules, full-size fusion shapes against the oracle on the GPU, and
CUDA-graph replay."""
import copy
import os

import pytest
import torch
import torch.nn.functional as F

from oracle import fusion_methods as fm, golden, make_golden_fusion_methods as mg, nets, procedural

pytestmark = pytest.mark.gpu

BF16_TOL = 2.5e-2
PREC = [("fp32", 1e-3), ("tc32", 1e-3), ("bf16", BF16_TOL)]


@pytest.fixture(autouse=True)
def _restore_precision():
    from heal_b200 import engine
    old = engine.PRECISION
    yield
    engine.set_precision(old)


def _tol_check(got, ref, tol, name):
    err = (got.float().cpu() - ref.float().cpu()).abs().max().item()
    scale = max(ref.abs().max().item(), 1.0)
    print(f"{name}: max|ref|={scale:.3f} max_abs_err={err:.3e}")
    assert err < tol * scale, (name, err, scale)


def _grid_sample(x, theta):
    """warp_affine_simple as the reference runs it: fp64 theta through affine_grid, grid cast to fp32, bilinear / zeros."""
    grid = F.affine_grid(theta.double(), list(x.shape), align_corners=False).to(x)
    return F.grid_sample(x, grid, align_corners=False)


def _thetas(n, seed, out_of_view=None):
    g = torch.Generator().manual_seed(seed)
    a = torch.rand(n, generator=g) * 6.3
    th = torch.zeros(n, 2, 3, dtype=torch.float64)
    th[:, 0, 0], th[:, 0, 1], th[:, 1, 0], th[:, 1, 1] = a.cos(), -a.sin() * 0.6, a.sin() / 0.6, a.cos()
    th[:, :, 2] = (torch.rand(n, 2, generator=g, dtype=torch.float64) - 0.5) * 1.2
    th[0] = torch.tensor([[1.0, 0, 0], [0, 1.0, 0]], dtype=torch.float64)
    if out_of_view is not None:
        th[out_of_view, :, 2] = torch.tensor([3.5, -2.7], dtype=torch.float64)      # the whole map lands outside the ego's view
    return th


@pytest.mark.parametrize("n", [1, 4])
def test_max_fuse_kernel_vs_grid_sample(n):
    from heal_b200 import ops
    g = torch.Generator().manual_seed(3)
    x = torch.randn(n, 64, 21, 37, generator=g)
    th = _thetas(n, 5, out_of_view=n - 1 if n > 1 else None)
    ref = _grid_sample(x, th).max(0)[0]
    out = ops.max_fuse(ops.to_act(x.cuda()), th.cuda())
    got = ops.act_to_nchw(out)[0].cpu()
    assert (got - ref).abs().max().item() <= 1e-6
    if n > 1:      # the out-of-view agent contributes zeros to the max
        assert (got >= 0).all()
    sp = ops.max_fuse(ops.to_act(x.cuda()), th.cuda(), out_fmt="split")
    merged = ops.merge_bf16(sp.t)[0].permute(2, 0, 1).cpu()
    assert ((merged - got).abs() <= got.abs() * 2 ** -16 + 1e-30).all()


def test_warp_affine_kernel_vs_grid_sample():
    from heal_b200 import ops
    g = torch.Generator().manual_seed(4)
    x = torch.randn(3, 32, 19, 26, generator=g)
    src = [2, 0, 0, 1, 2, 1]
    th = _thetas(len(src), 6, out_of_view=3)
    ref = torch.cat([_grid_sample(x[s:s + 1], th[k:k + 1]) for k, s in enumerate(src)])
    got = ops.act_to_nchw(ops.warp_affine(ops.to_act(x.cuda()), src, th.cuda())).cpu()
    assert (got - ref).abs().max().item() <= 1e-6
    assert got[3].abs().max().item() == 0.0
    sp = ops.warp_affine(ops.to_act(x.cuda()), src, th.cuda(), out_fmt="split")
    merged = ops.merge_bf16(sp.t).permute(0, 3, 1, 2).cpu()
    assert ((merged - got).abs() <= got.abs() * 2 ** -16 + 1e-30).all()
    # a channel slice of a wider buffer, one image
    wide = torch.randn(1, 19, 26, 48, device="cuda")
    sl = ops.Act(wide[..., 8:40], "f32")
    one = ops.act_to_nchw(ops.warp_affine(sl, [0], th[1:2].cuda())).cpu()
    assert (one - _grid_sample(wide[..., 8:40].permute(0, 3, 1, 2).cpu(), th[1:2])).abs().max().item() <= 1e-6


def _module_golden(golden_dir):
    return fm.load_module_golden(golden_dir)


@pytest.mark.parametrize("prec,tol", PREC)
def test_max_fusion_vs_reference_golden(golden_dir, prec, tol):
    from heal_b200 import engine
    from heal_b200.models.fuse_modules.fusion_in_one import MaxFusion
    engine.set_precision(prec)
    g = _module_golden(golden_dir)
    x = ops_in(g["x"], engine.act_fmt())
    out = MaxFusion().forward_nhwc(x, g["record_len"], g["affine"].cuda())
    from heal_b200 import ops
    _tol_check(ops.act_to_nchw(out)[:, ::2], g["max_s"], tol, f"max/{prec}")


def ops_in(x, fmt):
    from heal_b200 import ops
    return ops.convert(ops.to_act(x.cuda()), fmt)


@pytest.mark.parametrize("variant", ["avg_gru1", "max_gru1", "avg_gru0", "max_gru0"])
@pytest.mark.parametrize("prec,tol", PREC)
def test_v2vnet_fusion_vs_reference_golden(golden_dir, variant, prec, tol):
    from heal_b200 import engine
    from heal_b200.models.fuse_modules.fusion_in_one import V2VNetFusion
    engine.set_precision(prec)
    g = _module_golden(golden_dir)
    v = g["v2vnet"][variant]
    m = V2VNetFusion(copy.deepcopy(v["args"])).eval()
    m.load_state_dict(procedural.make_state_dict(v["shapes"]), strict=True)
    m = m.cuda()
    with torch.no_grad():
        out = m(g["x"].cuda(), g["record_len"], g["affine"].cuda())
    _tol_check(out[:, ::4], v["out_s"], tol, f"v2vnet/{variant}/{prec}")


def _to_cuda(d):
    if torch.is_tensor(d):
        return d.cuda()
    if isinstance(d, dict):
        return {k: _to_cuda(v) for k, v in d.items()}
    return d


@pytest.mark.parametrize("method", ["max", "v2vnet"])
@pytest.mark.parametrize("prec,tol", PREC)
def test_heter_model_baseline_vs_reference_golden(golden_dir, method, prec, tol):
    from heal_b200 import engine
    from heal_b200.models.heter_model_baseline import HeterModelBaseline
    engine.set_precision(prec)
    g = golden.load(os.path.join(golden_dir, f"heter_model_baseline_{method}_small.pt"))
    m = HeterModelBaseline(copy.deepcopy(g["args"])).eval()
    m.load_state_dict(procedural.make_state_dict(g["shapes"]), strict=True)
    m = m.cuda()
    data = _to_cuda(g["data"])
    data["record_len"] = g["data"]["record_len"]
    with torch.no_grad():
        out = m(data)
    for k in ("cls_preds", "reg_preds", "dir_preds"):
        _tol_check(out[k], g["out"][k], tol, f"{method}/{prec}/{k}")


def _fullsize_scene(n=5):
    """lidar_fcooper.yaml / lidar_v2vnet.yaml: 5 agents on the +-102.4 m range, within 40 m of the ego, any heading."""
    from heal_b200 import synth
    g = torch.Generator().manual_seed(19)
    poses = [[0, 0, 0, 0, 0, 0]] + [[float(v) for v in ((torch.rand(2, generator=g) - 0.5) * 80).tolist()] +
                                    [0, 0, float(torch.rand(1, generator=g) * 360 - 180), 0] for _ in range(n - 1)]
    pw = torch.from_numpy(synth.pairwise_t_matrix(poses, n)[None])
    return torch.tensor([n]), nets.normalize_pairwise_tfm(pw, 204.8, 204.8, 1)


@pytest.mark.parametrize("method,hw", [("max", 256), ("v2vnet", 128)])
def test_fullsize_fusion_vs_oracle_on_gpu(method, hw):
    """The fusion stage of a lidar_fcooper / lidar_v2vnet frame (5 agents, 256 channels; 256^2 and 128^2 maps) in tc32 against
    the literal oracle run by PyTorch on the GPU in fp32 with TF32 off."""
    from heal_b200 import engine
    from heal_b200.models.fuse_modules.fusion_in_one import MaxFusion, V2VNetFusion
    engine.set_precision("tc32")
    rl, aff = _fullsize_scene()
    x = torch.randn(5, 256, hw, hw, generator=torch.Generator().manual_seed(23)).cuda()
    aff = aff.cuda()
    tf32 = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.no_grad():
            if method == "max":
                ref = fm.max_fusion(x, rl, aff)
                got = MaxFusion()(x, rl, aff)
            else:
                args = mg.v2vnet_args(256, hw, hw)
                m = V2VNetFusion(copy.deepcopy(args)).eval()
                sd = procedural.make_state_dict(procedural.shapes_of(m))
                m.load_state_dict(sd, strict=True)
                m = m.cuda()
                ref = fm.v2vnet_fusion(x, {"f." + k: v.cuda() for k, v in sd.items()}, "f", args, rl, aff)
                got = m(x, rl, aff)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32
    _tol_check(got, ref, 1e-3, f"fullsize/{method}")


def test_v2vnet_graph_replay_is_bit_identical(golden_dir):
    from heal_b200 import engine, ops
    from heal_b200.models.fuse_modules.fusion_in_one import V2VNetFusion
    engine.set_precision("tc32")
    g = _module_golden(golden_dir)
    v = g["v2vnet"]["max_gru1"]
    m = V2VNetFusion(copy.deepcopy(v["args"])).eval()
    m.load_state_dict(procedural.make_state_dict(v["shapes"]), strict=True)
    m = m.cuda()
    x = ops.convert(ops.to_act(g["x"].cuda()), "split")
    aff = g["affine"].cuda()
    with torch.no_grad():
        eager = ops.act_to_nchw(m.forward_nhwc(x, g["record_len"], aff)).clone()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            m.forward_nhwc(x, g["record_len"], aff)
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, capture_error_mode="thread_local"):
            out = m.forward_nhwc(x, g["record_len"], aff)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(ops.act_to_nchw(out), eager)
