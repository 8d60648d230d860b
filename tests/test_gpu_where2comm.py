"""Where2commFusion and Who2comFusion on the GPU: heal_ego_mha against a float64 restatement in this file, the mirror modules
and HeterModelBaseline against goldens of the reference's own modules, a full-size 5-agent frame against the oracle, CUDA-graph
replay, and the reference's own create_model building the mirrors."""
import copy
import ctypes
import os
import sys

import pytest
import torch

from oracle import golden, make_golden_where2comm as mg, nets, procedural, ref_shim, where2comm as w2c

pytestmark = pytest.mark.gpu

BF16_TOL = 2.5e-2
PREC = [("fp32", 1e-3), ("tc32", 1e-3), ("bf16", BF16_TOL)]
C = 256

# heal_ego_mha against the float64 restatement below, on the kernel's own (stored) inputs: every step runs in fp32, so the error
# is a few fp32 roundings of the sampled k / v, the 32-term q.k sums and the softmax.  Bound: |err| <= MHA_TOL * max(max|ref|, 1)
# for logits of order 1, and MHA_TOL_LARGE for logits of order 100 (a logit error of eps * |s| moves every weight by as much).
MHA_TOL = 1e-5
MHA_TOL_LARGE = 2e-4


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
    assert err < tol * scale, (name, err, scale)


def _sample64(x, theta, H, W):
    """grid_sample of the maps x (n, H, W, K) float64 at the kernel's sample points: affine_grid in fp64, the grid cast to fp32,
    unnormalised in fp32 (align_corners=False), bilinear weights in fp32; the taps are then summed in float64."""
    n = x.shape[0]
    ow = torch.arange(W, dtype=torch.float64)
    oh = torch.arange(H, dtype=torch.float64)
    xb = ((2 * ow + 1) / W - 1).view(1, 1, W)
    yb = ((2 * oh + 1) / H - 1).view(1, H, 1)
    th = theta.double().cpu()
    gx = (th[:, 0, 0].view(n, 1, 1) * xb + th[:, 0, 1].view(n, 1, 1) * yb + th[:, 0, 2].view(n, 1, 1)).float()
    gy = (th[:, 1, 0].view(n, 1, 1) * xb + th[:, 1, 1].view(n, 1, 1) * yb + th[:, 1, 2].view(n, 1, 1)).float()
    ix, iy = ((gx + 1) * W - 1) / 2, ((gy + 1) * H - 1) / 2
    fx, fy = torch.floor(ix), torch.floor(iy)
    out = torch.zeros(n, H, W, x.shape[-1], dtype=torch.float64)
    flat = x.reshape(n, H * W, -1)
    for dy, dx in ((0, 0), (0, 1), (1, 0), (1, 1)):
        xi, yi = fx + dx, fy + dy
        w = ((ix - fx) if dx else (fx + 1 - ix)) * ((iy - fy) if dy else (fy + 1 - iy))
        ok = (xi >= 0) & (xi < W) & (yi >= 0) & (yi < H)
        idx = (yi.clamp(0, H - 1) * W + xi.clamp(0, W - 1)).long().view(n, H * W, 1).expand(n, H * W, x.shape[-1])
        out += torch.gather(flat, 1, idx).view(n, H, W, -1) * (w.double() * ok.double()).unsqueeze(-1)
    return out


def ego_mha_ref(q, kv, bias, theta, rl, heads=8):
    """float64: q (B,H,W,C), kv (N,H,W,2C) unwarped and bias-free, bias (2C) -> (B,H,W,C) per pixel and head
    sum_j softmax_j((q * dh^-0.5) . k_j) v_j with k | v = sample(kv_j, theta_j) + bias."""
    B, H, W, Cq = q.shape
    dh = Cq // heads
    scale = float(torch.tensor((1.0 / dh) ** 0.5, dtype=torch.float32))
    out, s0 = [], 0
    for b, n in enumerate(rl):
        kvs = _sample64(kv[s0:s0 + n].double(), theta[s0:s0 + n], H, W) + bias.double()
        qs = (q[b].double() * scale).view(H, W, heads, dh)
        k, v = kvs[..., :Cq].view(n, H, W, heads, dh), kvs[..., Cq:].view(n, H, W, heads, dh)
        a = torch.softmax(torch.einsum("hwmd,nhwmd->hwmn", qs, k), -1)
        out.append(torch.einsum("hwmn,nhwmd->hwmd", a, v).reshape(H, W, Cq))
        s0 += n
    return torch.stack(out)


def _thetas(n, g, out_of_view=None, subpixel=False):
    a = torch.rand(n, generator=g, dtype=torch.float64) * 6.3
    th = torch.zeros(n, 2, 3, dtype=torch.float64)
    th[:, 0, 0], th[:, 0, 1], th[:, 1, 0], th[:, 1, 1] = a.cos(), -a.sin() * 0.6, a.sin() / 0.6, a.cos()
    th[:, :, 2] = (torch.rand(n, 2, generator=g, dtype=torch.float64) - 0.5) * 1.2
    th[0] = torch.tensor([[1.0, 0, 0], [0, 1.0, 0]], dtype=torch.float64)
    if subpixel and n > 1:
        th[1] = torch.tensor([[1.0, 0, 0.013], [0, 1.0, -0.027]], dtype=torch.float64)
    if out_of_view is not None:
        th[out_of_view, :, 2] = torch.tensor([3.5, -2.7], dtype=torch.float64)
    return th


def _inputs(rl, H, W, fmt, seed, q_scale=1.0, out_of_view=None, kv_wide=False):
    from heal_b200 import ops
    g = torch.Generator().manual_seed(seed)
    B, N = len(rl), sum(rl)
    q = torch.randn(B, H, W, C, generator=g) * q_scale
    kvc = 2 * C + (96 if kv_wide else 0)
    kv = torch.randn(N, H, W, kvc, generator=g)
    bias = torch.randn(2 * C, generator=g) * 0.5
    th = torch.cat([_thetas(n, g, out_of_view if n > 1 else None, subpixel=True) for n in rl])
    qa = ops.convert(ops.Act(q.cuda(), "f32"), fmt)
    kva = ops.convert(ops.Act(kv.cuda(), "f32"), fmt)
    return qa, kva, bias.cuda(), th.cuda()


def _run_and_check(rl, H, W, fmt, seed, tol, **kw):
    from heal_b200 import ops
    off = 64 if kw.get("kv_wide") else 0
    qa, kva, bias, th = _inputs(rl, H, W, fmt, seed, **kw)
    out = ops.ego_mha(qa, kva, bias, th, rl, kv_coffset=off, out_fmt="f32")
    kv64 = ops.convert(kva, "f32").t.double().cpu()[..., off:off + 2 * C]
    ref = ego_mha_ref(ops.convert(qa, "f32").t.double().cpu(), kv64, bias.cpu(), th.cpu(), rl)
    _tol_check(out.t, ref, tol, f"ego_mha rl={rl} {H}x{W} {fmt}")
    return qa, kva, bias, th, out, off


@pytest.mark.parametrize("fmt", ["f32", "bf16", "split"])
@pytest.mark.parametrize("rl", [[1], [2], [5], [8], [1, 5, 8]])
def test_ego_mha_vs_float64(rl, fmt):
    """Agent counts 1, 2, 5, 8 and three scenes [1, 5, 8]; 13 x 19 pixels (not a multiple of the 4-pixel block); an agent of
    every multi-agent scene entirely out of view (its k = b_k, v = b_v) and one shifted by a fraction of a pixel."""
    _run_and_check(rl, 13, 19, fmt, 11 + len(rl) + sum(rl), MHA_TOL, out_of_view=-1)


def test_ego_mha_single_agent_is_its_value():
    """n = 1: the softmax weight is exactly 1, so the output is the ego's sampled v + b_v."""
    from heal_b200 import ops
    qa, kva, bias, th = _inputs([1], 16, 24, "f32", 3)
    out = ops.ego_mha(qa, kva, bias, th, [1]).t.double().cpu()[0]
    v = _sample64(kva.t.double().cpu()[:, ..., C:], th.cpu(), 16, 24)[0] + bias.cpu().double()[C:]
    assert (out - v).abs().max().item() <= 1e-5 * max(v.abs().max().item(), 1.0)


def test_ego_mha_large_logits():
    _run_and_check([5, 3], 17, 23, "f32", 21, MHA_TOL_LARGE, q_scale=40.0, out_of_view=2)


@pytest.mark.parametrize("fmt", ["f32", "split"])
def test_ego_mha_kv_channel_view(fmt):
    """kv read from channels 64 .. 64 + 2C of a wider map."""
    _run_and_check([3, 2], 12, 20, fmt, 31, MHA_TOL, kv_wide=True)


@pytest.mark.parametrize("fmt", ["bf16", "split"])
def test_ego_mha_output_formats_round_the_fp32_result(fmt):
    from heal_b200 import ops
    qa, kva, bias, th = _inputs([4, 2], 11, 18, fmt, 41)
    f32 = ops.ego_mha(qa, kva, bias, th, [4, 2], out_fmt="f32").t
    got = ops.ego_mha(qa, kva, bias, th, [4, 2], out_fmt=fmt).t
    assert torch.equal(got[0], f32.bfloat16())
    if fmt == "split":
        assert torch.equal(got[1], (f32 - got[0].float()).bfloat16())


def test_ego_mha_is_bit_identical_across_runs():
    from heal_b200 import ops
    qa, kva, bias, th = _inputs([5, 8, 1], 32, 48, "split", 51, out_of_view=1)
    a = ops.ego_mha(qa, kva, bias, th, [5, 8, 1]).t.clone()
    b = ops.ego_mha(qa, kva, bias, th, [5, 8, 1]).t
    assert torch.equal(a, b)


def test_ego_mha_rejected_arguments_launch_nothing():
    from heal_b200 import ops
    from heal_b200._lib import lib
    qa, kva, bias, th = _inputs([2, 3], 8, 8, "f32", 61)
    out = ops.act_zeros(2, 8, 8, C, "f32", qa.device)
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    ok = (ctypes.c_int * 2)(2, 3)

    def call(counts=ok, B=2, Cc=C, heads=8, bias_p=bias.data_ptr(), q=qa, kv=kva):
        return lib.heal_ego_mha(q.view(), kv.view(), ctypes.c_void_p(bias_p), ctypes.c_void_p(th.data_ptr()), counts, B, 8, 8,
                                Cc, heads, out.view(), s)

    torch.cuda.synchronize()
    before = lib.heal_launch_count()
    assert call(counts=(ctypes.c_int * 2)(2, 9)) == -1                 # HEAL_ERR_ARG: 9 agents, after a valid first scene
    assert call(counts=(ctypes.c_int * 2)(0, 3)) == -1
    assert call(Cc=128) == -4 and call(heads=4) == -4                   # HEAL_ERR_UNSUPPORTED
    assert call(bias_p=bias.data_ptr() + 4) == -4                       # bias not 16-byte aligned
    assert call(kv=ops.Act(kva.t[..., 2:], "f32")) == -4                # misaligned channel view
    assert call(bias_p=0) == -1 and call(B=-1) == -1
    torch.cuda.synchronize()
    assert lib.heal_launch_count() == before
    assert out.t.abs().max().item() == 0.0
    assert call() == 0 and lib.heal_launch_count() == before + 1


def _module(method, shapes):
    from heal_b200.models.fuse_modules.fusion_in_one import Where2commFusion, Who2comFusion
    m = (Where2commFusion if method == "where2comm" else Who2comFusion)(C).eval()
    m.load_state_dict(procedural.make_state_dict(shapes), strict=True)
    return m.cuda()


@pytest.mark.parametrize("method", mg.METHODS)
@pytest.mark.parametrize("prec,tol", PREC)
def test_fusion_mirror_vs_reference_golden(golden_dir, method, prec, tol):
    from heal_b200 import engine
    engine.set_precision(prec)
    g = w2c.load_module_golden(golden_dir)
    m = _module(method, g[method]["shapes"])
    with torch.no_grad():
        out = m(g["x"].cuda(), g["record_len"], g["affine"].cuda())
        assert out.shape == (3, C, 24, 40)
        _tol_check(out[:, ::16], g[method]["out_s"], tol, f"{method}/{prec}")
        # mixed-modality input arrives as f32 whatever the precision
        from heal_b200 import ops
        nhwc = m.forward_nhwc(ops.to_act(g["x"].cuda()), g["record_len"], g["affine"].cuda())
        _tol_check(ops.act_to_nchw(nhwc)[:, ::16], g[method]["out_s"], tol, f"{method}/{prec}/nhwc")


def _to_cuda(d):
    if torch.is_tensor(d):
        return d.cuda()
    if isinstance(d, dict):
        return {k: _to_cuda(v) for k, v in d.items()}
    return d


def _baseline_run(model, g):
    data = _to_cuda(g["data"])
    data["record_len"] = g["data"]["record_len"]
    with torch.no_grad():
        return model(data)


@pytest.mark.parametrize("method", mg.METHODS)
@pytest.mark.parametrize("prec,tol", PREC)
def test_heter_model_baseline_vs_reference_golden(golden_dir, method, prec, tol):
    from heal_b200 import engine
    from heal_b200.models.heter_model_baseline import HeterModelBaseline
    engine.set_precision(prec)
    g = golden.load(os.path.join(golden_dir, f"heter_model_baseline_{method}_small.pt"))
    m = HeterModelBaseline(copy.deepcopy(g["args"])).eval()
    m.load_state_dict(procedural.make_state_dict(g["shapes"]), strict=True)
    out = _baseline_run(m.cuda(), g)
    for k in ("cls_preds", "reg_preds", "dir_preds"):
        _tol_check(out[k], g["out"][k], tol, f"{method}/{prec}/{k}")


def _fullsize_scene(n=5):
    """A lidar baseline frame: 5 agents on the +-102.4 m range within 40 m of the ego, any heading."""
    from heal_b200 import synth
    g = torch.Generator().manual_seed(19)
    poses = [[0, 0, 0, 0, 0, 0]] + [[float(v) for v in ((torch.rand(2, generator=g) - 0.5) * 80).tolist()] +
                                    [0, 0, float(torch.rand(1, generator=g) * 360 - 180), 0] for _ in range(n - 1)]
    pw = torch.from_numpy(synth.pairwise_t_matrix(poses, n)[None])
    return torch.tensor([n]), nets.normalize_pairwise_tfm(pw, 204.8, 204.8, 1)


@pytest.mark.parametrize("method", mg.METHODS)
def test_fullsize_fusion_vs_oracle_on_gpu(method):
    """The fusion stage of a 5-agent frame at 256 x 256 x 256 in tc32 against the literal oracle run by PyTorch on the GPU in
    fp32 with TF32 off."""
    from heal_b200 import engine
    engine.set_precision("tc32")
    rl, aff = _fullsize_scene()
    x = torch.randn(5, C, 256, 256, generator=torch.Generator().manual_seed(23)).cuda()
    aff = aff.cuda()
    shapes = _fresh_shapes(method)
    m = _module(method, shapes)
    sd = {"f." + k: v.cuda() for k, v in procedural.make_state_dict(shapes).items()}
    tf32 = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.no_grad():
            ref = w2c.FUSIONS[method](x, sd, "f", rl, aff)
            got = m(x, rl, aff)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32
    _tol_check(got, ref, 1e-3, f"fullsize/{method}")


def _fresh_shapes(method):
    from heal_b200.models.fuse_modules.fusion_in_one import Where2commFusion, Who2comFusion
    return procedural.shapes_of((Where2commFusion if method == "where2comm" else Who2comFusion)(C))


@pytest.mark.parametrize("method", mg.METHODS)
def test_graph_replay_equals_eager(golden_dir, method):
    from heal_b200 import engine, ops
    engine.set_precision("tc32")
    g = w2c.load_module_golden(golden_dir)
    m = _module(method, g[method]["shapes"])
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


@pytest.fixture
def _isolate_opencood_modules():
    before = {k: v for k, v in sys.modules.items() if k.startswith(("opencood", "shapely", "turtle"))}
    yield
    for k in [k for k in sys.modules if k.startswith(("opencood", "shapely", "turtle"))]:
        del sys.modules[k]
    sys.modules.update(before)


@pytest.mark.parametrize("method", mg.METHODS)
def test_reference_create_model_builds_and_runs_the_mirror(golden_dir, method, _isolate_opencood_modules):
    """After install_into_opencood(), the reference's own train_utils.create_model builds the HeterModelBaseline mirror with
    the new fusion method from a `model:` block, a reference-keyed checkpoint loads strictly, and the frame matches the golden."""
    if not ref_shim.available():
        pytest.skip("oracle/_ref not built")
    import types
    from unittest.mock import MagicMock
    from heal_b200 import engine
    from heal_b200.models.fuse_modules.fusion_in_one import Where2commFusion, Who2comFusion
    from oracle import postprocess as opp
    sg = types.ModuleType("shapely.geometry")
    sg.Polygon, sg.Point, sg.MultiPoint = opp.QuadPolygon, MagicMock(), MagicMock()
    sh = types.ModuleType("shapely")
    sh.geometry = sg
    sys.modules["shapely"], sys.modules["shapely.geometry"] = sh, sg
    sys.modules.setdefault("opencood.utils.box_overlaps", MagicMock())
    mg.install_reference()
    from heal_b200 import install
    done = install.install_into_opencood()
    assert "opencood.models.heter_model_baseline" in done
    from opencood.tools.train_utils import create_model
    g = golden.load(os.path.join(golden_dir, f"heter_model_baseline_{method}_small.pt"))
    model = create_model({"model": {"core_method": "heter_model_baseline", "args": copy.deepcopy(g["args"])}})
    assert type(model).__module__ == "heal_b200.models.heter_model_baseline"
    assert isinstance(model.fusion_net, Where2commFusion if method == "where2comm" else Who2comFusion)
    res = model.load_state_dict(procedural.make_state_dict(g["shapes"]), strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    engine.set_precision("tc32")
    out = _baseline_run(model.cuda().eval(), g)
    for k in ("cls_preds", "reg_preds", "dir_preds"):
        _tol_check(out[k], g["out"][k], 1e-3, f"create_model/{method}/{k}")
