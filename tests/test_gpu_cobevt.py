"""CoBEVT on the GPU: heal_swap_attention and heal_mean_layernorm against float64 torch, the CoBEVT module and
HeterModelBaseline against goldens of the reference's own modules, the full-size fusion stage against the oracle on the GPU, and
CUDA-graph replay."""
import copy
import os

import pytest
import torch
import torch.nn.functional as F

from oracle import cobevt as cb, golden, procedural

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


def _attention_ref(qkv, rl, L, w, grid, bias):
    """float64 windowed / grid attention over NHWC qkv with the reference's token order and key mask (-inf, then softmax)."""
    BL, H, W, C3 = qkv.shape
    C, h = C3 // 3, C3 // 96
    X, Y = H // w, W // w
    if grid:       # 'b m (w1 x) (w2 y) d -> b m x y w1 w2 d'
        t = qkv.reshape(BL, w, X, w, Y, C3).permute(0, 2, 4, 1, 3, 5)
    else:          # 'b m (x w1) (y w2) d -> b m x y w1 w2 d'
        t = qkv.reshape(BL, X, w, Y, w, C3).permute(0, 1, 3, 2, 4, 5)
    B = BL // L
    t = t.reshape(B, L, X, Y, w, w, C3).permute(0, 2, 3, 1, 4, 5, 6).reshape(B * X * Y, L * w * w, C3)
    q, k, v = (t[..., i * C:(i + 1) * C].reshape(t.shape[0], -1, h, 32).permute(0, 2, 1, 3) for i in range(3))
    s = q @ k.transpose(-1, -2) + bias.transpose(-1, -2)[None]
    keep = torch.zeros(B, L * w * w, dtype=torch.bool)
    for b, n in enumerate(rl):
        keep[b, :n * w * w] = True
    keep = keep[:, None, None, :].expand(B, X * Y, 1, L * w * w).reshape(B * X * Y, 1, 1, -1)
    o = s.masked_fill(~keep, -float("inf")).softmax(-1) @ v
    o = o.permute(0, 2, 1, 3).reshape(B, X, Y, L, w, w, C).permute(0, 3, 1, 2, 4, 5, 6)
    if grid:
        o = o.permute(0, 1, 4, 2, 5, 3, 6)        # b l w1 x w2 y d
    else:
        o = o.permute(0, 1, 2, 4, 3, 5, 6)        # b l x w1 y w2 d
    return o.reshape(BL, H, W, C)


@pytest.mark.parametrize("fmt", ["f32", "bf16", "split"])
@pytest.mark.parametrize("grid", [False, True])
@pytest.mark.parametrize("rl,L,C,H,W", [([1, 3, 5], 5, 64, 12, 20), ([2, 1], 2, 96, 28, 44), ([5], 5, 256, 8, 8)])
def test_swap_attention_kernel_vs_float64(fmt, grid, rl, L, C, H, W):
    """Ragged scenes (1, 3, 5 real agents of 5 slots; max_cav 2), both modes, every input format; 15, 77 and 4 windows are not
    multiples of any launch tile."""
    from heal_b200 import ops
    w, n = 4, L * 16
    g = torch.Generator().manual_seed(31)
    qkv = torch.randn(len(rl) * L, H, W, 3 * C, generator=g)
    qkv[..., :C] *= 32 ** -0.5                                 # q pre-scaled, as to_qkv delivers it
    bias = torch.randn(C // 32, n, n, generator=g)
    a = ops.convert(ops.Act(qkv.cuda(), "f32"), fmt)
    qin = ops.convert(a, "f32").t.cpu().double()              # what the kernel reads after the format's rounding
    ref = _attention_ref(qin, rl, L, w, grid, bias.double())
    out = ops.swap_attention(a, rl, L, w, grid, bias.cuda(), out_fmt="f32")
    err = (out.t.cpu().double() - ref).abs().max().item()
    print(f"swap_attention {fmt} grid={grid} L={L}: {err:.3e}")
    assert err <= 1e-4 * max(1.0, ref.abs().max().item())
    sp = ops.swap_attention(a, rl, L, w, grid, bias.cuda(), out_fmt="split")
    assert (ops.merge_bf16(sp.t).cpu() - out.t.cpu()).abs().max().item() <= 2 ** -16 * out.t.abs().max().item()


def test_swap_attention_rejects_unsupported_shapes():
    from heal_b200 import ops
    qkv = ops.act_empty(6, 10, 10, 3 * 64, "f32", "cuda")
    with pytest.raises(RuntimeError):
        ops.swap_attention(qkv, [3], 6, 5, False, torch.zeros(2, 150, 150, device="cuda"))     # 150 tokens > 128


@pytest.mark.parametrize("fmt", ["f32", "split", "bf16"])
@pytest.mark.parametrize("n_avg", [1, 5])
def test_mean_layernorm_vs_float64(fmt, n_avg):
    from heal_b200 import ops
    g = torch.Generator().manual_seed(37)
    x = torch.randn(2 * n_avg, 9, 13, 256, generator=g) * 3 + 1
    lw, lb = torch.rand(256, generator=g) + 0.5, torch.randn(256, generator=g) * 0.1
    a = ops.convert(ops.Act(x.cuda(), "f32"), fmt)
    xin = ops.convert(a, "f32").t.cpu().double()
    ref = F.layer_norm(xin.reshape(2, n_avg, 9, 13, 256).mean(1), (256,), lw.double(), lb.double(), 1e-5)
    out = ops.mean_layernorm(a, n_avg, lw.cuda(), lb.cuda(), 1e-5, out_fmt="f32")
    assert (out.t.cpu().double() - ref).abs().max().item() <= 1e-5


def _loaded(args, shapes):
    from heal_b200.models.fuse_modules.fusion_in_one import CoBEVT
    m = CoBEVT(copy.deepcopy(args)).eval()
    sd = m.state_dict()
    sd.update(procedural.make_state_dict(cb.float_shapes(shapes)))
    m.load_state_dict(sd, strict=True)
    return m.cuda()


@pytest.mark.parametrize("case", ["c64", "c256", "l2"])
@pytest.mark.parametrize("prec,tol", PREC)
def test_cobevt_vs_reference_golden(golden_dir, case, prec, tol):
    from heal_b200 import engine
    engine.set_precision(prec)
    g = cb.load_module_golden(golden_dir)[case]
    x, rl, _ = cb.case_inputs(case)
    m = _loaded(g["args"], g["shapes"])
    with torch.no_grad():
        out = m(x.cuda(), rl, g["affine"].cuda())
    _tol_check(out[:, ::g["stride"]], g["out_s"], tol, f"cobevt/{case}/{prec}")


def _to_cuda(d):
    if torch.is_tensor(d):
        return d.cuda()
    if isinstance(d, dict):
        return {k: _to_cuda(v) for k, v in d.items()}
    return d


@pytest.mark.parametrize("prec,tol", PREC)
def test_heter_model_baseline_cobevt_vs_reference_golden(golden_dir, prec, tol):
    from heal_b200 import engine
    from heal_b200.models.heter_model_baseline import HeterModelBaseline
    engine.set_precision(prec)
    g = golden.load(os.path.join(golden_dir, "heter_model_baseline_cobevt_small.pt"))
    m = HeterModelBaseline(copy.deepcopy(g["args"])).eval()
    sd = m.state_dict()
    sd.update(procedural.make_state_dict(cb.float_shapes(g["shapes"])))
    m.load_state_dict(sd, strict=True)
    m = m.cuda()
    data = _to_cuda(g["data"])
    data["record_len"] = g["data"]["record_len"]
    with torch.no_grad():
        out = m(data)
    for k in ("cls_preds", "reg_preds", "dir_preds"):
        _tol_check(out[k], g["out"][k], tol, f"cobevt-model/{prec}/{k}")


def _fullsize_scene(n, L, H, W):
    """n agents within 40 m of the ego, any heading, on an H x W fusion map of 1.6 m cells, padded to L slots."""
    from heal_b200 import synth
    from oracle import nets
    g = torch.Generator().manual_seed(19)
    poses = [[0, 0, 0, 0, 0, 0]] + [[float(v) for v in ((torch.rand(2, generator=g) - 0.5) * 80).tolist()] +
                                    [0, 0, float(torch.rand(1, generator=g) * 360 - 180), 0] for _ in range(n - 1)]
    pw = torch.from_numpy(synth.pairwise_t_matrix(poses, L)[None])
    return torch.tensor([n]), nets.normalize_pairwise_tfm(pw, H * 0.8 * 2, W * 0.8 * 2, 1)


@pytest.mark.parametrize("name,n,L,H,W", [("lidar_cobevt", 5, 5, 128, 128), ("dairv2x", 2, 2, 128, 64)])
def test_fullsize_cobevt_vs_oracle_on_gpu(name, n, L, H, W):
    """The fusion stage of a lidar_cobevt frame (5 agents, 256 x 128^2) and of the dairv2x config (max_cav 2, 256 x 128 x 64)
    in tc32 against the literal oracle run by PyTorch on the GPU in fp32 with TF32 off."""
    from heal_b200 import engine
    engine.set_precision("tc32")
    rl, aff = _fullsize_scene(n, L, H, W)
    from heal_b200.models.fuse_modules.fusion_in_one import CoBEVT
    args = cb.cobevt_args(256, 3, L)
    shapes = procedural.shapes_of(CoBEVT(copy.deepcopy(args)))
    m = _loaded(args, shapes)
    sd = procedural.make_state_dict(cb.float_shapes(shapes))
    x = torch.randn(n, 256, H, W, generator=torch.Generator().manual_seed(23)).cuda()
    aff = aff.cuda()
    tf32 = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.no_grad():
            ref = cb.cobevt_fusion(x, {"f." + k: v.cuda() for k, v in sd.items()}, "f", args, rl, aff)
            got = m(x, rl, aff)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32
    _tol_check(got, ref, 1e-3, f"fullsize/{name}")


def test_cobevt_graph_replay_is_bit_identical(golden_dir):
    from heal_b200 import engine, ops
    engine.set_precision("tc32")
    g = cb.load_module_golden(golden_dir)["c64"]
    x, rl, _ = cb.case_inputs("c64")
    m = _loaded(g["args"], g["shapes"])
    xa = ops.convert(ops.to_act(x.cuda()), "split")
    aff = g["affine"].cuda()
    with torch.no_grad():
        eager = ops.act_to_nchw(m.forward_nhwc(xa, rl, aff)).clone()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            m.forward_nhwc(xa, rl, aff)
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, capture_error_mode="thread_local"):
            out = m.forward_nhwc(xa, rl, aff)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(ops.act_to_nchw(out), eager)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two CUDA devices")
def test_cobevt_on_a_device_that_is_not_current(golden_dir):
    """The library launches on the current device, so every ops wrapper makes its inputs' device current: CoBEVT on cuda:1
    run with cuda:0 current gives the bits it gives with cuda:1 current."""
    from heal_b200 import engine
    engine.set_precision("tc32")
    g = cb.load_module_golden(golden_dir)["c64"]
    x, rl, _ = cb.case_inputs("c64")
    m = _loaded(g["args"], g["shapes"]).to("cuda:1")
    x1, aff1 = x.to("cuda:1"), g["affine"].to("cuda:1")
    outs = []
    for current in (1, 0):
        with torch.cuda.device(current), torch.no_grad():
            outs.append(m(x1, rl, aff1).cpu())
    assert torch.equal(outs[0], outs[1])
