"""V2X-ViT on the GPU: heal_window_attention, heal_cav_attention, heal_split_attn and heal_sttf_resample against float64 torch
(or the reference's warp_affine chain), V2XViTFusion and HeterModelBaseline against goldens of the reference's own modules, the
full-size fusion stages against the oracle on the GPU, padded-slot independence and CUDA-graph replay."""
import copy
import os

import pytest
import torch
import torch.nn.functional as F

from oracle import golden, procedural, v2xvit as vx

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
    print(f"{name}: max|ref|={ref.abs().max().item():.3f} max_abs_err={err:.3e} rel={err / scale:.3e}"
          + (f" (1e-2 met: {err < 1e-2 * scale})" if tol == BF16_TOL else ""))
    assert err < tol * scale, (name, err, scale)


def _window_ref(qkv, coff, heads, dh, ws, bias):
    """float64 window attention over an NHWC qkv map: 'b (x w1) (y w2) (m c) -> b m (x y) (w1 w2) c', softmax(q k^T + bias) v."""
    N, H, W, _ = qkv.shape
    inner = heads * dh
    t = qkv[..., coff:coff + 3 * inner].reshape(N, H // ws, ws, W // ws, ws, 3, heads, dh).permute(5, 0, 1, 3, 6, 2, 4, 7)
    t = t.reshape(3, N, H // ws, W // ws, heads, ws * ws, dh)
    o = (t[0] @ t[1].transpose(-1, -2) + bias).softmax(-1) @ t[2]
    return o.reshape(N, H // ws, W // ws, heads, ws, ws, dh).permute(0, 1, 4, 2, 5, 3, 6).reshape(N, H, W, inner)


@pytest.mark.parametrize("fmt", ["f32", "split", "bf16"])
@pytest.mark.parametrize("ws", [4, 8, 16])
@pytest.mark.parametrize("dh", [16, 32, 64])
def test_window_attention_vs_float64(fmt, ws, dh):
    """3 images (not a multiple of any tile), 3 heads, q/k/v read from channel 6 of a wider map, the heads written to channels
    4 .. of a wider output whose other channels must stay untouched."""
    from heal_b200 import ops
    heads, N, H, W = 3, 3, 16, 32
    inner = heads * dh
    g = torch.Generator().manual_seed(41 + ws + dh)
    qkv = torch.randn(N, H, W, 3 * inner + 12, generator=g)
    qkv[..., 6:6 + inner] *= dh ** -0.5
    bias = torch.randn(ws * ws, ws * ws, generator=g)
    a = ops.convert(ops.Act(qkv.cuda(), "f32"), fmt)
    qin = ops.convert(a, "f32").t.cpu().double()
    ref = _window_ref(qin, 6, heads, dh, ws, bias.double())
    out = ops.Act(torch.full((N, H, W, inner + 10), 7.0, device="cuda"), "f32")
    ops.window_attention(a, heads, dh, ws, bias.cuda(), qkv_coffset=6, out=out, out_coffset=4)
    o = out.t.cpu()
    assert (o[..., :4] == 7.0).all() and (o[..., 4 + inner:] == 7.0).all()
    err = (o[..., 4:4 + inner].double() - ref).abs().max().item()
    tol = 2e-2 if fmt == "bf16" else 1e-4
    print(f"window_attention {fmt} w={ws} dh={dh}: {err:.3e}")
    assert err <= tol * max(1.0, ref.abs().max().item())


def test_window_attention_rejects_unsupported_shapes():
    from heal_b200 import ops
    qkv = ops.act_empty(1, 16, 16, 3 * 96, "f32", "cuda")
    with pytest.raises(RuntimeError):
        ops.window_attention(qkv, 1, 96, 4, torch.zeros(16, 16, device="cuda"))        # dim_head 96
    with pytest.raises(RuntimeError):
        ops.window_attention(qkv, 3, 32, 32, torch.zeros(1024, 1024, device="cuda"))   # window 32


def test_window_attention_rejects_a_misaligned_bias():
    from heal_b200 import ops
    qkv = ops.act_empty(1, 16, 16, 3 * 64, "f32", "cuda")
    storage = torch.zeros(16 * 16 + 1, device="cuda")
    with pytest.raises(RuntimeError):
        ops.window_attention(qkv, 2, 32, 4, storage[1:].view(16, 16))     # 4-byte offset: not float2-aligned


def test_cav_attention_checks_every_count_before_launching():
    """65 scenes need two launches; a bad count in the second must leave the output as it was."""
    from heal_b200 import ops
    rl = [1] * 64 + [0]
    qkv = ops.Act(torch.ones(64, 2, 2, 3 * 32, device="cuda"), "f32")
    out = ops.Act(torch.full((64, 2, 2, 32), 7.0, device="cuda"), "f32")
    with pytest.raises((RuntimeError, AssertionError)):
        ops.cav_attention(qkv, rl, False, out=out)
    assert (out.t == 7.0).all()


def _cav_ref(qkv, rl, ego_only):
    """float64 per-pixel attention over each scene's agents; images egos first, then each scene's others."""
    B, C = len(rl), qkv.shape[-1] // 3
    heads = C // 32
    N, H, W = qkv.shape[:3]
    other = B
    outs = torch.zeros(B if ego_only else N, H, W, C, dtype=qkv.dtype)
    for b, n in enumerate(rl):
        idx = [b] + list(range(other, other + n - 1))
        other += n - 1
        q = qkv[idx, ..., :C].reshape(n, H, W, heads, 32)
        k = qkv[idx, ..., C:2 * C].reshape(n, H, W, heads, 32)
        v = qkv[idx, ..., 2 * C:].reshape(n, H, W, heads, 32)
        s = torch.einsum("ihwmc,jhwmc->hwmij", q, k).softmax(-1)
        o = torch.einsum("hwmij,jhwmc->ihwmc", s, v).reshape(n, H, W, C)
        if ego_only:
            outs[b] = o[0]
        else:
            outs[idx] = o
    return outs


@pytest.mark.parametrize("fmt", ["f32", "split", "bf16"])
@pytest.mark.parametrize("ego_only", [False, True])
def test_cav_attention_vs_float64(fmt, ego_only):
    """Scenes of 1 .. 5 agents; a 5 x 7 map so the last block is partly empty."""
    from heal_b200 import ops
    rl, C, H, W = [1, 2, 3, 4, 5], 256, 5, 7
    g = torch.Generator().manual_seed(43)
    qkv = torch.randn(sum(rl), H, W, 3 * C, generator=g)
    qkv[..., :C] *= 32 ** -0.5
    a = ops.convert(ops.Act(qkv.cuda(), "f32"), fmt)
    qin = ops.convert(a, "f32").t.cpu().double()
    ref = _cav_ref(qin, rl, ego_only)
    out = ops.cav_attention(a, rl, ego_only, out_fmt="f32")
    err = (out.t.cpu().double() - ref).abs().max().item()
    print(f"cav_attention {fmt} ego_only={ego_only}: {err:.3e}")
    assert err <= 1e-5 * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize("fmt", ["f32", "split", "bf16"])
def test_split_attn_vs_float64(fmt):
    from heal_b200 import ops
    N, H, W, C = 3, 9, 13, 256
    g = torch.Generator().manual_seed(47)
    o = torch.randn(N, H, W, 3 * C, generator=g)
    x = torch.randn(N, H, W, C, generator=g)
    fc1 = torch.randn(C, C, generator=g) / 16
    fc2 = torch.randn(3 * C, C, generator=g) / 16
    lw, lb = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g) * 0.1
    oa = ops.convert(ops.Act(o.cuda(), "f32"), fmt)
    xa = ops.convert(ops.Act(x.cuda(), "f32"), fmt)
    oi, xi = ops.convert(oa, "f32").t.cpu().double(), ops.convert(xa, "f32").t.cpu().double()
    sw, mw, bw = oi[..., :C], oi[..., C:2 * C], oi[..., 2 * C:]
    gap = (sw + mw + bw).mean((1, 2))
    gt = F.relu(F.layer_norm(gap @ fc1.double().t(), (C,), lw.double(), lb.double(), 1e-5))
    gt = (gt @ fc2.double().t()).reshape(N, 3, C).softmax(1)
    ref = sw * gt[:, None, None, 0] + mw * gt[:, None, None, 1] + bw * gt[:, None, None, 2] + xi
    fc1_t, fc2_t = fc1.t().contiguous().cuda(), fc2.t().contiguous().cuda()
    out = ops.split_attn(oa, xa, fc1_t, lw.cuda(), lb.cuda(), 1e-5, fc2_t, out_fmt="f32")
    again = ops.split_attn(oa, xa, fc1_t, lw.cuda(), lb.cuda(), 1e-5, fc2_t, out_fmt="f32")
    assert torch.equal(out.t, again.t)
    err = (out.t.cpu().double() - ref).abs().max().item()
    print(f"split_attn {fmt}: {err:.3e}")
    assert err <= 1e-5 * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize("H,W", [(128, 128), (64, 128), (20, 36)])
def test_sttf_resample_vs_reference_warp_affine(H, W):
    """The STTF matrix of the identity correction and a rotated, shifted one, against the reference's warp_affine chain."""
    from heal_b200 import ops
    from heal_b200.models.sub_modules.v2xvit_basic import STTF
    g = torch.Generator().manual_seed(53)
    src = torch.randn(2, 64, H, W, generator=g)
    scm = torch.eye(4).expand(1, 3, 4, 4)
    M = vx.sttf_matrix(scm, H, W, 0.4, 4)                                   # (2, 2, 3)
    c, s = float(torch.cos(torch.tensor(0.3))), float(torch.sin(torch.tensor(0.3)))
    M[1] = torch.tensor([[c, -s, 2.5], [s, c, -1.25]])
    ref = vx.warp_affine(src, M, (H, W))
    theta = vx.warp_affine_matrix(M, (H, W), (H, W)).contiguous()
    assert torch.equal(theta[0], STTF({"voxel_size": [0.4, 0.4, 4], "downsample_rate": 4}).theta(H, W))
    out = ops.sttf_resample(ops.to_act(src.cuda()), theta.cuda(), out_fmt="f32")
    got = ops.act_to_nchw(out).cpu()
    err = (got - ref).abs().max().item()
    change = (ref[0] - src[0]).abs().max().item()
    err0 = (got[0] - ref[0]).abs().max().item()
    print(f"sttf_resample {H}x{W}: {err:.3e}; identity correction: change {change:.2e}, error {err0:.2e}")
    assert err <= 2e-5
    assert err0 <= max(1e-6, 0.1 * change)


def _loaded(args, shapes):
    from heal_b200.models.fuse_modules.fusion_in_one import V2XViTFusion
    m = V2XViTFusion(copy.deepcopy(args)).eval()
    m.load_state_dict(procedural.make_state_dict(shapes), strict=True)
    return m.cuda()


@pytest.mark.parametrize("case", ["c256", "l2"])
@pytest.mark.parametrize("prec,tol", PREC)
def test_v2xvit_vs_reference_golden(golden_dir, case, prec, tol):
    from heal_b200 import engine
    engine.set_precision(prec)
    g = vx.load_module_golden(golden_dir)[case]
    x, rl, _ = vx.case_inputs(case)
    m = _loaded(g["args"], g["shapes"])
    with torch.no_grad():
        out = m(x.cuda(), rl, g["affine"].cuda())
    _tol_check(out[:, ::g["stride"]], g["out_s"], tol, f"v2xvit/{case}/{prec}")


def _to_cuda(d):
    if torch.is_tensor(d):
        return d.cuda()
    if isinstance(d, dict):
        return {k: _to_cuda(v) for k, v in d.items()}
    return d


@pytest.mark.parametrize("prec,tol", PREC)
def test_heter_model_baseline_v2xvit_vs_reference_golden(golden_dir, prec, tol):
    from heal_b200 import engine
    from heal_b200.models.heter_model_baseline import HeterModelBaseline
    engine.set_precision(prec)
    g = golden.load(os.path.join(golden_dir, "heter_model_baseline_v2xvit_small.pt"))
    m = HeterModelBaseline(copy.deepcopy(g["args"])).eval()
    m.load_state_dict(procedural.make_state_dict(g["shapes"]), strict=True)
    m = m.cuda()
    data = _to_cuda(g["data"])
    data["record_len"] = g["data"]["record_len"]
    with torch.no_grad():
        out = m(data)
    for k in ("cls_preds", "reg_preds", "dir_preds"):
        _tol_check(out[k], g["out"][k], tol, f"v2xvit-model/{prec}/{k}")


def _fullsize_scene(n, L, H, W):
    """n agents within 40 m of the ego, any heading, on an H x W fusion map of 1.6 m cells, padded to L slots."""
    from heal_b200 import synth
    from oracle import nets
    g = torch.Generator().manual_seed(19)
    poses = [[0, 0, 0, 0, 0, 0]] + [[float(v) for v in ((torch.rand(2, generator=g) - 0.5) * 80).tolist()] +
                                    [0, 0, float(torch.rand(1, generator=g) * 360 - 180), 0] for _ in range(n - 1)]
    pw = torch.from_numpy(synth.pairwise_t_matrix(poses, L)[None])
    return torch.tensor([n]), nets.normalize_pairwise_tfm(pw, H * 0.8 * 2, W * 0.8 * 2, 1)


@pytest.mark.parametrize("name,n,L,H,W", [("lidar_v2xvit", 5, 5, 128, 128), ("dairv2x", 2, 2, 64, 128)])
def test_fullsize_v2xvit_vs_oracle_on_gpu(name, n, L, H, W):
    """The fusion stage of a lidar_v2xvit frame (5 agents, 256 x 128^2) and of a dairv2x config (max_cav 2, 256 x 64 x 128) in
    tc32 against the literal oracle run by PyTorch on the GPU in fp32 with TF32 off."""
    from heal_b200 import engine
    from heal_b200.models.fuse_modules.fusion_in_one import V2XViTFusion
    engine.set_precision("tc32")
    rl, aff = _fullsize_scene(n, L, H, W)
    args = vx.v2xvit_args()
    shapes = procedural.shapes_of(V2XViTFusion(copy.deepcopy(args)))
    m = _loaded(args, shapes)
    sd = procedural.make_state_dict(shapes)
    x = torch.randn(n, 256, H, W, generator=torch.Generator().manual_seed(23)).cuda()
    aff = aff.cuda()
    tf32 = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.no_grad():
            ref = vx.v2xvit_fusion(x, {"f." + k: v.cuda() for k, v in sd.items()}, "f", args, rl, aff)
            got = m(x, rl, aff)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32
    _tol_check(got, ref, 1e-3, f"fullsize/{name}")


def test_padded_slots_are_bit_identical(golden_dir):
    """A 3-agent scene in L = 5 and in L = 3 slots."""
    from heal_b200 import engine
    engine.set_precision("tc32")
    g = vx.load_module_golden(golden_dir)["c256"]
    m = _loaded(g["args"], g["shapes"])
    x = torch.randn(3, 256, 16, 32, generator=torch.Generator().manual_seed(5)).cuda()
    aff5 = g["affine"][:1].cuda()
    with torch.no_grad():
        y5 = m(x, torch.tensor([3]), aff5)
        y3 = m(x, torch.tensor([3]), aff5[:, :3, :3].contiguous())
    assert torch.equal(y5, y3)


def test_v2xvit_graph_replay_is_bit_identical(golden_dir):
    from heal_b200 import engine, ops
    engine.set_precision("tc32")
    g = vx.load_module_golden(golden_dir)["c256"]
    x, rl, _ = vx.case_inputs("c256")
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
        first = ops.act_to_nchw(out).clone()
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(first, eager) and torch.equal(ops.act_to_nchw(out), eager)
