"""GPU parity tests of the individual sm_90a kernels against the CPU oracle (run with -m gpu on an H100).
Integer outputs are bit-exact; fp32 outputs are within 1e-3 (north_star tolerance), usually ~1e-5."""
import numpy as np
import pytest
import torch

from oracle import golden
import torch.nn.functional as F

from oracle import nets, voxelizer

pytestmark = pytest.mark.gpu

PP_RANGE = [-102.4, -102.4, -3, 102.4, 102.4, 1]
PP_VOXEL = [0.4, 0.4, 4]


def _cuda(x):
    return torch.from_numpy(x).cuda() if isinstance(x, np.ndarray) else x.cuda()


def _vox_case(clouds, rng_, vs, T, maxv):
    from heal_b200 import ops
    per_agent = [voxelizer.points_to_voxel_c(p, vs, rng_, T, maxv) for p in clouds]
    ref = voxelizer.collate(per_agent)
    offs = np.concatenate([[0], np.cumsum([p.shape[0] for p in clouds])]).astype(np.int32)
    pts = np.concatenate(clouds).astype(np.float32) if sum(p.shape[0] for p in clouds) else np.zeros((0, 4), np.float32)
    v, c, n, nv = ops.voxelize(_cuda(pts).contiguous(), _cuda(offs), rng_, vs, T, maxv)
    torch.cuda.synchronize()
    got = ops.trim_voxels(v, c, n, nv)
    assert nv.cpu().tolist()[1:] == [a[0].shape[0] for a in per_agent]
    assert np.array_equal(got["voxel_coords"].cpu().numpy(), ref["voxel_coords"])
    assert np.array_equal(got["voxel_num_points"].cpu().numpy(), ref["voxel_num_points"])
    assert np.array_equal(got["voxel_features"].cpu().numpy().view(np.uint32), ref["voxel_features"].view(np.uint32))
    return got, ref


def test_voxelize_bit_exact_scene():
    from heal_b200 import synth
    sc = synth.scene(3, n_agents=5)
    _vox_case(sc["points"], PP_RANGE, PP_VOXEL, 32, 70000)                      # PointPillars config
    _vox_case(sc["points"][:2], PP_RANGE, [0.1, 0.1, 0.1], 5, 70000)            # SECOND config (T=5)


def test_voxelize_edge_cases():
    rng = np.random.default_rng(0)
    dense = np.concatenate([rng.uniform(-1, 1, (4000, 3)), rng.uniform(0, 1, (4000, 1))], 1).astype(np.float32)
    spread = np.concatenate([rng.uniform(-110, 110, (6000, 2)), rng.uniform(-4, 2, (6000, 1)), rng.uniform(0, 1, (6000, 1))], 1).astype(np.float32)
    _vox_case([dense, spread], PP_RANGE, PP_VOXEL, 32, 70000)     # >32 and >>32 points per voxel, out-of-range points
    _vox_case([spread, dense], PP_RANGE, PP_VOXEL, 3, 50)         # max_voxels clamp per agent + tiny T
    _vox_case([spread[:1], dense[:0], spread[:7]], PP_RANGE, PP_VOXEL, 32, 70000)   # ragged: 1-point and empty agents
    on_edges = np.array([[-102.4, -102.4, -3, .1], [102.4, 0, 0, .2], [0, 102.39999, 0.99999, .3], [-102.40001, 0, 0, .4],
                         [0.4, 0.8, 1.0, .5], [0.39999998, 0.8000001, -3.0, .6]], dtype=np.float32)
    _vox_case([on_edges], PP_RANGE, PP_VOXEL, 32, 70000)


def test_mean_vfe():
    from heal_b200 import ops
    rng = np.random.default_rng(1)
    v = rng.normal(size=(1000, 5, 4)).astype(np.float32)
    n = rng.integers(0, 6, size=1000).astype(np.int32)
    for i in range(1000):
        v[i, n[i]:] = 0
    got = ops.mean_vfe(_cuda(v), _cuda(n)).cpu()
    ref = torch.from_numpy(v).sum(1) / torch.clamp_min(torch.from_numpy(n).view(-1, 1), 1.0).float()
    torch.testing.assert_close(got, ref, rtol=1e-6, atol=1e-6)


def test_pillar_vfe_scatter_vs_oracle():
    from heal_b200 import ops, synth
    from oracle import procedural
    sc = synth.scene(5, n_agents=2)
    per_agent = [voxelizer.points_to_voxel_c(p, PP_VOXEL, PP_RANGE, 32, 70000) for p in sc["points"]]
    col = {k: torch.from_numpy(v) for k, v in voxelizer.collate(per_agent).items()}
    shapes = {"vfe.pfn_layers.0.linear.weight": (64, 10), "vfe.pfn_layers.0.norm.weight": (64,),
              "vfe.pfn_layers.0.norm.bias": (64,), "vfe.pfn_layers.0.norm.running_mean": (64,),
              "vfe.pfn_layers.0.norm.running_var": (64,)}
    sd = procedural.make_state_dict(shapes)
    ref_pf = nets.pillar_vfe(sd, "vfe", col["voxel_features"], col["voxel_num_points"], col["voxel_coords"], PP_VOXEL, PP_RANGE)
    ref_canvas = nets.scatter(ref_pf, col["voxel_coords"], 512, 512)
    w, b = ops.fold_linear_bn(sd["vfe.pfn_layers.0.linear.weight"], sd["vfe.pfn_layers.0.norm.weight"],
                              sd["vfe.pfn_layers.0.norm.bias"], sd["vfe.pfn_layers.0.norm.running_mean"],
                              sd["vfe.pfn_layers.0.norm.running_var"], 1e-3)
    pf, canvas = ops.pillar_vfe_scatter(col["voxel_features"].cuda(), col["voxel_num_points"].cuda(), col["voxel_coords"].cuda(),
                                        w.cuda(), b.cuda(), PP_VOXEL, PP_RANGE, 512, 512, 2, want_pillar_features=True)
    torch.testing.assert_close(pf.cpu(), ref_pf, rtol=1e-4, atol=1e-4)
    cv = ops.act_to_nchw(canvas)
    assert cv.shape == (2, 64, 512, 512)
    torch.testing.assert_close(cv.cpu().contiguous(), ref_canvas, rtol=1e-4, atol=1e-4)
    _, canvas_s = ops.pillar_vfe_scatter(col["voxel_features"].cuda(), col["voxel_num_points"].cuda(), col["voxel_coords"].cuda(),
                                         w.cuda(), b.cuda(), PP_VOXEL, PP_RANGE, 512, 512, 2, canvas_fmt="split")
    torch.testing.assert_close(ops.act_to_nchw(canvas_s).cpu().contiguous(), ref_canvas, rtol=2e-4, atol=2e-4)


CONV_CASES = [
    # (N, Cin, H, W, Cout, k, stride, pad, groups, bias, bn, relu, residual)
    (2, 64, 40, 56, 64, 3, 1, 1, 1, False, True, True, True),
    (1, 64, 41, 57, 64, 3, 2, 1, 1, False, True, True, False),
    (2, 64, 32, 32, 128, 1, 1, 0, 1, False, True, True, False),
    (1, 64, 32, 32, 128, 1, 2, 0, 1, False, True, False, False),
    (1, 384, 24, 24, 256, 3, 1, 1, 1, True, False, True, False),
    (1, 256, 16, 16, 20, 1, 1, 0, 1, True, False, False, False),
    (1, 64, 20, 20, 1, 1, 1, 0, 1, True, False, False, False),
    (2, 128, 24, 40, 128, 3, 1, 1, 32, False, True, True, False),
    (1, 256, 24, 40, 256, 3, 2, 1, 32, False, True, True, False),
    (1, 512, 16, 24, 512, 3, 1, 1, 32, False, True, True, False),
    (1, 512, 17, 23, 512, 3, 2, 1, 32, False, True, True, False),
    (1, 12, 9, 11, 36, 3, 1, 1, 1, True, False, False, False),
]


@pytest.mark.parametrize("case", CONV_CASES)
def test_conv2d_f32_vs_torch(case):
    from heal_b200 import ops
    N, Cin, H, W, Cout, k, s, p, g, bias, bn, relu, res = case
    gen = torch.Generator().manual_seed(hash(case) & 0xFFFF)
    conv = torch.nn.Conv2d(Cin, Cout, k, stride=s, padding=p, groups=g, bias=bias)
    bnm = torch.nn.BatchNorm2d(Cout, eps=1e-3) if bn else None
    with torch.no_grad():
        conv.weight.copy_(torch.randn(conv.weight.shape, generator=gen) * (1.0 / (Cin // g * k * k)) ** 0.5)
        if bias:
            conv.bias.copy_(torch.randn(Cout, generator=gen) * 0.1)
        if bn:
            bnm.weight.copy_(torch.rand(Cout, generator=gen) + 0.5)
            bnm.bias.copy_(torch.randn(Cout, generator=gen) * 0.1)
            bnm.running_mean.copy_(torch.randn(Cout, generator=gen) * 0.1)
            bnm.running_var.copy_(torch.rand(Cout, generator=gen) + 0.5)
            bnm.eval()
    x = torch.randn(N, Cin, H, W, generator=gen)
    with torch.no_grad():
        y = conv(x)
        if bn:
            y = bnm(y)
        r = torch.randn(y.shape, generator=gen) if res else None
        if res:
            y = y + r
        if relu:
            y = F.relu(y)
    pc = ops.pack_conv(conv, bnm, relu).to("cuda")
    out = ops.conv2d_simt(ops.to_act(x.cuda()), pc, residual=ops.to_act(r.cuda()) if res else None)
    torch.testing.assert_close(ops.act_to_nchw(out).cpu().contiguous(), y, rtol=1e-4, atol=1e-4)
    # same kernel with split-bf16 storage on both sides (fp32 math, 16-bit-mantissa storage)
    outs = ops.conv2d_simt(ops.convert(ops.to_act(x.cuda()), "split"), pc,
                           residual=ops.convert(ops.to_act(r.cuda()), "split") if res else None, out_fmt="split")
    torch.testing.assert_close(ops.act_to_nchw(outs).cpu().contiguous(), y, rtol=2e-4, atol=2e-4)


@pytest.mark.parametrize("up", [1, 2, 4])
def test_deconv_concat_slice(up):
    from heal_b200 import ops
    gen = torch.Generator().manual_seed(up)
    de = torch.nn.ConvTranspose2d(128, 128, up, stride=up, bias=False)
    bnm = torch.nn.BatchNorm2d(128, eps=1e-3).eval()
    with torch.no_grad():
        de.weight.copy_(torch.randn(de.weight.shape, generator=gen) * 0.1)
        bnm.running_mean.copy_(torch.randn(128, generator=gen) * 0.1)
        bnm.running_var.copy_(torch.rand(128, generator=gen) + 0.5)
    x = torch.randn(2, 128, 12, 20, generator=gen)
    with torch.no_grad():
        y = F.relu(bnm(de(x)))
    pc = ops.pack_deconv(de, bnm, True).to("cuda")
    buf = torch.full((2, 12 * up, 20 * up, 384), -7.0, device="cuda")
    ops.conv2d_simt(ops.to_act(x.cuda()), pc, out=ops.Act(buf, "f32"), out_coffset=128)
    torch.testing.assert_close(buf[..., 128:256].permute(0, 3, 1, 2).cpu().contiguous(), y, rtol=1e-4, atol=1e-4)
    assert torch.all(buf[..., :128] == -7.0) and torch.all(buf[..., 256:] == -7.0)


def _poses_affine(n, H_m, W_m, seed):
    from heal_b200 import synth
    rng = np.random.default_rng(seed)
    poses = [[0, 0, 0, 0, 0, 0]] + [[rng.uniform(-0.3 * W_m, 0.3 * W_m), rng.uniform(-0.3 * H_m, 0.3 * H_m), 0, 0,
                                     rng.uniform(-180, 180), 0] for _ in range(n - 1)]
    pw = torch.from_numpy(synth.pairwise_t_matrix(poses, 5)[None])
    return nets.normalize_pairwise_tfm(pw, H_m, W_m, 1)


@pytest.mark.parametrize("n,C,H,W,align", [(5, 64, 64, 96, False), (3, 128, 33, 47, False), (2, 256, 16, 16, True), (1, 64, 8, 8, False)])
def test_pyramid_fuse_level_vs_oracle(n, C, H, W, align):
    from heal_b200 import ops
    gen = torch.Generator().manual_seed(n * 100 + C)
    x = torch.randn(n, C, H, W, generator=gen)
    occ = torch.randn(n, 1, H, W, generator=gen) * 2
    aff = _poses_affine(n, 0.4 * H, 0.4 * W, seed=C)
    score = torch.sigmoid(occ) + 1e-4
    ref = nets.weighted_fuse(x, score, torch.tensor([n]), aff, align)[0]
    out = ops.pyramid_fuse_level(ops.to_act(x.cuda()), occ.view(n, H, W).cuda().contiguous(), aff[0, 0, :n].cuda(), align)
    torch.testing.assert_close(ops.act_to_nchw(out)[0].cpu().contiguous(), ref, rtol=1e-4, atol=1e-4)
    outs = ops.pyramid_fuse_level(ops.convert(ops.to_act(x.cuda()), "split"), occ.view(n, H, W).cuda().contiguous(),
                                  aff[0, 0, :n].cuda(), align)
    assert outs.fmt == "split"
    torch.testing.assert_close(ops.act_to_nchw(outs)[0].cpu().contiguous(), ref, rtol=2e-4, atol=2e-4)


def test_pyramid_fuse_crop_mask_and_all_masked():
    from heal_b200 import ops
    gen = torch.Generator().manual_seed(5)
    n, C, H, W = 3, 64, 32, 32
    x = torch.randn(n, C, H, W, generator=gen)
    occ = torch.randn(n, 1, H, W, generator=gen)
    aff = _poses_affine(n, 0.4 * H, 0.4 * W, seed=9)
    win = torch.tensor([[0, H, 0, W], [6, 26, 6, 26], [10, 22, 10, 22]], dtype=torch.int32)
    score = torch.sigmoid(occ) + 1e-4
    mask = torch.zeros_like(score)
    for j in range(n):
        mask[j, :, win[j, 0]:win[j, 1], win[j, 2]:win[j, 3]] = 1
    ref = nets.weighted_fuse(x, score * mask, torch.tensor([n]), aff, False)[0]
    out = ops.pyramid_fuse_level(ops.to_act(x.cuda()), occ.view(n, H, W).cuda().contiguous(), aff[0, 0, :n].cuda(), False,
                                 crop_windows=win.cuda())
    torch.testing.assert_close(ops.act_to_nchw(out)[0].cpu().contiguous(), ref, rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("n,C,H,W", [(5, 256, 32, 48), (3, 128, 24, 40), (1, 384, 8, 8)])
def test_att_fuse_vs_oracle(n, C, H, W):
    from heal_b200 import ops
    gen = torch.Generator().manual_seed(n + C)
    x = torch.randn(n, C, H, W, generator=gen)
    aff = _poses_affine(n, 0.4 * H, 0.4 * W, seed=n)
    ref = nets.att_fusion(x, torch.tensor([n]), aff)[0]
    out = ops.att_fuse(ops.to_act(x.cuda()), aff[0, 0, :n].cuda())
    torch.testing.assert_close(ops.act_to_nchw(out)[0].cpu().contiguous(), ref, rtol=1e-4, atol=1e-4)


def test_warp_att_golden(golden_dir):
    """AttFusion output of the UNMODIFIED reference (tests/golden/warp_att.pt)."""
    import os
    from heal_b200 import ops
    g = golden.load(os.path.join(golden_dir, "warp_att.pt"))
    out = ops.att_fuse(ops.to_act(g["x"].cuda()), g["affine"][0, 0, :3].cuda())
    torch.testing.assert_close(ops.act_to_nchw(out)[0].cpu().contiguous(), g["att"][0], rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("prec", ["fp32", "tc32", "tc32-mma", "tc32-gather"])
def test_sparse_stem_equals_dense_canvas_path_and_oracle(prec):
    """scatter + first residual block straight from the pillar list == the same block on the materialised canvas == the oracle."""
    from heal_b200 import ops, synth, engine
    from heal_b200.models.sub_modules.resblock import BasicBlock, conv1x1
    from oracle import procedural
    old, old_tc, old_gather = engine.PRECISION, engine.STEM_TC, ops.STEM_GATHER_TC
    ops.STEM_GATHER_TC = (prec == "tc32-gather")   # opt-in wgmma gather-GEMM stem (stem rulebook + heal_spconv_gather_gemm_tc)
    engine.STEM_TC = prec.endswith("-mma")          # heal_sparse_stem_tc (mma.sync, split-bf16) instead of the fp32 gather kernel
    prec = prec.split("-")[0]
    engine.set_precision(prec)
    try:
        sc = synth.scene(9, n_agents=2, rings=32, azimuth=512)
        per_agent = [voxelizer.points_to_voxel_c(p, PP_VOXEL, PP_RANGE, 32, 70000) for p in sc["points"]]
        col = {k: torch.from_numpy(v).cuda() for k, v in voxelizer.collate(per_agent).items()}
        shapes = {"vfe.pfn_layers.0.linear.weight": (64, 10), "vfe.pfn_layers.0.norm.weight": (64,), "vfe.pfn_layers.0.norm.bias": (64,),
                  "vfe.pfn_layers.0.norm.running_mean": (64,), "vfe.pfn_layers.0.norm.running_var": (64,)}
        sd = procedural.make_state_dict(shapes)
        w, b = ops.fold_linear_bn(sd["vfe.pfn_layers.0.linear.weight"], sd["vfe.pfn_layers.0.norm.weight"], sd["vfe.pfn_layers.0.norm.bias"],
                                  sd["vfe.pfn_layers.0.norm.running_mean"], sd["vfe.pfn_layers.0.norm.running_var"], 1e-3)
        blk = BasicBlock(64, 64, 2, torch.nn.Sequential(conv1x1(64, 64, 2), torch.nn.BatchNorm2d(64))).eval()
        blk_sd = procedural.make_state_dict(procedural.shapes_of(blk))
        blk.load_state_dict(blk_sd, strict=True)
        blk = blk.cuda()
        args = (col["voxel_features"], col["voxel_num_points"], col["voxel_coords"], w.cuda(), b.cuda(), PP_VOXEL, PP_RANGE, 512, 512, 2)
        # tc32 (default engine path): PillarVFE also emits split rows and the stem runs as two wgmma gather-GEMMs
        sparse = ops.pillar_vfe_sparse(*args, want_split_rows=ops.STEM_GATHER_TC)
        _, dense = ops.pillar_vfe_scatter(*args, canvas_fmt=engine.act_fmt())
        with torch.no_grad():
            a = ops.act_to_nchw(blk.forward_nhwc(sparse)).cpu()
            engine.SPARSE_STEM = False
            d = ops.act_to_nchw(blk.forward_nhwc(dense)).cpu()
            d2 = ops.act_to_nchw(blk.forward_nhwc(sparse)).cpu()          # SparseCanvas.dense() fallback
        assert torch.equal(d, d2)
        # fp32: same fp32 FMAs in a different order; tc32: the dense path additionally rounds the canvas and conv1's output to
        # 16-bit-mantissa split storage, so allow 1e-4 of the tensor's magnitude (1e-3 is the parity bar)
        scale = d.abs().max().item()
        tol = (1e-5 if prec == "fp32" else 1e-4) * max(scale, 1.0)
        err = (a - d).abs().max().item()
        assert err < tol, (err, tol, scale)
        # ... and against the ORACLE (PillarVFE -> scatter -> BasicBlock on CPU, oracle/nets.py), not only against our own dense path
        from oracle import nets
        cpu = {k: v.cpu() for k, v in col.items()}
        with torch.no_grad():
            pf = nets.pillar_vfe(sd, "vfe", cpu["voxel_features"], cpu["voxel_num_points"], cpu["voxel_coords"], PP_VOXEL, PP_RANGE)
            ref = nets.basic_block(nets.scatter(pf, cpu["voxel_coords"], 512, 512), {"blk." + k: v for k, v in blk_sd.items()}, "blk", 2, True)
        err_o = (a - ref).abs().max().item()
        assert err_o < 1e-3 * max(ref.abs().max().item(), 1.0), (err_o, ref.abs().max().item())
    finally:
        engine.SPARSE_STEM = True
        engine.STEM_TC = old_tc
        ops.STEM_GATHER_TC = old_gather
        engine.set_precision(old)


@pytest.mark.gpu
@pytest.mark.parametrize("use_perm,remove_ego", [(False, True), (True, True), (True, False)])
def test_mask_points_bit_exact(use_perm, remove_ego):
    """heal_mask_points == shuffle -> mask_ego_points -> mask_points_by_range (oracle/pcd.py, pinned to pcd_utils.py:41-95), per agent,
    order included; then the voxeliser on the filtered cloud equals the oracle voxeliser on the oracle-filtered cloud."""
    from heal_b200 import ops
    from oracle import pcd
    rng = np.random.default_rng(17)
    clouds = []
    for n in (30000, 1, 0, 12345):
        p = rng.uniform(-120, 120, size=(n, 4)).astype(np.float32)
        if n:
            p[:, 2] = rng.uniform(-4, 2, size=n)
            p[: n // 10, :2] = rng.uniform(-3, 3, size=(n // 10, 2))
        clouds.append(p)
    clouds[0][:4] = [[-1.95, 1.1, 0, 1], [102.4, 0, 0, 1], [5, 5, -3, 1], [2.95, -1.1, 0.5, 1]]
    offs = np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds])]).astype(np.int32)
    pts = np.concatenate(clouds)
    perms = [rng.permutation(c.shape[0]) for c in clouds] if use_perm else [None] * len(clouds)
    gperm = np.concatenate([pm + o for pm, o in zip(perms, offs[:-1])]).astype(np.int32) if use_perm else None
    ref = [pcd.filter_cloud(c, PP_RANGE, pm, remove_ego) for c, pm in zip(clouds, perms)]
    ref_offs = np.concatenate([[0], np.cumsum([r.shape[0] for r in ref])]).astype(np.int32)
    # capacity larger than the live count: the tail rows must be ignored
    cap = np.concatenate([pts, np.full((100, 4), 7.0, np.float32)])
    out, o2 = ops.mask_points(_cuda(cap).contiguous(), _cuda(offs), PP_RANGE, remove_ego,
                              _cuda(gperm) if use_perm else None)
    assert np.array_equal(o2.cpu().numpy(), ref_offs)
    assert np.array_equal(out[: ref_offs[-1]].cpu().numpy(), np.concatenate(ref))
    v, c, n, nv = ops.voxelize(out, o2, PP_RANGE, PP_VOXEL, 32, 70000)
    per_agent = [voxelizer.points_to_voxel_c(r, PP_VOXEL, PP_RANGE, 32, 70000) for r in ref]
    col = voxelizer.collate(per_agent)
    got = ops.trim_voxels(v, c, n, nv)
    assert np.array_equal(got["voxel_coords"].cpu().numpy(), col["voxel_coords"])
    assert np.array_equal(got["voxel_features"].cpu().numpy().view(np.uint32), col["voxel_features"].view(np.uint32))
