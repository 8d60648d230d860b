"""Lift-Splat-Shoot kernels vs the oracle and the reference-derived golden."""
import os

import numpy as np
import pytest
import torch

from oracle import golden

from oracle import lss

pytestmark = pytest.mark.gpu


def _mats(g):
    B, N = g["trans"].shape[:2]
    post_inv = torch.inverse(g["post_rots"]).reshape(B * N, 3, 3)
    combine = g["rots"].matmul(torch.inverse(g["intrins"])).reshape(B * N, 3, 3)
    return B, N, post_inv, combine


def test_lss_cell_index_and_pool_vs_golden(golden_dir):
    from heal_b200 import ops
    g = golden.load(os.path.join(golden_dir, "lss_small.pt"))
    cfg = g["cfg"]
    fr = lss.create_frustum(cfg["grid_conf"], cfg["data_aug_conf"]["final_dim"], cfg["img_downsample"])
    dx, bx, nx = lss.gen_dx_bx(cfg["grid_conf"]["xbound"], cfg["grid_conf"]["ybound"], cfg["grid_conf"]["zbound"])
    B, N, post_inv, combine = _mats(g)
    ref_cell = lss.cell_index(g["geom"], dx, bx, nx).view(B * N, *fr.shape[:3])
    cell = ops.lss_cell_index(fr.cuda(), post_inv.cuda(), g["post_trans"].reshape(B * N, 3).cuda(), combine.cuda(),
                              g["trans"].reshape(B * N, 3).cuda(), (bx - dx / 2.).tolist(), dx.tolist(), nx.tolist())
    got = cell.cpu().long()
    mism = (got != ref_cell)
    # the reference's own geometry is not reproducible to the last ulp across devices (torch.inverse / matmul), so a
    # frustum point within ~1e-5 cells of a boundary may legitimately land next door; bound the count and check that
    # every mismatch is such a boundary case
    frac = mism.float().mean().item()
    print(f"cell index mismatches: {int(mism.sum())} of {mism.numel()} ({frac:.2e})")
    assert frac < 2e-4
    v = ((g["geom"] - (bx - dx / 2.)) / dx).view(B * N, *fr.shape[:3], 3)
    near = ((v - v.round()).abs() < 1e-3).any(-1)
    assert bool((near | ~mism).all())
    # pooling with the ORACLE's indices (bit-identical inputs): fp tolerance only
    bev = ops.lss_pool(g["depth_logits"].cuda(), g["feat"].cuda(), ref_cell.int().cuda(), N, int(nx[0]), int(nx[1]))
    x = lss.outer_product(g["depth_logits"], g["feat"]).view(B, N, -1, *fr.shape[:3]).permute(0, 1, 3, 4, 5, 2)
    ref_exact = lss.voxel_pooling(g["geom"], x, dx, bx, nx, exact=True)
    got_bev = ops.act_to_nchw(bev).cpu().contiguous()
    torch.testing.assert_close(got_bev, ref_exact, rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(got_bev, g["bev"], rtol=1e-3, atol=1e-3)      # vs the unmodified reference (cumsum trick)


def test_lss_full_size_properties():
    """BASELINE config-4 shapes (4 cams, 704x256 -> 32x88, D=48, C=128, 256x256 BEV): mass conservation + linearity."""
    from heal_b200 import ops, synth
    grid_conf = {"xbound": [-51.2, 51.2, 0.4], "ybound": [-51.2, 51.2, 0.4], "zbound": [-10, 10, 20.0], "ddiscr": [2, 50, 48], "mode": "LID"}
    fr = lss.create_frustum(grid_conf, [256, 704], 8)
    dx, bx, nx = lss.gen_dx_bx(grid_conf["xbound"], grid_conf["ybound"], grid_conf["zbound"])
    rots, trans, intr, post_rots, post_trans = [torch.from_numpy(a) for a in synth.camera_rig(2, 4, 256, 704)]
    g = {"rots": rots, "trans": trans, "intrins": intr, "post_rots": post_rots, "post_trans": post_trans}
    B, N, post_inv, combine = _mats(g)
    cell = ops.lss_cell_index(fr.cuda(), post_inv.cuda(), post_trans.reshape(B * N, 3).cuda(), combine.cuda(),
                              trans.reshape(B * N, 3).cuda(), (bx - dx / 2.).tolist(), dx.tolist(), nx.tolist())
    gen = torch.Generator().manual_seed(0)
    logits = torch.randn(B * N, 48, 32, 88, generator=gen).cuda()
    feat = torch.randn(B * N, 128, 32, 88, generator=gen).cuda()
    bev = ops.lss_pool(logits, feat, cell, N, 256, 256).t
    # every in-grid frustum point deposits prob*feat: total mass per agent and channel
    prob = torch.softmax(logits, 1)
    w = (prob * (cell >= 0)).sum(1)                                  # (BN, fH, fW)
    expect = (feat * w.unsqueeze(1)).view(B, N, 128, -1).sum((1, 3))   # (B, C)
    torch.testing.assert_close(bev.sum((1, 2)), expect, rtol=2e-3, atol=2e-2)
    bev2 = ops.lss_pool(logits, 2 * feat, cell, N, 256, 256).t
    torch.testing.assert_close(bev2, 2 * bev, rtol=1e-4, atol=1e-4)   # linear in the features (atomics reorder only)


def test_lss_pool_sorted_vs_golden_both_layouts_and_deterministic(golden_dir):
    """heal_lss_pool_sorted (cell-sorted interval sums, no atomics): equals the exact per-cell sum, the unmodified reference's
    cumsum output within its own rounding, for NCHW inputs and for the channels-last fused-heads layout, bit-identical run to run."""
    from heal_b200 import ops
    g = golden.load(os.path.join(golden_dir, "lss_small.pt"))
    cfg = g["cfg"]
    fr = lss.create_frustum(cfg["grid_conf"], cfg["data_aug_conf"]["final_dim"], cfg["img_downsample"])
    dx, bx, nx = lss.gen_dx_bx(cfg["grid_conf"]["xbound"], cfg["grid_conf"]["ybound"], cfg["grid_conf"]["zbound"])
    B, N, _, _ = _mats(g)
    D, fH, fW = fr.shape[:3]
    C = g["feat"].shape[1]
    HW = fH * fW
    ref_cell = lss.cell_index(g["geom"], dx, bx, nx).view(B * N, D, fH, fW).int().cuda().contiguous()
    x = lss.outer_product(g["depth_logits"], g["feat"]).view(B, N, -1, D, fH, fW).permute(0, 1, 3, 4, 5, 2)
    ref_exact = lss.voxel_pooling(g["geom"], x, dx, bx, nx, exact=True)
    lg, ft = g["depth_logits"].cuda().contiguous(), g["feat"].cuda().contiguous()
    a = ops.lss_pool_sorted(lg, (D * HW, HW, 1), ft, (C * HW, HW, 1), ref_cell, N, D, C, fH, fW, int(nx[0]), int(nx[1]))
    got = ops.act_to_nchw(a).cpu().contiguous()
    torch.testing.assert_close(got, ref_exact, rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(got, g["bev"], rtol=1e-3, atol=1e-3)
    # channels-last fused heads: (BN, fH, fW, D + C)
    fused = torch.cat([lg.permute(0, 2, 3, 1), ft.permute(0, 2, 3, 1)], -1).contiguous()
    S = D + C
    b = ops.lss_pool_sorted(fused, (HW * S, 1, S), fused[..., D:], (HW * S, 1, S), ref_cell, N, D, C, fH, fW, int(nx[0]), int(nx[1]))
    assert torch.equal(b.t, a.t)                                      # same sums in the same order from either layout
    for _ in range(3):
        again = ops.lss_pool_sorted(lg, (D * HW, HW, 1), ft, (C * HW, HW, 1), ref_cell, N, D, C, fH, fW, int(nx[0]), int(nx[1]))
        assert torch.equal(again.t, a.t)                              # deterministic, unlike the atomicAdd kernel
    s = ops.lss_pool_sorted(lg, (D * HW, HW, 1), ft, (C * HW, HW, 1), ref_cell, N, D, C, fH, fW, int(nx[0]), int(nx[1]), out_fmt="split")
    assert (ops.act_to_nchw(s).cpu() - got).abs().max().item() < 1e-4 * max(got.abs().max().item(), 1.0)


def test_camera_trunk_on_the_conv_engine_vs_torch():
    """CamEncode_Resnet101.heads_nhwc (space-to-depth stem on wgmma, heal_maxpool3x3s2, Bottlenecks, fused heads) == the torch
    modules' own forward (torchvision resnet101 conv1..layer2 + 1x1 heads, lss_submodule.py:140-233) on CPU."""
    from heal_b200 import engine
    from heal_b200.models.heter_encoders import CamEncode_Resnet101
    from workloads import procedural
    old = engine.PRECISION
    try:
        m = CamEncode_Resnet101(48, 128, 8, [2, 50, 48], "LID", False, False).eval()
        m.load_state_dict(procedural.make_state_dict(procedural.shapes_of(m)), strict=True)
        x = torch.randn(2, 3, 64, 96, generator=torch.Generator().manual_seed(2))
        with torch.no_grad():
            dl, ft = m.heads(x)
        m = m.cuda()
        for prec, tol in (("tc32", 1e-3), ("fp32", 1e-3), ("bf16", 2.5e-2)):
            engine.set_precision(prec)
            with torch.no_grad():
                y = m.heads_nhwc(x.cuda()).t.cpu()
            assert y.shape == (2, 8, 12, 48 + 128)
            ref = torch.cat([dl, ft], 1).permute(0, 2, 3, 1)
            err = (y - ref).abs().max().item()
            scale = max(ref.abs().max().item(), 1.0)
            print(f"camera trunk {prec}: max|ref|={scale:.3f} err={err:.3e}")
            assert err <= tol * scale
    finally:
        engine.set_precision(old)


def test_lift_splat_shoot_voxel_equals_lss_for_single_slice_grid():
    """LiftSplatShootVoxel (heter_encoders.py:244-301) differs from LiftSplatShoot only in how z slices are merged (max vs concat);
    with the single-slice grids of every HEAL yaml (zbound [-10, 10, 20]) both reduce to the same (B,C,ny,nx) map."""
    from heal_b200 import synth
    from heal_b200.models.heter_encoders import LiftSplatShoot, LiftSplatShootVoxel
    from oracle import make_golden
    from workloads import procedural
    cfg = make_golden.lss_small_cfg()
    a, b = LiftSplatShoot(dict(cfg)).eval(), LiftSplatShootVoxel(dict(cfg)).eval()
    sd = procedural.make_state_dict(procedural.shapes_of(a))
    a.load_state_dict(sd, strict=True)
    b.load_state_dict(sd, strict=True)
    a, b = a.cuda(), b.cuda()
    rots, trans, intr, post_rots, post_trans = [torch.from_numpy(v).cuda() for v in synth.camera_rig(1, 2, 64, 128)]
    imgs = torch.randn(1, 2, 3, 64, 128, generator=torch.Generator().manual_seed(8)).cuda()
    dd = {"inputs_m2": {"imgs": imgs, "rots": rots, "trans": trans, "intrins": intr, "post_rots": post_rots, "post_trans": post_trans}}
    with torch.no_grad():
        ya, yb = a(dd, "m2"), b(dd, "m2")
    assert ya.shape == (1, 32, 64, 64) and torch.equal(ya, yb)


def test_camera_matrices_vs_torch_inverse_and_graph_capture():
    """heal_lss_camera_matrices == (inverse(post_rots), rots @ inverse(intrins)) to fp32 rounding, and the whole LSS encoder
    (trunk, heads, camera algebra, cell index, sorted pooling) captures into a CUDA graph whose replay equals the eager forward."""
    from heal_b200 import engine, ops, synth
    from heal_b200.models.heter_encoders import LiftSplatShoot
    from oracle import make_golden
    from workloads import procedural
    rots, trans, intr, post_rots, post_trans = [torch.from_numpy(v) for v in synth.camera_rig(2, 4, 256, 704)]
    pi, cb = ops.lss_camera_matrices(rots.cuda(), intr.cuda(), post_rots.cuda())
    pi_ref = torch.inverse(post_rots.double()).reshape(-1, 3, 3)
    cb_ref = rots.double().matmul(torch.inverse(intr.double())).reshape(-1, 3, 3)
    assert (pi.cpu().double() - pi_ref).abs().max() <= 2e-7 * pi_ref.abs().max()
    assert (cb.cpu().double() - cb_ref).abs().max() <= 4e-7 * cb_ref.abs().max()
    # same cells as with torch.inverse's fp32 LU except frustum points on a cell boundary
    engine.set_precision("bf16")
    try:
        cfg = make_golden.lss_small_cfg()
        m = LiftSplatShoot(dict(cfg)).eval()
        m.load_state_dict(procedural.make_state_dict(procedural.shapes_of(m)), strict=True)
        m = m.cuda()
        r2, t2, k2, pr2, pt2 = [torch.from_numpy(v).cuda() for v in synth.camera_rig(1, 2, 64, 128)]
        cell = m.cell_index(r2, t2, k2, pr2, pt2)
        cell_t = ops.lss_cell_index(m.frustum, torch.inverse(pr2).reshape(-1, 3, 3), pt2.reshape(-1, 3),
                                    r2.matmul(torch.inverse(k2)).reshape(-1, 3, 3), t2.reshape(-1, 3), m._lower_host, m._dx_host,
                                    m._nx_host)
        assert (cell != cell_t).float().mean().item() < 2e-4
        imgs = torch.randn(1, 2, 3, 64, 128, generator=torch.Generator().manual_seed(8)).cuda()
        dd = {"inputs_m2": {"imgs": imgs, "rots": r2, "trans": t2, "intrins": k2, "post_rots": pr2, "post_trans": pt2}}
        with torch.no_grad():
            eager = m(dd, "m2").clone()
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                m(dd, "m2")
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, capture_error_mode="thread_local"):
                out = m(dd, "m2")
            imgs.normal_()          # the graph reads the static input buffers: new images, same graph
            g.replay()
            torch.cuda.synchronize()
            assert torch.equal(out, m(dd, "m2")) and not torch.equal(out, eager)
    finally:
        engine.set_precision("tc32")
