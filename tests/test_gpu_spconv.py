"""Sparse 3-D convolution kernels + SECOND encoder vs the CPU oracle (oracle/sparse_conv.py)."""
import numpy as np
import pytest
import torch

from oracle import sparse_conv as sc, procedural, voxelizer

pytestmark = pytest.mark.gpu


def _random_sparse(rng, batch, shape, n, cin):
    cells = rng.choice(batch * shape[0] * shape[1] * shape[2], size=n, replace=False)
    c = np.zeros((n, 4), dtype=np.int32)
    k = cells.copy()
    c[:, 3] = k % shape[2]; k //= shape[2]
    c[:, 2] = k % shape[1]; k //= shape[1]
    c[:, 1] = k % shape[0]; c[:, 0] = k // shape[0]
    return torch.from_numpy(rng.standard_normal((n, cin)).astype(np.float32)), c


def _lin(c, shape):
    c = np.asarray(c).astype(np.int64)
    return ((c[:, 0] * shape[0] + c[:, 1]) * shape[1] + c[:, 2]) * shape[2] + c[:, 3]


@pytest.mark.parametrize("cin,cout,n", [(4, 16, 5000), (16, 16, 777), (32, 32, 3000), (64, 64, 2000)])
def test_subm_conv_vs_oracle(cin, cout, n):
    from heal_b200 import ops
    rng = np.random.default_rng(cin + cout)
    shape, B = [21, 64, 64], 2
    feats, coords = _random_sparse(rng, B, shape, n, cin)
    w = torch.from_numpy((rng.standard_normal((cout, 3, 3, 3, cin)) / np.sqrt(27 * cin)).astype(np.float32))
    bias = torch.from_numpy(rng.standard_normal(cout).astype(np.float32))
    ref = torch.relu(sc.subm_conv3d(feats, coords, w, shape) + bias)
    st = ops.SparseTensor(feats.cuda(), torch.from_numpy(coords).cuda(), None, shape, B)
    nbr = ops.sp_subm_neighbors(st, (3, 3, 3))
    wp = w.reshape(cout, 27, cin).permute(1, 2, 0).contiguous().cuda()
    out = ops.sp_gather_gemm(st.feats, nbr, None, wp, bias.cuda(), True)
    torch.testing.assert_close(out.cpu(), ref, rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("ksize,stride,pad,shape", [((3, 3, 3), (2, 2, 2), (1, 1, 1), [41, 64, 64]),
                                                     ((3, 3, 3), (2, 2, 2), (0, 1, 1), [11, 32, 48]),
                                                     ((3, 1, 1), (2, 1, 1), (0, 0, 0), [5, 32, 32])])
def test_strided_conv_vs_oracle(ksize, stride, pad, shape):
    from heal_b200 import ops
    rng = np.random.default_rng(sum(shape))
    B, cin, cout = 3, 16, 32
    feats, coords = _random_sparse(rng, B, shape, 4000, cin)
    K = ksize[0] * ksize[1] * ksize[2]
    w = torch.from_numpy((rng.standard_normal((cout, *ksize, cin)) / np.sqrt(K * cin)).astype(np.float32))
    ref, rc, oshape = sc.sparse_conv3d(feats, coords, w, shape, stride, pad)
    st = ops.SparseTensor(feats.cuda(), torch.from_numpy(coords).cuda(), None, shape, B)
    out_st, nbr = ops.sp_strided(st, ksize, stride, pad, out_capacity=8 * 4000)   # random (non-surface) inputs dilate up to 8x
    assert out_st.spatial_shape == oshape
    m = int(out_st.rows_dev.item())                               # live rows stay on the device (no host sync inside sp_strided)
    assert m == len(rc) and m <= out_st.capacity                  # same active output set size
    wp = w.reshape(cout, K, cin).permute(1, 2, 0).contiguous().cuda()
    out = ops.sp_gather_gemm(st.feats, nbr, None, wp, None, False)[:m].cpu()
    oc = out_st.coords[:m].cpu().numpy()
    order = np.argsort(_lin(oc, oshape))
    assert np.array_equal(oc[order], rc)                          # identical site set (oracle order = sorted)
    torch.testing.assert_close(out[torch.from_numpy(order)], ref, rtol=1e-4, atol=1e-4)
    # determinism of the output ordering: a second build gives the same coords row for row
    out_st2, _ = ops.sp_strided(st, ksize, stride, pad, out_capacity=8 * 4000)
    assert torch.equal(out_st2.coords[:m], out_st.coords[:m])
    # the site -> row table of the new level serves SubM lookups: every output site finds itself at the centre offset
    nb2 = ops.sp_subm_neighbors(out_st, (3, 3, 3))
    assert torch.equal(nb2[:m, 13].cpu(), torch.arange(m, dtype=torch.int32))


@pytest.mark.parametrize("cin,cout,n", [(16, 16, 777), (16, 32, 5000), (32, 32, 3000), (32, 64, 4100), (64, 64, 2000), (64, 128, 1500)])
def test_subm_conv_tensor_core_vs_oracle(cin, cout, n):
    """heal_spconv_gather_gemm_tc (wgmma, split-bf16 rows, cp.async gather) vs the oracle: fp32-equivalent (2^-16 per product)."""
    from heal_b200 import ops
    rng = np.random.default_rng(100 + cin + cout)
    shape, B = [21, 64, 64], 2
    feats, coords = _random_sparse(rng, B, shape, n, cin)
    w = torch.from_numpy((rng.standard_normal((cout, 3, 3, 3, cin)) / np.sqrt(27 * cin)).astype(np.float32))
    bias = torch.from_numpy(rng.standard_normal(cout).astype(np.float32))
    ref = torch.relu(sc.subm_conv3d(feats, coords, w, shape) + bias)
    st = ops.SparseTensor(feats.cuda(), torch.from_numpy(coords).cuda(), None, shape, B)
    nbr = ops.sp_subm_neighbors(st, (3, 3, 3))
    wp = w.reshape(cout, 27, cin).permute(1, 2, 0).contiguous().cuda()
    pk = ops.pack_spconv_tc(wp)
    fs = ops.rows_to_split(st.feats, None)
    assert torch.allclose(fs[:, :cin].float() + fs[:, cin:].float(), st.feats, rtol=0, atol=1e-4)
    out32 = ops.sp_gather_gemm_tc(fs, nbr, None, pk, bias.cuda(), True, cin, cout, want_f32=True)
    outs = ops.sp_gather_gemm_tc(fs, nbr, None, pk, bias.cuda(), True, cin, cout, want_f32=False)
    scale = max(ref.abs().max().item(), 1.0)
    assert (out32.cpu() - ref).abs().max().item() < 1e-4 * scale
    merged = outs[:, :cout].float() + outs[:, cout:].float()
    assert (merged.cpu() - ref).abs().max().item() < 1e-4 * scale
    # a live-row count on the device smaller than the capacity: rows beyond it are not written
    m_dev = torch.tensor([n // 2], dtype=torch.int32, device="cuda")
    part = ops.sp_gather_gemm_tc(fs, nbr, m_dev, pk, bias.cuda(), True, cin, cout, want_f32=True)
    assert torch.equal(part[: n // 2], out32[: n // 2])


def test_strided_conv_tensor_core_vs_oracle():
    from heal_b200 import ops
    ksize, stride, pad, shape = (3, 3, 3), (2, 2, 2), (1, 1, 1), [41, 64, 64]
    rng = np.random.default_rng(4242)
    B, cin, cout = 3, 32, 64
    feats, coords = _random_sparse(rng, B, shape, 6000, cin)
    w = torch.from_numpy((rng.standard_normal((cout, *ksize, cin)) / np.sqrt(27 * cin)).astype(np.float32))
    ref, rc, oshape = sc.sparse_conv3d(feats, coords, w, shape, stride, pad)
    st = ops.SparseTensor(feats.cuda(), torch.from_numpy(coords).cuda(), None, shape, B)
    out_st, nbr = ops.sp_strided(st, ksize, stride, pad, out_capacity=8 * 6000)
    m = int(out_st.rows_dev.item())
    assert m == len(rc)
    pk = ops.pack_spconv_tc(w.reshape(cout, 27, cin).permute(1, 2, 0).contiguous().cuda())
    out = ops.sp_gather_gemm_tc(ops.rows_to_split(st.feats, None), nbr, out_st.rows_dev, pk, None, False, cin, cout, want_f32=True)[:m].cpu()
    order = np.argsort(_lin(out_st.coords[:m].cpu().numpy(), oshape))
    assert (out[torch.from_numpy(order)] - ref).abs().max().item() < 1e-4 * max(ref.abs().max().item(), 1.0)


def test_strided_overflow_is_reported():
    from heal_b200 import ops
    rng = np.random.default_rng(1)
    shape, B = [41, 64, 64], 1
    feats, coords = _random_sparse(rng, B, shape, 4000, 16)
    st = ops.SparseTensor(feats.cuda(), torch.from_numpy(coords).cuda(), None, shape, B)
    out_st, _ = ops.sp_strided(st, (3, 3, 3), (2, 2, 2), (1, 1, 1), out_capacity=100)
    with pytest.raises(RuntimeError):
        ops.sp_check_overflow([out_st])


def _second_args(rng_):
    return {"voxel_size": [0.1, 0.1, 0.1], "lidar_range": rng_, "mean_vfe": {"num_point_features": 4},
            "spconv": {"num_features_in": 4, "num_features_out": 64}, "map2bev": {"feature_num": 128}}


@pytest.mark.parametrize("rng_,n_agents,rings", [([-25.6, -25.6, -3, 25.6, 25.6, 1], 2, 32), ([-102.4, -102.4, -3, 102.4, 102.4, 1], 2, 64)])
def test_second_encoder_vs_oracle(rng_, n_agents, rings):
    from heal_b200 import synth
    from heal_b200.models.heter_encoders import SECOND
    args = _second_args(rng_)
    enc = SECOND(args).eval()
    sd = procedural.make_state_dict(procedural.shapes_of(enc))
    enc.load_state_dict(sd, strict=True)
    enc = enc.cuda()
    sc_ = synth.scene(17, n_agents=n_agents, rings=rings, azimuth=1024 if rings == 64 else 512)
    per_agent = [voxelizer.points_to_voxel_c(p, args["voxel_size"], rng_, 5, 70000) for p in sc_["points"]]
    col = {k: torch.from_numpy(v) for k, v in voxelizer.collate(per_agent).items()}
    with torch.no_grad():
        ref = sc.second_encoder(sd, "", {**args}, col) if False else sc.second_encoder({("x." + k): v for k, v in sd.items()}, "x", args, col)
        got = enc({"inputs_m3": {k: v.cuda() for k, v in col.items()}}, "m3")
    assert got.shape == ref.shape
    err = (got.cpu() - ref).abs().max().item()
    print(f"SECOND {rng_[3]}m M={col['voxel_coords'].shape[0]}: out {tuple(ref.shape)} max|ref|={ref.abs().max().item():.3f} err={err:.3e}")
    assert err < 1e-3
    # GPU-voxelized raw-point input path gives the same BEV map
    offs = np.concatenate([[0], np.cumsum([p.shape[0] for p in sc_["points"]])]).astype(np.int32)
    with torch.no_grad():
        got2 = enc({"inputs_m3": {"points": torch.from_numpy(np.concatenate(sc_["points"])).cuda(),
                                  "agent_offsets": torch.from_numpy(offs).cuda()}}, "m3")
    torch.testing.assert_close(got2, got, rtol=1e-5, atol=1e-5)
