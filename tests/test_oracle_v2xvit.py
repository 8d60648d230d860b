"""V2X-ViT (fusion_method v2xvit) on the CPU: the oracle against the reference's own modules (goldens), the mirror modules'
parameter tables, the structural facts the GPU path relies on (padded slots never reach a real one, the ROI mask is all ones),
the shape and scope errors, and the GPU formulation (real agents only, egos first, HGT relations and scale folded into one
qkv Linear, ego-only last layer, one STTF resample, SplitAttn as pool / gate / combine) restated in float64 against the literal
oracle."""
import copy
import os

import pytest
import torch
import torch.nn.functional as F

from oracle import fusion_methods, golden, make_golden_v2xvit as mg, procedural, v2xvit as vx


def _rel_err(got, ref):
    return (got - ref).abs().max().item() / max(ref.abs().max().item(), 1e-30)


def _sd(shapes, dtype=torch.float32):
    return {"f." + k: v.to(dtype) for k, v in procedural.make_state_dict(shapes).items()}


@pytest.mark.parametrize("case", ["c256", "l2"])
def test_v2xvit_oracle_vs_reference(golden_dir, case):
    g = vx.load_module_golden(golden_dir)[case]
    x, rl, pw = vx.case_inputs(case)
    assert torch.equal(rl, g["record_len"]) and torch.equal(pw, g["pairwise_t_matrix"])
    aff = vx.case_affine(pw)
    assert torch.equal(aff, g["affine"])
    with torch.no_grad():
        out = vx.v2xvit_fusion(x, _sd(g["shapes"]), "f", g["args"], rl, aff)
    assert _rel_err(out[:, ::g["stride"]], g["out_s"]) <= 1e-5


def test_heter_model_baseline_v2xvit_oracle_vs_reference(golden_dir):
    g = golden.load(os.path.join(golden_dir, "heter_model_baseline_v2xvit_small.pt"))
    sd = procedural.make_state_dict(g["shapes"])
    with torch.no_grad():
        out = vx.heter_model_baseline(sd, g["args"], g["data"])
    for k in ("cls_preds", "reg_preds", "dir_preds"):
        assert _rel_err(out[k], g["out"][k]) <= 1e-5, k


def test_mirror_parameter_tables_match_reference(golden_dir):
    from heal_b200.models.fuse_modules.fusion_in_one import V2XViTFusion
    from heal_b200.models.heter_model_baseline import HeterModelBaseline
    for case, g in vx.load_module_golden(golden_dir).items():
        assert procedural.shapes_of(V2XViTFusion(copy.deepcopy(g["args"]))) == g["shapes"], case
    assert len(vx.load_module_golden(golden_dir)["c256"]["shapes"]) == 134
    gm = golden.load(os.path.join(golden_dir, "heter_model_baseline_v2xvit_small.pt"))
    assert procedural.shapes_of(HeterModelBaseline(copy.deepcopy(gm["args"]))) == gm["shapes"]


def test_mirror_sttf_matrix_is_the_reference_chain():
    from heal_b200.models.sub_modules.v2xvit_basic import STTF
    for H, W in ((128, 128), (64, 128), (32, 32), (16, 32), (256, 256), (100, 252)):
        scm = torch.eye(4).expand(1, 2, 4, 4)
        T = vx.sttf_matrix(scm, H, W, 0.4, 4)
        want = vx.warp_affine_matrix(T, (H, W), (H, W))[0]
        got = STTF({"voxel_size": [0.4, 0.4, 4], "downsample_rate": 4}).theta(H, W)
        assert got.dtype == torch.float32 and torch.equal(got, want), (H, W)


# ---- structural facts ---------------------------------------------------------------------------------------------
SHIPPED_SHAPES = [(128, 128), (64, 128), (256, 256), (48, 176), (100, 252)]
TEST_SHAPES = [(16, 32), (16, 16), (32, 32)]


@pytest.mark.parametrize("HW", SHIPPED_SHAPES + TEST_SHAPES)
def test_roi_mask_is_the_cav_mask(HW):
    H, W = HW
    mask = torch.tensor([[1, 1, 1, 0, 0], [1, 1, 0, 0, 0]])
    scm = torch.eye(4).expand(2, 5, 4, 4)
    com = vx.get_roi_and_cav_mask((2, 5, H, W, 8), mask, scm, 0.4, 4)
    assert com.shape == (2, H, W, 1, 5)
    assert torch.equal(com, mask[:, None, None, None, :].float().expand(2, H, W, 1, 5))


def test_padded_slots_do_not_change_the_output(golden_dir):
    g = vx.load_module_golden(golden_dir)["c256"]
    sd = _sd(g["shapes"])
    x = torch.randn(3, 256, 16, 32, generator=torch.Generator().manual_seed(5))
    _, _, pw = vx.case_inputs("c256")
    aff5 = vx.case_affine(pw)[:1]
    with torch.no_grad():
        y5 = vx.v2xvit_fusion(x, sd, "f", g["args"], torch.tensor([3]), aff5)
        y3 = vx.v2xvit_fusion(x, sd, "f", g["args"], torch.tensor([3]), aff5[:, :3, :3].contiguous())
    assert torch.equal(y5, y3)


# ---- errors ---------------------------------------------------------------------------------------------------------
def test_shape_errors():
    from heal_b200.models.fuse_modules.fusion_in_one import V2XViTFusion
    m = V2XViTFusion(vx.v2xvit_args()).eval()
    _, _, pw = vx.case_inputs("c256")
    aff = vx.case_affine(pw)
    with pytest.raises(ValueError, match="not divisible"):
        m(torch.zeros(5, 256, 16, 24), torch.tensor([3, 2]), aff)
    with pytest.raises(ValueError, match="dim 256"):
        V2XViTFusion(vx.v2xvit_args(dim=128))
    with pytest.raises(ValueError, match="channels"):
        m(torch.zeros(5, 128, 16, 32), torch.tensor([3, 2]), aff)


def test_record_len_that_does_not_fit_raises_before_any_launch():
    from heal_b200.models.fuse_modules.fusion_in_one import V2XViTFusion
    m = V2XViTFusion(vx.v2xvit_args()).eval()

    class FakeAct:
        N, H, W, C = 7, 16, 32, 256
    _, _, pw = vx.case_inputs("c256")
    aff = vx.case_affine(pw)
    for rl in ([6, 1], [3], [3, 0], [2, 2]):
        with pytest.raises(ValueError, match="record_len"):
            m.forward_nhwc(FakeAct(), rl, aff)


@pytest.mark.parametrize("edit,what", [
    (lambda e: e.update(use_RTE=True) or e["cav_att_config"].update(use_RTE=True), "use_RTE"),
    (lambda e: e["cav_att_config"].update(use_hetero=False), "use_hetero"),
    (lambda e: e["pwindow_att_config"].update(fusion_method="naive"), "naive"),
])
def test_unbuilt_variants_name_the_scope(edit, what):
    from heal_b200.models.fuse_modules.fusion_in_one import V2XViTFusion
    args = vx.v2xvit_args()
    edit(args["transformer"]["encoder"])
    with pytest.raises(NotImplementedError, match=f"{what}.*outside the heal_b200 hot-path scope"):
        V2XViTFusion(args)


def test_baseline_without_v2xvit_block_names_the_scope():
    from heal_b200.models.heter_model_baseline import HeterModelBaseline
    args = mg.baseline_v2xvit_args()
    del args["v2xvit"]
    with pytest.raises(NotImplementedError, match="outside the heal_b200 hot-path scope"):
        HeterModelBaseline(args)


# ---- the GPU formulation in float64 -----------------------------------------------------------------------------------
def gpu_formulation(x, sd, p, args, record_len, aff):
    """What V2XViTFusion.forward_nhwc launches, in plain torch over NHWC maps of the real agents only, egos first."""
    from heal_b200.models.sub_modules.v2xvit_basic import STTF
    enc = args["transformer"]["encoder"]
    cav, pw = enc["cav_att_config"], enc["pwindow_att_config"]
    _, C, H, W = x.shape
    rl = [int(n) for n in record_len]
    B = len(rl)
    starts = [sum(rl[:b]) for b in range(B)]
    ego = torch.cat([fusion_methods.warp_affine_simple(x[starts[b]:starts[b] + 1], aff[b, 0, :1], (H, W)) for b in range(B)])
    others = [fusion_methods.warp_affine_simple(x[starts[b] + 1:starts[b] + rl[b]], aff[b, 0, 1:rl[b]], (H, W))
              for b in range(B) if rl[b] > 1]
    X = ego
    if others:
        o = torch.cat(others)
        th = STTF(enc["sttf"]).theta(H, W).expand(o.shape[0], 2, 3)
        grid = F.affine_grid(th, list(o.shape), align_corners=True).to(o.dtype)
        X = torch.cat([ego, F.grid_sample(o, grid, align_corners=True, padding_mode="zeros")])
    X = X.permute(0, 2, 3, 1)                                                   # N H W C, egos first
    other0 = [B + sum(r - 1 for r in rl[:b]) for b in range(B)]
    members = [[b] + list(range(other0[b], other0[b] + rl[b] - 1)) for b in range(B)]

    def ln(t, q):
        return F.layer_norm(t, (C,), sd[q + ".weight"], sd[q + ".bias"], 1e-5)

    hd, dh = cav["heads"], cav["dim_head"]
    for i in range(enc["depth"]):
        last = i == enc["depth"] - 1
        bp = f"{p}.fusion_net.encoder.layers.{i}.0.layers.0"
        hp = bp + ".0.fn"
        ra, rm = sd[hp + ".relation_att"][0], sd[hp + ".relation_msg"][0]
        wq = torch.einsum("mpq,mpc->mqc", ra, sd[hp + ".q_linears.0.weight"].reshape(hd, dh, -1)).reshape(hd * dh, -1)
        bq = torch.einsum("mpq,mp->mq", ra, sd[hp + ".q_linears.0.bias"].reshape(hd, dh)).reshape(-1)
        wv = torch.einsum("mpc,mpk->mck", rm, sd[hp + ".v_linears.0.weight"].reshape(hd, dh, -1)).reshape(hd * dh, -1)
        bv = torch.einsum("mpc,mp->mc", rm, sd[hp + ".v_linears.0.bias"].reshape(hd, dh)).reshape(-1)
        w = torch.cat([wq * dh ** -0.5, sd[hp + ".k_linears.0.weight"], wv])
        b_ = torch.cat([bq * dh ** -0.5, sd[hp + ".k_linears.0.bias"], bv])
        qkv = F.linear(ln(X, bp + ".0.norm"), w, b_)
        inner = hd * dh
        outs = []
        for b in range(B):
            idx = members[b]
            q = qkv[idx[:1] if last else idx, ..., :inner].reshape(-1, H, W, hd, dh)
            k = qkv[idx, ..., inner:2 * inner].reshape(len(idx), H, W, hd, dh)
            v = qkv[idx, ..., 2 * inner:].reshape(len(idx), H, W, hd, dh)
            s = torch.einsum("ihwmc,jhwmc->hwmij", q, k).softmax(-1)
            outs.append(torch.einsum("hwmij,jhwmc->ihwmc", s, v).reshape(-1, H, W, inner))
        a = torch.cat(outs) if last else torch.zeros_like(X[..., :inner]).index_copy(
            0, torch.tensor([j for m in members for j in m]), torch.cat(outs))
        X = (X[:B] if last else X) + F.linear(a, sd[hp + ".a_linears.0.weight"], sd[hp + ".a_linears.0.bias"])
        y = ln(X, bp + ".1.norm")
        n = X.shape[0]
        wp = bp + ".1.fn"
        br = []
        for kb, (heads, dhw, ws) in enumerate(zip(pw["heads"], pw["dim_head"], pw["window_size"])):
            q_ = f"{wp}.pwmsa.{kb}"
            inner_w = heads * dhw
            wt = sd[q_ + ".to_qkv.weight"]
            t = F.linear(y, torch.cat([wt[:inner_w] * dhw ** -0.5, wt[inner_w:]]))
            t = t.reshape(n, H // ws, ws, W // ws, ws, 3, heads, dhw).permute(5, 0, 1, 3, 6, 2, 4, 7)
            t = t.reshape(3, n, H // ws, W // ws, heads, ws * ws, dhw)
            ri = vx.relative_indices(ws)
            bias = sd[q_ + ".pos_embedding"][ri[:, :, 0], ri[:, :, 1]]
            o = (t[0] @ t[1].transpose(-1, -2) + bias).softmax(-1) @ t[2]
            o = o.reshape(n, H // ws, W // ws, heads, ws, ws, dhw).permute(0, 1, 4, 2, 5, 3, 6).reshape(n, H, W, inner_w)
            br.append(F.linear(o, sd[q_ + ".to_out.0.weight"], sd[q_ + ".to_out.0.bias"]))
        sp = wp + ".split_attn"
        pooled = (br[0] + br[1] + br[2]).sum((1, 2)) / (H * W)
        gt = F.relu(F.layer_norm(pooled @ sd[sp + ".fc1.weight"].t(), (C,), sd[sp + ".bn1.weight"], sd[sp + ".bn1.bias"], 1e-5))
        gt = (gt @ sd[sp + ".fc2.weight"].t()).reshape(n, 3, C).softmax(1)
        X = br[0] * gt[:, None, None, 0] + br[1] * gt[:, None, None, 1] + br[2] * gt[:, None, None, 2] + X
        fp = f"{p}.fusion_net.encoder.layers.{i}.1"
        h = F.gelu(F.linear(ln(X, fp + ".norm"), sd[fp + ".fn.net.0.weight"], sd[fp + ".fn.net.0.bias"]))
        X = F.linear(h, sd[fp + ".fn.net.3.weight"], sd[fp + ".fn.net.3.bias"]) + X
    return X.permute(0, 3, 1, 2)


@pytest.mark.parametrize("case", ["c256", "l2"])
def test_gpu_formulation_matches_oracle_float64(golden_dir, case):
    g = vx.load_module_golden(golden_dir)[case]
    x, rl, pw = vx.case_inputs(case)
    aff = vx.case_affine(pw).double()
    sd = _sd(g["shapes"], torch.float64)
    with torch.no_grad():
        ref = vx.v2xvit_fusion(x.double(), sd, "f", g["args"], rl, aff)
        got = gpu_formulation(x.double(), sd, "f", g["args"], rl, aff)
    assert got.shape == ref.shape
    assert _rel_err(got, ref) <= 1e-10
