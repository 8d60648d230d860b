"""CoBEVT (fusion_method cobevt) on the CPU: the oracle against the reference's own modules (goldens), the mirror modules'
parameter tables and relative_position_index, the shape errors, and the GPU formulation (address-rule token gather, dense
key-major bias, masked keys skipped, Linears as 1x1 convs, scale folded into the q rows) restated in float64 against the
literal oracle."""
import copy
import os

import pytest
import torch
import torch.nn.functional as F

from oracle import cobevt as cb, golden, make_golden_cobevt as mg, nets, procedural


def _rel_err(got, ref):
    return (got - ref).abs().max().item() / max(ref.abs().max().item(), 1e-30)


def _sd(shapes, dtype=torch.float32):
    return {"f." + k: v.to(dtype) for k, v in procedural.make_state_dict(cb.float_shapes(shapes)).items()}


@pytest.mark.parametrize("case", ["c64", "c256", "l2"])
def test_cobevt_oracle_vs_reference(golden_dir, case):
    g = cb.load_module_golden(golden_dir)[case]
    x, rl, pw = cb.case_inputs(case)
    assert torch.equal(rl, g["record_len"]) and torch.equal(pw, g["pairwise_t_matrix"])
    aff = cb.case_affine(pw)
    assert torch.equal(aff, g["affine"])
    with torch.no_grad():
        out = cb.cobevt_fusion(x, _sd(g["shapes"]), "f", g["args"], rl, aff)
    assert _rel_err(out[:, ::g["stride"]], g["out_s"]) <= 1e-5


def test_heter_model_baseline_cobevt_oracle_vs_reference(golden_dir):
    g = golden.load(os.path.join(golden_dir, "heter_model_baseline_cobevt_small.pt"))
    sd = procedural.make_state_dict(cb.float_shapes(g["shapes"]))
    with torch.no_grad():
        out = cb.heter_model_baseline(sd, g["args"], g["data"])
    for k in ("cls_preds", "reg_preds", "dir_preds"):
        assert _rel_err(out[k], g["out"][k]) <= 1e-5, k


def test_mirror_parameter_tables_and_index_match_reference(golden_dir):
    from heal_b200.models.fuse_modules.fusion_in_one import CoBEVT
    from heal_b200.models.heter_model_baseline import HeterModelBaseline
    for case, g in cb.load_module_golden(golden_dir).items():
        m = CoBEVT(copy.deepcopy(g["args"]))
        assert procedural.shapes_of(m) == g["shapes"], case
        for blk in m.layers:
            for att in (blk.window_attention, blk.grid_attention):
                idx = att.fn.relative_position_index
                assert idx.dtype == torch.int64 and torch.equal(idx, g["index"]), case
        assert torch.equal(cb.relative_position_index(g["args"]["agent_size"], 4), g["index"])
    gm = golden.load(os.path.join(golden_dir, "heter_model_baseline_cobevt_small.pt"))
    assert procedural.shapes_of(HeterModelBaseline(copy.deepcopy(gm["args"]))) == gm["shapes"]


def _token_pixels(H, W, L, w, grid):
    """(windows, n) row / column / agent of every token (l, w1, w2) of every window (x, y) by the kernel's address rule."""
    X, Y = H // w, W // w
    x, y, l, w1, w2 = torch.meshgrid(torch.arange(X), torch.arange(Y), torch.arange(L), torch.arange(w), torch.arange(w),
                                     indexing="ij")
    row = w1 * X + x if grid else x * w + w1
    col = w2 * Y + y if grid else y * w + w2
    return l.reshape(X * Y, -1), row.reshape(X * Y, -1), col.reshape(X * Y, -1)


def swap_attention_formulation(qkv, rl, L, w, grid, bias):
    """heal_swap_attention in plain torch: qkv (B*L, H, W, 3C) NHWC, bias (h, j, i) key-major -> (B*L, H, W, C)."""
    BL, H, W, C3 = qkv.shape
    C, h = C3 // 3, C3 // 96
    l, row, col = _token_pixels(H, W, L, w, grid)
    out = torch.empty(BL, H, W, C, dtype=qkv.dtype)
    for b, nb in enumerate(rl):
        tok = qkv[b * L + l, row, col]                                       # (windows, n, 3C)
        q, k, v = (tok[..., i * C:(i + 1) * C].reshape(tok.shape[0], tok.shape[1], h, 32).permute(0, 2, 1, 3) for i in range(3))
        nk = int(nb) * w * w                                                 # keys of the real agents only
        s = q @ k[:, :, :nk].transpose(-1, -2) + bias[:, :nk, :].transpose(-1, -2)
        o = s.softmax(-1) @ v[:, :, :nk]
        out[b * L + l, row, col] = o.permute(0, 2, 1, 3).reshape(tok.shape[0], tok.shape[1], C)
    return out


def cobevt_gpu_formulation(x, sd, p, args, record_len, aff):
    """What CoBEVT.forward_nhwc launches, in plain torch (NHWC residual stream of B*L slots)."""
    _, C, H, W = x.shape
    B, L = aff.shape[:2]
    w = args["window_size"]
    rl = [int(n) for n in record_len]
    X = torch.zeros(B * L, H, W, C, dtype=x.dtype)
    start = 0
    for b, n in enumerate(rl):
        X[b * L:b * L + n] = nets.warp_affine_simple(x[start:start + n], aff[b, 0, :n], (H, W)).permute(0, 2, 3, 1)
        start += n

    def ln(t, q):
        return F.layer_norm(t, (C,), sd[q + ".weight"], sd[q + ".bias"], 1e-5)

    def conv1x1(t, wt, bias=None):
        return F.conv2d(t.permute(0, 3, 1, 2), wt[:, :, None, None], bias).permute(0, 2, 3, 1)

    idx = cb.relative_position_index(L, w)
    for i in range(args["depth"]):
        for grid, kind in enumerate(("window", "grid")):
            pa, pf = f"{p}.layers.{i}.{kind}_attention", f"{p}.layers.{i}.{kind}_ffd"
            wq = sd[pa + ".fn.to_qkv.weight"].clone()
            wq[:C] *= 32 ** -0.5
            bias = sd[pa + ".fn.relative_position_bias_table.weight"][idx].permute(2, 1, 0)
            a = swap_attention_formulation(conv1x1(ln(X, pa + ".norm"), wq), rl, L, w, grid, bias)
            X = conv1x1(a, sd[pa + ".fn.to_out.0.weight"]) + X
            hdn = F.gelu(conv1x1(ln(X, pf + ".norm"), sd[pf + ".fn.net.0.weight"], sd[pf + ".fn.net.0.bias"]))
            X = conv1x1(hdn, sd[pf + ".fn.net.3.weight"], sd[pf + ".fn.net.3.bias"]) + X
    y = ln(X.reshape(B, L, H, W, C).mean(1), p + ".mlp_head.2")
    return conv1x1(y, sd[p + ".mlp_head.3.weight"], sd[p + ".mlp_head.3.bias"]).permute(0, 3, 1, 2)


@pytest.mark.parametrize("case", ["c64", "l2"])
def test_cobevt_gpu_formulation_is_exact_float64(golden_dir, case):
    g = cb.load_module_golden(golden_dir)[case]
    x, rl, pw = cb.case_inputs(case)
    aff = cb.case_affine(pw)
    sd = _sd(g["shapes"], torch.float64)
    with torch.no_grad():
        ref = cb.cobevt_fusion(x.double(), sd, "f", g["args"], rl, aff)
        got = cobevt_gpu_formulation(x.double(), sd, "f", g["args"], rl, aff)
    assert _rel_err(got, ref) <= 1e-10


def test_padded_slots_are_queries_and_count_in_the_mean(golden_dir):
    """Padded slots enter as zero maps but are queries: after the first block they carry non-zero values, which the head's
    mean over all L slots then includes."""
    g = cb.load_module_golden(golden_dir)["c64"]
    x, rl, pw = cb.case_inputs("c64")
    aff = cb.case_affine(pw)
    sd = _sd(g["shapes"], torch.float64)
    feats, mask = cb.regroup(x.double(), rl, 5)
    xx = torch.stack([cb.fusion_methods.warp_affine_simple(feats[b], aff[b, 0], (24, 40)) for b in range(2)])
    com = mask[:, None, None, None, :].expand(2, 24, 40, 1, 5)
    y = cb.swap_fusion_block_mask(xx, com, sd, "f.layers.0", g["args"])
    assert y[0, 3:].abs().max() > 0 and y[1, 2:].abs().max() > 0


def _module(args):
    from heal_b200.models.fuse_modules.fusion_in_one import CoBEVT
    return CoBEVT(copy.deepcopy(args)).eval()


def test_cobevt_shape_errors_name_the_reason():
    x, rl, pw = cb.case_inputs("c64")
    aff = cb.case_affine(pw)
    with pytest.raises(ValueError, match="agent_size"):
        _module(cb.cobevt_args(64, 1, 4, 128))(x, rl, aff)                    # L = 5 slots, agent_size 4
    with pytest.raises(ValueError, match="window_size"):
        _module(cb.cobevt_args(64, 1, 5, 128))(x[:, :, :22], rl, aff)       # 22 rows
    a = cb.cobevt_args(64, 1, 5, 128)
    a["dim_head"] = 16
    with pytest.raises(NotImplementedError, match="dim_head"):
        _module(a)(x, rl, aff)
    a = cb.cobevt_args(64, 1, 5, 128)
    a["window_size"] = 6                                                       # 5 * 36 = 180 tokens
    with pytest.raises(NotImplementedError, match="128 tokens"):
        _module(a)(x[..., :36], rl, aff)
    m = _module(cb.cobevt_args(64, 1, 5, 128)).train()
    with pytest.raises(NotImplementedError, match="inference"):
        m(x, rl, aff)


def test_heter_model_baseline_builds_cobevt():
    from heal_b200.models.fuse_modules.fusion_in_one import CoBEVT
    from heal_b200.models.heter_model_baseline import HeterModelBaseline
    m = HeterModelBaseline(copy.deepcopy(mg.baseline_cobevt_args()))
    assert isinstance(m.fusion_net, CoBEVT)
    args = mg.baseline_cobevt_args()
    args["fusion_method"] = "where2comm"
    with pytest.raises(NotImplementedError, match="cobevt"):
        HeterModelBaseline(args)


def test_library_exports_cobevt_kernels():
    import __graft_entry__
    __graft_entry__.build()
    from heal_b200 import _lib
    for s in ("heal_swap_attention", "heal_mean_layernorm"):
        assert hasattr(_lib.lib, s) and s in _lib.SIGNATURES
