"""MaxFusion / V2VNetFusion (fusion_method max / v2vnet) on the CPU: the oracle against the reference's own modules (goldens),
the mirror modules' parameter tables, and the GPU formulation of V2VNet (K-split message conv, zero-hidden GRU with only its
live weight blocks, node-0-only last iteration) restated in float64 against the literal oracle."""
import copy
import os

import pytest
import torch
import torch.nn.functional as F

from oracle import fusion_methods as fm, golden, make_golden_fusion_methods as mg, nets, procedural


def _load(golden_dir, name):
    return golden.load(os.path.join(golden_dir, name))


def _rel_err(got, ref):
    return (got - ref).abs().max().item() / max(ref.abs().max().item(), 1e-30)


def test_max_fusion_oracle_vs_reference(golden_dir):
    g = fm.load_module_golden(golden_dir)
    aff = nets.normalize_pairwise_tfm(g["pairwise_t_matrix"], g["H"], g["W"], 1)
    assert torch.equal(aff, g["affine"])
    out = fm.max_fusion(g["x"], g["record_len"], aff)
    assert _rel_err(out[:, ::2], g["max_s"]) <= 1e-5


@pytest.mark.parametrize("variant", ["avg_gru1", "max_gru1", "avg_gru0", "max_gru0"])
def test_v2vnet_oracle_vs_reference(golden_dir, variant):
    g = fm.load_module_golden(golden_dir)
    v = g["v2vnet"][variant]
    sd = {"f." + k: t for k, t in procedural.make_state_dict(v["shapes"]).items()}
    with torch.no_grad():
        out = fm.v2vnet_fusion(g["x"], sd, "f", v["args"], g["record_len"], g["affine"])
    assert _rel_err(out[:, ::4], v["out_s"]) <= 1e-5


@pytest.mark.parametrize("method", ["max", "v2vnet"])
def test_heter_model_baseline_oracle_vs_reference(golden_dir, method):
    g = _load(golden_dir, f"heter_model_baseline_{method}_small.pt")
    sd = procedural.make_state_dict(g["shapes"])
    with torch.no_grad():
        out = fm.heter_model_baseline(sd, g["args"], g["data"])
    for k in ("cls_preds", "reg_preds", "dir_preds"):
        assert _rel_err(out[k], g["out"][k]) <= 1e-5, k


def test_mirror_parameter_tables_match_reference(golden_dir):
    from heal_b200.models.fuse_modules.fusion_in_one import MaxFusion, V2VNetFusion
    from heal_b200.models.heter_model_baseline import HeterModelBaseline
    g = fm.load_module_golden(golden_dir)
    for v in g["v2vnet"].values():
        assert procedural.shapes_of(V2VNetFusion(copy.deepcopy(v["args"]))) == v["shapes"]
    assert procedural.shapes_of(MaxFusion()) == {}
    for method in ("max", "v2vnet"):
        gm = _load(golden_dir, f"heter_model_baseline_{method}_small.pt")
        assert procedural.shapes_of(HeterModelBaseline(copy.deepcopy(gm["args"]))) == gm["shapes"]


def test_unbuilt_fusion_methods_name_the_reason():
    from heal_b200.models.heter_model_baseline import HeterModelBaseline
    args = mg.baseline_fusion_args("max")
    args["fusion_method"] = "disconet"
    with pytest.raises(NotImplementedError, match="disco_fuse"):
        HeterModelBaseline(copy.deepcopy(args))
    args["fusion_method"] = "v2xvit"
    with pytest.raises(NotImplementedError, match="scope"):
        HeterModelBaseline(copy.deepcopy(args))


def test_conv_gru_size_mismatch_raises():
    from heal_b200.models.fuse_modules.fusion_in_one import V2VNetFusion
    m = V2VNetFusion(mg.v2vnet_args(64, 16, 16)).eval()
    rl, pw = mg.fusion_scenes()
    aff = nets.normalize_pairwise_tfm(pw, 9.6, 16.0, 1)
    with pytest.raises(ValueError, match=r"\(16, 16\).*\(24, 40\)"):
        m(torch.zeros(5, 64, 24, 40), rl, aff)
    with pytest.raises(ValueError):
        fm.v2vnet_fusion(torch.zeros(5, 64, 24, 40), {}, "f", mg.v2vnet_args(64, 16, 16), rl, aff)


def v2v_gpu_formulation(x, sd, p, args, record_len, aff):
    """What V2VNetFusion.forward_nhwc launches, in plain torch: Q = W[:, :C] * warp(x_j) per pair, P = W[:, C:] * x_i + b per
    node, msg = mask * (Q + P), one stacked GRU conv (update-gate rows of conv_gates over conv_can, input columns only) and
    sigmoid(z) * tanh(c), node 0 alone in the last iteration, mlp as a 1x1 conv."""
    _, C, H, W = x.shape
    wm, bm = sd[p + ".msg_cnn.weight"], sd[p + ".msg_cnn.bias"]
    cell = p + ".conv_gru.cell_list.0"
    wg = torch.cat([sd[cell + ".conv_gates.weight"][C:2 * C, :2 * C], sd[cell + ".conv_can.weight"][:, :2 * C]])
    bg = torch.cat([sd[cell + ".conv_gates.bias"][C:2 * C], sd[cell + ".conv_can.bias"]])
    rl = [int(n) for n in record_len]
    feats = list(torch.split(x, rl))
    T = args["num_iteration"]
    for it in range(T):
        last = it == T - 1
        new = []
        for b, n in enumerate(rl):
            xb = feats[b]
            P = F.conv2d(xb, wm[:, C:], bm, padding=1)
            outs = []
            for i in range(1 if last else n):
                th = aff[b, i, :n]
                Q = F.conv2d(nets.warp_affine_simple(xb, th, (H, W)), wm[:, :C], None, padding=1)
                mask = nets.warp_affine_simple(torch.ones(n, 1, H, W, dtype=x.dtype), th, (H, W))
                msg = mask * (Q + P[i])
                agg = msg.mean(0) if args["agg_operator"] == "avg" else msg.max(0)[0]
                if args["gru_flag"]:
                    z = F.conv2d(torch.cat([xb[i], agg])[None], wg, bg, padding=1)[0]
                    outs.append(torch.sigmoid(z[:C]) * torch.tanh(z[C:]))
                else:
                    outs.append(xb[i] + agg)
            new.append(torch.stack(outs))
        feats = new
    out = torch.stack([f[0] for f in feats])
    return F.conv2d(out, sd[p + ".mlp.weight"][:, :, None, None], sd[p + ".mlp.bias"])


@pytest.mark.parametrize("agg,gru", mg.V2V_VARIANTS)
@pytest.mark.parametrize("scenes", ["3+2", "1"])
def test_v2vnet_gpu_formulation_is_exact_float64(golden_dir, agg, gru, scenes):
    g = fm.load_module_golden(golden_dir)
    x, rl, aff = g["x"].double(), g["record_len"], g["affine"]
    if scenes == "1":
        x, rl, aff = x[3:4], torch.tensor([1]), aff[1:2]
    args = mg.v2vnet_args(64, 24, 40, agg, gru)
    sd = {"f." + k: v.double() for k, v in procedural.make_state_dict(g["v2vnet"]["avg_gru1"]["shapes"]).items()}
    with torch.no_grad():
        ref = fm.v2vnet_fusion(x, sd, "f", args, rl, aff)
        got = v2v_gpu_formulation(x, sd, "f", args, rl, aff)
    assert _rel_err(got, ref) <= 1e-10


def test_v2vnet_dead_gru_weights_do_not_matter(golden_dir):
    """With the zero hidden state, the reset-gate rows, the reset-gate bias and the hidden-state columns of both GRU convs
    never reach the output."""
    g = fm.load_module_golden(golden_dir)
    v = g["v2vnet"]["avg_gru1"]
    sd = {"f." + k: t for k, t in procedural.make_state_dict(v["shapes"]).items()}
    C = 64
    with torch.no_grad():
        ref = fm.v2vnet_fusion(g["x"], sd, "f", v["args"], g["record_len"], g["affine"])
        sd2 = {k: t.clone() for k, t in sd.items()}
        cell = "f.conv_gru.cell_list.0"
        sd2[cell + ".conv_gates.weight"][:C] += 1.0
        sd2[cell + ".conv_gates.bias"][:C] -= 3.0
        sd2[cell + ".conv_gates.weight"][:, 2 * C:] += 1.0
        sd2[cell + ".conv_can.weight"][:, 2 * C:] += 1.0
        out = fm.v2vnet_fusion(g["x"], sd2, "f", v["args"], g["record_len"], g["affine"])
    assert (out - ref).abs().max().item() == 0.0


def test_library_exports_fusion_method_kernels():
    import __graft_entry__
    __graft_entry__.build()
    from heal_b200 import _lib
    for s in ("heal_max_fuse", "heal_warp_affine", "heal_v2v_aggregate", "heal_gru_gate"):
        assert hasattr(_lib.lib, s) and s in _lib.SIGNATURES


def test_device_aware_warp_equals_oracle_warp(golden_dir):
    """fusion_methods.warp_affine_simple (any device) is oracle/nets.py's restatement, which tests/test_oracle_golden.py pins
    to the reference."""
    g = fm.load_module_golden(golden_dir)
    for b in range(2):
        th = g["affine"][b, 0]
        assert torch.equal(fm.warp_affine_simple(g["x"], th, (24, 40)), nets.warp_affine_simple(g["x"], th, (24, 40)))
