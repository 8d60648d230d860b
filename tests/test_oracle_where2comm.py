"""Where2commFusion / Who2comFusion (fusion_method where2comm / who2com) on the CPU: the oracle against the reference's own
modules (goldens), the project-then-sample form of Where2comm's k | v projection against the literal sample-then-project in
float64, the mirrors' parameter tables, HeterModelBaseline's constructor errors and the new library export."""
import copy
import os

import pytest
import torch

from oracle import fusion_methods as fm, golden, make_golden_where2comm as mg, nets, procedural, where2comm as w2c


def _rel_err(got, ref):
    return (got - ref).abs().max().item() / max(ref.abs().max().item(), 1e-30)


def _sd(shapes, dtype=torch.float32):
    return {"f." + k: v.to(dtype) for k, v in procedural.make_state_dict(shapes).items()}


def test_golden_scenes_pin_the_ego_transform(golden_dir):
    g = w2c.load_module_golden(golden_dir)
    rl, pw = mg.fusion_scenes()
    assert torch.equal(rl, g["record_len"]) and torch.equal(pw, g["pairwise_t_matrix"])
    assert torch.equal(nets.normalize_pairwise_tfm(pw, 9.6, 16.0, 1), g["affine"])
    eye = torch.tensor([[1.0, 0, 0], [0, 1.0, 0]], dtype=g["affine"].dtype)
    assert torch.equal(g["affine"][0, 0, 0], eye) and not torch.allclose(g["affine"][2, 0, 0], eye)


@pytest.mark.parametrize("method", mg.METHODS)
def test_fusion_oracle_vs_reference(golden_dir, method):
    g = w2c.load_module_golden(golden_dir)
    with torch.no_grad():
        out = w2c.FUSIONS[method](g["x"], _sd(g[method]["shapes"]), "f", g["record_len"], g["affine"])
    assert out.shape == (3, 256, 24, 40)
    assert _rel_err(out[:, ::16], g[method]["out_s"]) <= 1e-5


@pytest.mark.parametrize("method", mg.METHODS)
def test_heter_model_baseline_oracle_vs_reference(golden_dir, method):
    g = golden.load(os.path.join(golden_dir, f"heter_model_baseline_{method}_small.pt"))
    with torch.no_grad():
        out = w2c.heter_model_baseline(procedural.make_state_dict(g["shapes"]), g["args"], g["data"])
    for k in ("cls_preds", "reg_preds", "dir_preds"):
        assert _rel_err(out[k], g["out"][k]) <= 1e-5, k


def _identity_scene():
    """Two scenes in float64: a sub-pixel shift, a rotated agent with a border band, and an agent entirely out of view."""
    th = torch.zeros(2, 5, 5, 2, 3, dtype=torch.float64)
    th[..., 0, 0] = th[..., 1, 1] = 1.0
    th[0, 0, 1, :, 2] = torch.tensor([0.013, -0.021], dtype=torch.float64)          # sub-pixel
    a = torch.tensor(0.6, dtype=torch.float64)
    th[0, 0, 2] = torch.tensor([[a.cos(), -a.sin(), 0.3], [a.sin(), a.cos(), -0.2]], dtype=torch.float64)
    th[0, 0, 3, :, 2] = torch.tensor([3.5, -2.7], dtype=torch.float64)               # out of view
    th[1, 0, 0, :, 2] = torch.tensor([0.11, 0.05], dtype=torch.float64)              # ego-to-ego not the identity
    th[1, 0, 1, :, 2] = torch.tensor([-0.4, 0.5], dtype=torch.float64)
    x = torch.randn(6, 256, 12, 20, generator=torch.Generator().manual_seed(5), dtype=torch.float64)
    return x, torch.tensor([4, 2]), th


def test_projection_commutes_with_the_warp_float64():
    """warp(W x) + b == W warp(x) + b per pixel, on border pixels (fractional tap weights) and fully out-of-view ones (= b)."""
    x, _, th = _identity_scene()
    g = torch.Generator().manual_seed(8)
    w = torch.randn(512, 256, generator=g, dtype=torch.float64) / 16
    b = torch.randn(512, generator=g, dtype=torch.float64)
    t = th[0, 0, :4]
    lit = torch.einsum("oc,nchw->nohw", w, fm.warp_affine_simple(x[:4], t, (12, 20))) + b[:, None, None]
    proj = fm.warp_affine_simple(torch.einsum("oc,nchw->nohw", w, x[:4]), t, (12, 20)) + b[:, None, None]
    assert (proj - lit).abs().max().item() <= 1e-12 * max(lit.abs().max().item(), 1.0)
    assert torch.equal(proj[3], b[:, None, None].expand(512, 12, 20))                  # out of view: exactly the bias
    ones = fm.warp_affine_simple(torch.ones(4, 1, 12, 20, dtype=torch.float64), t, (12, 20))
    border = (ones > 1e-3) & (ones < 1 - 1e-3)
    assert border[2].any() and border[1].any()                                          # the check covers partial taps


def test_where2comm_projected_form_equals_literal_float64(golden_dir):
    g = w2c.load_module_golden(golden_dir)
    sd = _sd(g["where2comm"]["shapes"], torch.float64)
    x, rl, th = _identity_scene()
    with torch.no_grad():
        for xs, rls, ths in ((x, rl, th), (g["x"].double(), g["record_len"], g["affine"])):
            ref = w2c.where2comm_fusion(xs, sd, "f", rls, ths)
            got = w2c.where2comm_fusion_projected(xs, sd, "f", rls, ths)
            assert _rel_err(got, ref) <= 1e-12


def test_where2comm_residual_is_the_warped_ego_and_who2com_decodes_the_unwarped_one(golden_dir):
    """Scene 2 of the golden has a non-identity affine[2, 0, 0]: replacing the warped ego with the unwarped one (Where2comm) or
    the reverse (Who2com) moves the output well outside the oracle's tolerance."""
    g = w2c.load_module_golden(golden_dir)
    x, rl, aff = g["x"], g["record_len"], g["affine"].clone()
    aff_id = aff.clone()
    aff_id[2, 0, 0] = torch.tensor([[1.0, 0, 0], [0, 1.0, 0]], dtype=aff.dtype)
    for method in mg.METHODS:
        with torch.no_grad():
            out = w2c.FUSIONS[method](x, _sd(g[method]["shapes"]), "f", rl, aff_id)
        assert _rel_err(out[:2, ::16], g[method]["out_s"][:2]) <= 1e-5
        assert _rel_err(out[2:, ::16], g[method]["out_s"][2:]) > 1e-2


def test_mirror_parameter_tables_match_reference(golden_dir):
    from heal_b200.models.fuse_modules.fusion_in_one import Where2commFusion, Who2comFusion
    from heal_b200.models.heter_model_baseline import HeterModelBaseline
    g = w2c.load_module_golden(golden_dir)
    assert procedural.shapes_of(Where2commFusion(256)) == g["where2comm"]["shapes"]
    assert procedural.shapes_of(Who2comFusion(256)) == g["who2com"]["shapes"]
    assert g["where2comm"]["shapes"]["mha_fusion.attn.in_proj_weight"] == (768, 256)
    assert g["who2com"]["shapes"]["decode_layer.weight"] == (256, 512, 3, 3)
    for method, cls in zip(mg.METHODS, (Where2commFusion, Who2comFusion)):
        gm = golden.load(os.path.join(golden_dir, f"heter_model_baseline_{method}_small.pt"))
        m = HeterModelBaseline(copy.deepcopy(gm["args"]))
        assert isinstance(m.fusion_net, cls)
        assert procedural.shapes_of(m) == gm["shapes"]
        res = m.load_state_dict(procedural.make_state_dict(gm["shapes"]), strict=True)
        assert not res.missing_keys and not res.unexpected_keys


@pytest.mark.parametrize("method", mg.METHODS)
def test_constructor_errors_name_the_reason(method):
    from heal_b200.models.heter_model_baseline import HeterModelBaseline
    args = mg.baseline_args(method)
    del args[method]
    with pytest.raises(NotImplementedError, match=f"`{method}:` block.*where2comm, who2com"):
        HeterModelBaseline(copy.deepcopy(args))
    for bad in ("256", 256.0, True, {"feat_dim": 256}, 128):
        args[method] = bad
        with pytest.raises(NotImplementedError, match="heal_b200 hot-path scope"):
            HeterModelBaseline(copy.deepcopy(args))


def test_where2comm_mirror_rejects_unbuilt_shapes():
    from heal_b200.models.fuse_modules.fusion_in_one import Where2commFusion
    with pytest.raises(NotImplementedError, match="256 channels in 8 heads"):
        Where2commFusion(128).eval()(torch.zeros(2, 128, 4, 4), torch.tensor([2]), torch.zeros(1, 2, 2, 2, 3))
    with pytest.raises(ValueError, match="feature_dims is 256"):
        Where2commFusion(256).eval()(torch.zeros(2, 64, 4, 4), torch.tensor([2]), torch.zeros(1, 2, 2, 2, 3))
    with pytest.raises(NotImplementedError, match="inference"):
        Where2commFusion(256).train()(torch.zeros(2, 256, 4, 4), torch.tensor([2]), torch.zeros(1, 2, 2, 2, 3))


def test_library_exports_ego_mha():
    import __graft_entry__
    __graft_entry__.build()
    from heal_b200 import _lib, ops
    assert hasattr(_lib.lib, "heal_ego_mha") and "heal_ego_mha" in _lib.SIGNATURES
    assert hasattr(ops.ego_mha, "device_arg")
    assert _lib.lib.heal_abi_version() == 3
