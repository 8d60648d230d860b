"""HeterModelBaselineMs (`core_method: heter_model_baseline_ms`, the CoAlign configs) on the CPU: the oracle restatement against the
reference's own model (goldens), the mirror's state-dict table against the reference's, and the errors the mirror raises at
construction."""
import copy

import pytest
import torch

from oracle import coalign, procedural


def _rel_err(got, ref):
    return (got - ref).abs().max().item() / max(ref.abs().max().item(), 1e-30)


@pytest.mark.parametrize("name", coalign.GOLDENS)
def test_oracle_vs_reference_golden(golden_dir, name):
    g = coalign.load_golden(golden_dir, name)
    sd = procedural.make_state_dict(g["shapes"])
    with torch.no_grad():
        out = coalign.heter_model_baseline_ms(sd, g["args"], copy.deepcopy(g["data"]))
    assert set(out) == set(g["out"])
    for k, ref in g["out"].items():
        assert out[k].shape == ref.shape, k
        assert _rel_err(out[k], ref) <= 1e-5, (k, _rel_err(out[k], ref))


def test_hetero_golden_crops_the_camera_map():
    """The camera grid (+-19.2 m) is wider than the lidar range (+-12.8 m): its 48 x 48 level-0 map is cropped to 32 x 32."""
    a = coalign.hetero_args()
    g = a["m4"]["camera_mask_args"]["grid_conf"]
    n = round((g["xbound"][1] - g["xbound"][0]) / g["xbound"][2]) // 2
    assert n == 48 and int(n * a["lidar_range"][3] / g["xbound"][1]) == 32


@pytest.mark.parametrize("name", coalign.GOLDENS)
def test_mirror_state_dict_matches_reference(golden_dir, name):
    """Same keys and shapes as the reference (the fusion backbone's never-run layer0 included); strict loading succeeds."""
    from heal_b200.models.heter_model_baseline_ms import HeterModelBaselineMs
    g = coalign.load_golden(golden_dir, name)
    m = HeterModelBaselineMs(copy.deepcopy(g["args"]))
    assert procedural.shapes_of(m) == g["shapes"]
    assert any(k.startswith("backbone.resnet.layer0.") for k in g["shapes"])
    m.load_state_dict(procedural.make_state_dict(g["shapes"]), strict=True)


@pytest.mark.parametrize("method", ["v2vnet", "cobevt", "v2xvit", "disconet", "pyramid"])
def test_unbuilt_fusion_method_raises(method):
    from heal_b200.models.heter_model_baseline_ms import HeterModelBaselineMs
    args = coalign.coalign_args("max")
    args["fusion_method"] = method
    with pytest.raises(NotImplementedError, match="att, max"):
        HeterModelBaselineMs(args)


@pytest.mark.parametrize("feat_dim", [[64, 128, 128], [128, 128, 256], 256])
def test_feat_dim_mismatch_raises(feat_dim):
    """The kernel scales by 1/sqrt(C); a feat_dim other than the level's channel count cannot be matched."""
    from heal_b200.models.heter_model_baseline_ms import HeterModelBaselineMs
    args = coalign.coalign_args("att")
    args["att"]["feat_dim"] = feat_dim
    with pytest.raises(ValueError):
        HeterModelBaselineMs(args)


@pytest.mark.parametrize("feat_dim", [[64, 128], [64, 128, 256, 256]])
def test_feat_dim_length_mismatch_raises(feat_dim):
    from heal_b200.models.heter_model_baseline_ms import HeterModelBaselineMs
    args = coalign.coalign_args("att")
    args["att"]["feat_dim"] = feat_dim
    with pytest.raises(ValueError, match="entries"):
        HeterModelBaselineMs(args)
