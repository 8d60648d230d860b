"""ConvNeXt aligner (SURVEY.md 8f-3) on the GPU vs the golden produced by the UNMODIFIED reference AlignNet
(opencood/models/sub_modules/feature_alignnet.py:12-39 -> feature_alignnet_modules.py:299-360), and the ResNet-stem max pooling."""
import copy
import os

import pytest
import torch

from oracle import golden

from workloads import procedural

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _restore_precision():
    from heal_b200 import engine
    old = engine.PRECISION
    yield
    engine.set_precision(old)


@pytest.mark.parametrize("prec,tol", [("fp32", 1e-3), ("tc32", 1e-3), ("bf16", 2.5e-2)])
def test_convnext_aligner_vs_reference_golden(golden_dir, prec, tol):
    from heal_b200 import engine
    from heal_b200.models.sub_modules.feature_alignnet import AlignNet
    engine.set_precision(prec)
    g = golden.load(os.path.join(golden_dir, "convnext_aligner.pt"))
    m = AlignNet(copy.deepcopy(g["cfg"])).eval()
    assert procedural.shapes_of(m) == g["shapes"]                  # same state-dict keys and shapes as the reference module
    m.load_state_dict(procedural.make_state_dict(g["shapes"]), strict=True)
    m = m.cuda()
    with torch.no_grad():
        y = m(g["x"].cuda())
    err = (y.cpu() - g["y"]).abs().max().item()
    scale = max(g["y"].abs().max().item(), 1.0)
    print(f"convnext/{prec}: max|ref|={scale:.3f} err={err:.3e}")
    assert y.shape == g["y"].shape and err <= tol * scale


def test_dwconv_layernorm_kernel_vs_torch():
    from heal_b200 import ops
    gen = torch.Generator().manual_seed(3)
    for C, k in ((64, 7), (128, 3)):
        x = torch.randn(2, C, 19, 23, generator=gen)
        w = torch.randn(C, 1, k, k, generator=gen) * 0.2
        b = torch.randn(C, generator=gen) * 0.1
        lw, lb = torch.rand(C, generator=gen) + 0.5, torch.randn(C, generator=gen) * 0.1
        ref = torch.nn.functional.layer_norm(torch.nn.functional.conv2d(x, w, b, padding=k // 2, groups=C).permute(0, 2, 3, 1), (C,), lw, lb, 1e-6)
        out = ops.dwconv_layernorm(ops.to_act(x.cuda()), w.reshape(C, k * k).t().contiguous().cuda(), b.cuda(), k, lw.cuda(), lb.cuda(), 1e-6,
                                   out_fmt="f32")
        assert (out.t.cpu() - ref).abs().max().item() < 2e-5


def test_maxpool3x3s2_vs_torch():
    from heal_b200 import ops
    gen = torch.Generator().manual_seed(4)
    x = torch.randn(3, 64, 37, 50, generator=gen)
    ref = torch.nn.functional.max_pool2d(x, 3, 2, 1)
    for fmt in ("f32", "split"):
        out = ops.act_to_nchw(ops.maxpool3x3s2(ops.convert(ops.to_act(x.cuda()), fmt))).cpu()
        assert out.shape == ref.shape
        assert (out - ref).abs().max().item() < (1e-6 if fmt == "f32" else 1e-4)


def test_heter_pyramid_collab_with_convnext_aligner_vs_oracle():
    """HEAL stage-2 shape: a lidar modality whose features pass through the ConvNeXt aligner before the pyramid fusion."""
    import numpy as np
    from oracle import nets, make_golden
    from heal_b200 import engine
    from heal_b200.models.heter_pyramid_collab import HeterPyramidCollab
    engine.set_precision("tc32")
    args = make_golden.small_model_args()
    args["m1"]["aligner_args"] = {"core_method": "convnext", "spatial_align": False, "args": {"num_of_blocks": 3, "dim": 64}}
    m = HeterPyramidCollab(copy.deepcopy(args)).eval()
    sd = procedural.make_state_dict(procedural.shapes_of(m))
    m.load_state_dict(sd, strict=True)
    m = m.cuda()
    g = golden.load(os.path.join(os.path.dirname(__file__), "golden", "heter_pyramid_collab_small.pt"))
    data = g["data"]
    with torch.no_grad():
        ref = nets.heter_pyramid_collab(sd, args, copy.deepcopy(data))
        out = m({"inputs_m1": {k: v.cuda() for k, v in data["inputs_m1"].items()}, "agent_modality_list": data["agent_modality_list"],
                 "record_len": data["record_len"], "pairwise_t_matrix": data["pairwise_t_matrix"].cuda()})
    for k in ("cls_preds", "reg_preds", "dir_preds"):
        err = (out[k].cpu() - ref[k]).abs().max().item()
        assert err <= 1e-3 * max(ref[k].abs().max().item(), 1.0), (k, err)
