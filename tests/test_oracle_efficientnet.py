"""EfficientNet-B0 camera encoder without a GPU: the mirror's state-dict keys against a literal table, its topology against
torchvision's efficientnet_b0 (the one independent implementation available), its torch path against the golden made from the
unmodified reference CamEncode, and the configurations that now construct."""
import copy
import os

import pytest
import torch
import torch.nn.functional as F

from oracle import efficientnet as oe
from oracle import golden

# (kernel, stride, expand, Cin, Cout) of the 16 blocks, written out
BLOCKS = [(3, 1, 1, 32, 16), (3, 2, 6, 16, 24), (3, 1, 6, 24, 24), (5, 2, 6, 24, 40), (5, 1, 6, 40, 40), (3, 2, 6, 40, 80),
          (3, 1, 6, 80, 80), (3, 1, 6, 80, 80), (5, 1, 6, 80, 112), (5, 1, 6, 112, 112), (5, 1, 6, 112, 112), (5, 2, 6, 112, 192),
          (5, 1, 6, 192, 192), (5, 1, 6, 192, 192), (5, 1, 6, 192, 192), (3, 1, 6, 192, 320)]


def _bn_keys(prefix, c):
    return {f"{prefix}.weight": (c,), f"{prefix}.bias": (c,), f"{prefix}.running_mean": (c,), f"{prefix}.running_var": (c,),
            f"{prefix}.num_batches_tracked": ()}


def expected_trunk_shapes():
    """The state dict of efficientnet_pytorch's EfficientNet.from_name('efficientnet-b0')."""
    t = {"_conv_stem.weight": (32, 3, 3, 3), **_bn_keys("_bn0", 32)}
    for i, (k, s, e, cin, cout) in enumerate(BLOCKS):
        mid, sq, p = cin * e, max(1, cin // 4), f"_blocks.{i}"
        if e != 1:
            t[f"{p}._expand_conv.weight"] = (mid, cin, 1, 1)
            t.update(_bn_keys(f"{p}._bn0", mid))
        t[f"{p}._depthwise_conv.weight"] = (mid, 1, k, k)
        t.update(_bn_keys(f"{p}._bn1", mid))
        t[f"{p}._se_reduce.weight"], t[f"{p}._se_reduce.bias"] = (sq, mid, 1, 1), (sq,)
        t[f"{p}._se_expand.weight"], t[f"{p}._se_expand.bias"] = (mid, sq, 1, 1), (mid,)
        t[f"{p}._project_conv.weight"] = (cout, mid, 1, 1)
        t.update(_bn_keys(f"{p}._bn2", cout))
    t["_conv_head.weight"] = (1280, 320, 1, 1)
    t.update(_bn_keys("_bn1", 1280))
    t["_fc.weight"], t["_fc.bias"] = (1000, 1280), (1000,)
    return t


def _cam_encode(ds=8, D=oe.TRUNK_D, C=oe.TRUNK_C):
    from heal_b200.models.heter_encoders import CamEncode
    return CamEncode(D, C, ds, oe.TRUNK_DDISCR, "LID", False, False).eval()


def test_state_dict_keys_match_the_package_table_the_oracle_and_the_golden(golden_dir):
    from heal_b200.models.sub_modules.efficientnet_b0 import EfficientNetB0
    want = expected_trunk_shapes()
    trunk = EfficientNetB0()
    got = {k: tuple(v.shape) for k, v in trunk.state_dict().items()}
    assert got == want
    assert {k: tuple(v.shape) for k, v in oe.EfficientNet().state_dict().items()} == want
    assert sum(p.numel() for p in trunk.parameters()) == 5288548
    import torchvision
    assert sum(p.numel() for p in torchvision.models.efficientnet_b0(weights=None).parameters()) == 5288548
    g = golden.load(os.path.join(golden_dir, "efficientnet_trunk.pt"))
    for ds in (8, 16):
        m = _cam_encode(ds)
        shapes = {k: tuple(v.shape) for k, v in m.state_dict().items()}
        assert shapes == g["cases"][ds]["shapes"]                      # the unmodified reference CamEncode's keys
        assert {"trunk._blocks.15._project_conv.weight", "up1.conv.0.weight", "up1.conv.4.running_var", "depth_head.bias"} <= set(shapes)
        assert ("up2.conv.4.running_var" in shapes) == (ds == 8) and hasattr(m, "up2") == (ds == 8)
        assert shapes["up1.conv.0.weight"] == (512, 432, 3, 3)
    assert not any("cache" in k or "_pk_" in k for k in shapes)


def _torchvision_twin(trunk):
    """torchvision's efficientnet_b0 carrying `trunk`'s weights, with eps 1e-3 and the static asymmetric pads on the stride-2 convs."""
    import torchvision
    tv = torchvision.models.efficientnet_b0(weights=None).eval()
    feats = tv.features

    def copy_bn(dst, src):
        dst.load_state_dict(src.state_dict())

    feats[0][0].weight.data.copy_(trunk._conv_stem.weight)
    copy_bn(feats[0][1], trunk._bn0)
    tv_blocks = [b for stage in feats[1:8] for b in stage]
    assert len(tv_blocks) == 16
    for tb, b in zip(tv_blocks, trunk._blocks):
        layers = list(tb.block)
        if hasattr(b, "_expand_conv"):
            exp = layers.pop(0)
            exp[0].weight.data.copy_(b._expand_conv.weight)
            copy_bn(exp[1], b._bn0)
        dw, se, proj = layers
        dw[0].weight.data.copy_(b._depthwise_conv.weight)
        copy_bn(dw[1], b._bn1)
        se.fc1.load_state_dict(b._se_reduce.state_dict())
        se.fc2.load_state_dict(b._se_expand.state_dict())
        proj[0].weight.data.copy_(b._project_conv.weight)
        copy_bn(proj[1], b._bn2)
    for mod in tv.modules():
        if isinstance(mod, torch.nn.BatchNorm2d):
            mod.eps = 1e-3
        if isinstance(mod, torch.nn.Conv2d) and mod.stride == (2, 2):
            k = mod.kernel_size[0]
            pad = {3: (0, 1, 0, 1), 5: (1, 2, 1, 2)}[k]
            mod.padding = (0, 0)
            mod.register_forward_pre_hook(lambda m, inp, pad=pad: (F.pad(inp[0], pad),))
    return tv


def test_topology_equals_torchvision_efficientnet_b0():
    """Same weights in torchvision's efficientnet_b0 (its own MBConv, SE and block order; only eps and the stride-2 pads adjusted)
    give the same endpoints: catches a wrong expand ratio, SE width, kernel size, stride or skip rule."""
    from heal_b200.models.sub_modules.efficientnet_b0 import EfficientNetB0
    trunk = EfficientNetB0().eval()
    trunk.load_state_dict(oe.state_dict_of({k: tuple(v.shape) for k, v in trunk.state_dict().items()}), strict=True)
    tv = _torchvision_twin(trunk)
    x = oe.trunk_images()[:, :3]
    with torch.no_grad():
        ep = trunk.endpoints(x)
        y, taps = x, {}
        for i, stage in enumerate(tv.features[:8]):
            y = stage(y)
            taps[i] = y
        oracle_trunk = oe.EfficientNet().eval()
        oracle_trunk.load_state_dict(trunk.state_dict(), strict=True)
        z = oracle_trunk._swish(oracle_trunk._bn0(oracle_trunk._conv_stem(x)))
        for blk in oracle_trunk._blocks:
            z = blk(z)
    assert [tuple(ep[f"reduction_{i}"].shape[1:]) for i in range(1, 6)] == [(16, 32, 48), (24, 16, 24), (40, 8, 12), (112, 4, 6), (320, 2, 3)]
    for name, stage in (("reduction_1", 1), ("reduction_2", 2), ("reduction_3", 3), ("reduction_4", 5), ("reduction_5", 7)):
        torch.testing.assert_close(ep[name], taps[stage], rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(ep["reduction_5"], z, rtol=1e-5, atol=1e-5)         # the oracle's restatement agrees too


@pytest.mark.parametrize("ds", [8, 16])
def test_torch_path_equals_reference_cam_encode_golden(golden_dir, ds):
    g = golden.load(os.path.join(golden_dir, "efficientnet_trunk.pt"))
    case = g["cases"][ds]
    m = _cam_encode(ds)
    m.load_state_dict(oe.state_dict_of(case["shapes"]), strict=True)
    x = oe.trunk_images()
    with torch.no_grad():
        ep = m.trunk.endpoints(x[:, :3])
        dl, ft = m.heads(x)
        dl3, ft3 = m.heads(x[:, :3])
    assert torch.equal(dl, dl3) and torch.equal(ft, ft3)
    for k, v in case["endpoints"].items():
        assert (ep[k] - v).abs().max().item() <= 1e-5 * max(v.abs().max().item(), 1.0), k
    for got, ref in ((dl, case["depth_logits"]), (ft, case["feat"])):
        assert got.shape == ref.shape == (2, ref.shape[1], 64 // ds, 96 // ds)
        assert (got - ref).abs().max().item() <= 1e-5 * ref.abs().max().item()


def test_lift_splat_shoot_selects_the_encoder_and_rejects_what_it_cannot_run():
    from heal_b200.models.heter_encoders import CamEncode, CamEncode_Resnet101, LiftSplatShoot
    cfg = oe.lss_cfg()
    m = LiftSplatShoot(copy.deepcopy(cfg))
    assert isinstance(m.camencode, CamEncode) and hasattr(m.camencode, "up2")
    assert isinstance(LiftSplatShoot(dict(copy.deepcopy(cfg), camera_encoder="Resnet101")).camencode, CamEncode_Resnet101)
    m16 = LiftSplatShoot(dict(copy.deepcopy(cfg), img_downsample=16))
    assert not hasattr(m16.camencode, "up2") and m16.frustum.shape[1:3] == (4, 8)
    with pytest.raises(NotImplementedError, match="camera_encoder"):
        LiftSplatShoot(dict(copy.deepcopy(cfg), camera_encoder="Resnet50"))
    with pytest.raises(NotImplementedError, match="use_depth_gt"):
        LiftSplatShoot(dict(copy.deepcopy(cfg), use_depth_gt=True))
    enc = m.camencode.eval()
    with pytest.raises(ValueError, match="48"):
        enc.heads(torch.zeros(1, 3, 48, 64))                           # 48 -> 6, 3, 1: the /32 map upsampled is 2, not 3
    with pytest.raises(ValueError, match="width 72"):
        enc.heads_nhwc(torch.zeros(1, 3, 64, 72))                      # raised before any kernel is launched
    m.train()
    dd = {"inputs_m2": oe.cam_inputs()}
    with pytest.raises(NotImplementedError, match="inference"):
        m.forward_act(dd, "m2")


def test_checkpoint_keys_load_strictly_into_the_heal_m2_agent(golden_dir):
    """The m2 blocks of HEAL/stage1/m2_pyramid.yaml and HEAL/final_infer/m1m2m3m4.yaml (scaled down) construct, and a state dict
    with the reference model's keys (efficientnet_pytorch names under encoder_m2.camencode.trunk) loads with strict=True."""
    from heal_b200.models.heter_pyramid_collab import HeterPyramidCollab
    g = golden.load(os.path.join(golden_dir, "heter_pyramid_collab_effnet_small.pt"))
    m = HeterPyramidCollab(copy.deepcopy(g["args"])).eval()
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == g["shapes"]
    m.load_state_dict(oe.state_dict_of(g["shapes"]), strict=True)
    assert "encoder_m2.camencode.trunk._blocks.3._se_reduce.bias" in g["shapes"]


def test_heterogeneous_coalign_m2_block_constructs():
    """m2 of opv2v/MoreModality/4_modality_end2end_training/m1m2m3m4_coalign.yaml (Lift-Splat-Shoot, EfficientNet) beside a
    PointPillar m1 in HeterModelBaselineMs, with `att: {feat_dim: [...]}` supplied."""
    from heal_b200.models.heter_model_baseline_ms import HeterModelBaselineMs
    from oracle import coalign
    args = coalign.hetero_args()
    args["m2"] = args.pop("m4")
    args["m2"]["encoder_args"]["camera_encoder"] = "EfficientNet"
    m = HeterModelBaselineMs(copy.deepcopy(args))
    assert any(k.startswith("encoder_m2.camencode.trunk._blocks.15.") for k in m.state_dict())


def test_library_exports_mbconv_kernels():
    import __graft_entry__
    __graft_entry__.build()
    from heal_b200 import _lib
    for s in ("heal_stem_conv_swish", "heal_dwconv_bn_swish", "heal_se_gate", "heal_pwconv", "heal_upsample2x_concat"):
        assert hasattr(_lib.lib, s) and s in _lib.SIGNATURES
