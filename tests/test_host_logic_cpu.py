"""CPU-only host logic: pre-processor registry entry, the opencood aliasing used for the drop-in, state-dict key parity
with the reference's checkpoints (key table recorded in the goldens), launch-free module construction."""
import copy
import os

import numpy as np
import torch

from oracle import golden

from oracle import make_golden


def test_gpu_voxel_preprocessor_contract():
    from heal_b200.data_utils.pre_processor import build_preprocessor
    cfg = {"core_method": "GpuVoxelPreprocessor", "cav_lidar_range": [-102.4, -102.4, -3, 102.4, 102.4, 1],
           "args": {"voxel_size": [0.4, 0.4, 4], "max_points_per_voxel": 32, "max_voxel_train": 32000, "max_voxel_test": 70000}}
    pp = build_preprocessor(cfg, train=False)
    assert pp.max_voxels == 70000 and list(pp.grid_size) == [512, 512, 1]
    a = pp.preprocess(np.random.rand(10, 4).astype(np.float32))
    b = pp.preprocess(np.random.rand(7, 5).astype(np.float32))
    out = pp.collate_batch([a, b])
    assert out["points"].shape == (17, 4) and out["agent_offsets"].tolist() == [0, 10, 17]
    out2 = pp.collate_batch({"points": [a["points"], b["points"]]})
    assert torch.equal(out2["points"], out["points"])
    assert "filter_points" not in out
    # filter_on_gpu: the shuffle permutation is drawn from numpy's global RNG exactly where shuffle_points would draw it
    cfg["args"]["filter_on_gpu"] = True
    pp = build_preprocessor(cfg, train=False)
    np.random.seed(11)
    a2, b2 = pp.preprocess(a["points"]), pp.preprocess(b["points"])
    np.random.seed(11)
    pa, pb = np.random.permutation(10), np.random.permutation(7)
    out3 = pp.collate_batch([a2, b2])
    assert out3["filter_points"] is True and out3["remove_ego"] is True
    assert out3["shuffle_perm"].tolist() == list(pa) + [int(x) + 10 for x in pb]


def test_state_dict_keys_match_reference(golden_dir):
    """The goldens record the UNMODIFIED reference models' {key: shape} tables; the mirrors must reproduce them exactly."""
    from heal_b200.models.heter_pyramid_collab import HeterPyramidCollab
    from heal_b200.models.heter_model_baseline import HeterModelBaseline
    g = golden.load(os.path.join(golden_dir, "heter_pyramid_collab_small.pt"))
    m = HeterPyramidCollab(copy.deepcopy(g["args"]))
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == {k: tuple(v) for k, v in g["shapes"].items()}
    g = golden.load(os.path.join(golden_dir, "heter_model_baseline_att_small.pt"))
    m = HeterModelBaseline(copy.deepcopy(g["args"]))
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == {k: tuple(v) for k, v in g["shapes"].items()}
    g = golden.load(os.path.join(golden_dir, "base_bev_backbone_small.pt"))
    from heal_b200.models.sub_modules.base_bev_backbone import BaseBEVBackbone
    m = BaseBEVBackbone(copy.deepcopy(g["cfg"]), 64)
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == {k: tuple(v) for k, v in g["shapes"].items()}


def test_install_aliases_and_create_model_lookup():
    """train_utils.create_model picks the class whose lower-cased name == core_method without underscores
    (opencood/tools/train_utils.py:141-174); the aliased modules must satisfy that lookup."""
    import importlib
    import sys
    from heal_b200.install import install_into_opencood
    done = install_into_opencood()
    try:
        for core in ("heter_pyramid_collab", "heter_model_baseline", "point_pillar"):
            lib = importlib.import_module("opencood.models." + core)
            target = core.replace("_", "")
            cls = next((c for n, c in lib.__dict__.items() if n.lower() == target.lower()), None)
            assert cls is not None and cls.__module__.startswith("heal_b200.")
        enc = importlib.import_module("opencood.models.heter_encoders")
        for name in ("PointPillar", "SECOND", "LiftSplatShoot", "LiftSplatShootVoxel"):
            assert hasattr(enc, name)
    finally:
        for k in done:
            sys.modules.pop(k, None)


def test_training_mode_is_rejected_loudly():
    import pytest
    from heal_b200.models.sub_modules.base_bev_backbone_resnet import ResNetBEVBackbone
    bb = ResNetBEVBackbone({"layer_nums": [1], "layer_strides": [1], "num_filters": [64]})
    bb.train()
    with pytest.raises(NotImplementedError):
        bb({"spatial_features": torch.zeros(1, 64, 4, 4)})


def test_postprocessor_anchor_box_equals_reference_golden(golden_dir):
    """heal_b200's VoxelPostprocessor.generate_anchor_box (host logic) against the anchors the unmodified reference generated."""
    import copy
    import os
    import numpy as np
    import torch
    from heal_b200.data_utils.post_processor import build_postprocessor
    g = golden.load(os.path.join(golden_dir, "postprocess.pt"))
    pp = build_postprocessor(copy.deepcopy(g["params"]), train=False)
    a = pp.generate_anchor_box()
    assert a.dtype == np.float64 and np.array_equal(a, g["anchors"].numpy())
    import pytest
    with pytest.raises(NotImplementedError):
        pp.generate_label()
    with pytest.raises(NotImplementedError):      # anchor-free (CenterPoint) heads are outside the GPU post-processor
        pp.post_process({"a": {"anchor_box": g["anchors"]}},
                        {"a": {"cls_preds": torch.zeros(1, 2, 4, 4), "reg_preds": torch.zeros(1, 32, 7), "iou_preds": torch.zeros(1, 2, 4, 4)}})
