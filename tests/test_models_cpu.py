"""The five HEAL mirrors built on the CPU from every model golden's `args`: the state dict has the golden's keys, shapes and order
(what `parameters()` and saved checkpoints follow), loads strictly, and the attributes read outside the models (graph.py,
parallel.py, the scene-graph tests and the profiles) are there for every modality."""
import copy
import glob
import os
import re

import pytest
import torch.nn as nn

from oracle import golden
from workloads import procedural

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
NAMES = sorted(os.path.basename(p)[:-len(".pt.xz")] for p in glob.glob(os.path.join(GOLDEN, "heter_*.pt.xz")))

# longest prefix first: heter_model_baseline_ms_* also starts with heter_model_baseline_
PREFIXES = ["heter_model_baseline_ms_", "heter_model_baseline_", "heter_pyramid_collab_", "heter_model_late_",
            "heter_pyramid_single_"]
WITH_ALIGNER = {"HeterPyramidCollab", "HeterModelBaselineMs", "HeterPyramidSingle"}
WITH_SHRINK = {"HeterPyramidCollab", "HeterModelBaseline", "HeterModelBaselineMs", "HeterPyramidSingle"}
# children that may hold no state: a parameterless fusion (MaxFusion) and an identity aligner
STATELESS = re.compile(r"fusion_net|aligner_m\d+")


def test_every_model_golden_is_covered():
    assert len(NAMES) >= 20
    assert all(any(n.startswith(p) for p in PREFIXES) for n in NAMES)


def _model(name):
    from heal_b200.models.heter_model_baseline import HeterModelBaseline
    from heal_b200.models.heter_model_baseline_ms import HeterModelBaselineMs
    from heal_b200.models.heter_model_late import HeterModelLate
    from heal_b200.models.heter_pyramid_collab import HeterPyramidCollab
    from heal_b200.models.heter_pyramid_single import HeterPyramidSingle
    classes = [HeterModelBaselineMs, HeterModelBaseline, HeterPyramidCollab, HeterModelLate, HeterPyramidSingle]
    cls = next(c for p, c in zip(PREFIXES, classes) if name.startswith(p))
    g = golden.load(os.path.join(GOLDEN, f"{name}.pt"))
    return cls(copy.deepcopy(g["args"])), g


@pytest.mark.parametrize("name", NAMES)
def test_state_dict_layout(name):
    model, g = _model(name)
    sd = model.state_dict()
    assert [(k, tuple(v.shape)) for k, v in sd.items()] == list(g["shapes"].items())
    r = model.load_state_dict(procedural.make_state_dict(g["shapes"]), strict=True)
    assert not r.missing_keys and not r.unexpected_keys
    for n, _ in model.named_children():
        assert any(k.startswith(n + ".") for k in sd) or STATELESS.fullmatch(n), n


@pytest.mark.parametrize("name", NAMES)
def test_attributes_read_outside_the_model(name):
    model, _ = _model(name)
    cls = type(model).__name__
    assert list(model.sensor_type_dict) == model.modality_name_list
    for m in model.modality_name_list:
        assert isinstance(getattr(model, f"encoder_{m}"), nn.Module)
        assert isinstance(getattr(model, f"backbone_{m}"), nn.Module)
        if cls in WITH_ALIGNER:
            assert isinstance(getattr(model, f"aligner_{m}"), nn.Module)
        if model.sensor_type_dict[m] == "camera":
            assert isinstance(getattr(model, f"crop_ratio_W_{m}"), float)
            assert isinstance(getattr(model, f"crop_ratio_H_{m}"), float)
    if cls in WITH_SHRINK:
        assert isinstance(model.shrink_flag, bool)
        assert isinstance(getattr(model, "shrink_conv", None), nn.Module) == model.shrink_flag
    if cls == "HeterModelLate":
        assert list(model._heads) == model.modality_name_list
        heads = list(model._heads.values())
        for m in model.modality_name_list:
            assert all(isinstance(getattr(model, f"{h}_head_{m}"), nn.Conv2d) for h in ("cls", "reg", "dir"))
    else:
        heads = [model._heads]
        assert model._heads.heads == [model.cls_head, model.reg_head, model.dir_head]
    assert not any(isinstance(h, nn.Module) for h in heads)
    assert not any(isinstance(v, nn.Module) for v in vars(model).values())      # modules live in _modules, nowhere else
