"""Single-agent models and late fusion without a GPU: the restatements of oracle/late.py against the goldens made from the
unmodified reference HeterModelLate / HeterPyramidSingle, the mirrors' state-dict keys and modality parsing against the reference's,
and forward_late's grouping of cavs by modality."""
import copy
import os
from collections import OrderedDict

import pytest
import torch

from oracle import efficientnet as oe
from oracle import golden, late

MODELS = {"heter_model_late_m1": (late.heter_model_late, "m1"), "heter_model_late_m2eff": (late.heter_model_late, "m2"),
          "heter_pyramid_single_m1": (late.heter_pyramid_single, "m1"),
          "heter_pyramid_single_m2_convnext": (late.heter_pyramid_single, "m2")}


def _inputs(mod):
    return {"inputs_m1": late.lidar_cav(31)} if mod == "m1" else {"inputs_m2": oe.cam_inputs()}


def _bar(ref):
    return 1e-4 * max(1.0, float(ref.abs().max()))


@pytest.mark.parametrize("name", sorted(MODELS))
def test_oracle_matches_reference_golden(golden_dir, name):
    g = golden.load(os.path.join(golden_dir, f"{name}_small.pt"))
    fn, mod = MODELS[name]
    out = fn(oe.state_dict_of(g["shapes"]), g["args"], _inputs(mod))
    for k in ("cls_preds", "reg_preds", "dir_preds"):
        assert out[k].shape == g["out"][k].shape
        err = (out[k] - g["out"][k]).abs().max().item()
        assert err <= _bar(g["out"][k]), (k, err)
    for a, b in zip(out.get("occ_single_list", []), g["out"].get("occ_single_list", [])):
        assert (a - b).abs().max().item() <= _bar(b)


def test_scene_heads_match_the_oracle(golden_dir):
    g = golden.load(os.path.join(golden_dir, "late_fusion_scene_small.pt"))
    sd = oe.state_dict_of(g["shapes"])
    sd["cls_head_m1.bias"] = sd["cls_head_m1.bias"] + g["cls_bias"]
    batch = late.scene_batch(g["anchors"])
    assert list(batch) == list(g["heads"]) == ["ego", "cav1", "cav2"]
    for cav, content in batch.items():
        assert torch.equal(content["transformation_matrix"], g["transforms"][cav])
        out = late.heter_model_late(sd, g["args"], content)
        for k, ref in g["heads"][cav].items():
            assert (out[k] - ref).abs().max().item() <= _bar(ref), (cav, k)
    assert g["boxes"].shape[0] == g["scores"].shape[0] > 50


@pytest.mark.parametrize("name", sorted(MODELS))
def test_mirror_state_dict_keys_equal_the_reference(golden_dir, name):
    from heal_b200.models.heter_model_late import HeterModelLate
    from heal_b200.models.heter_pyramid_single import HeterPyramidSingle
    g = golden.load(os.path.join(golden_dir, f"{name}_small.pt"))
    cls = HeterModelLate if name.startswith("heter_model_late") else HeterPyramidSingle
    m = cls(copy.deepcopy(g["args"]))
    shapes = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert shapes == g["shapes"]
    mod = MODELS[name][1]
    if cls is HeterModelLate:
        assert any(k.startswith(f"layers_{mod}.resnet.layer0.") for k in shapes)     # never run, still in the checkpoint
        assert not any(k.startswith("aligner_") for k in shapes)                      # aligner_args are not built
        assert {f"cls_head_{mod}.weight", f"reg_head_{mod}.bias", f"dir_head_{mod}.weight"} <= set(shapes)
    else:
        assert {"pyramid_backbone.single_head_2.weight", "cls_head.weight", "shrink_conv.layers.0.double_conv.0.weight"} <= set(shapes)
    r = m.load_state_dict(oe.state_dict_of(g["shapes"]), strict=True)
    assert not r.missing_keys and not r.unexpected_keys


@pytest.mark.parametrize("key", ["inputs_m1", "inputs_m2", "inputs_m12", "inputs_mus"])
def test_modality_parsing_matches_the_reference(key):
    from heal_b200.models.heter_model_late import modality_of
    expect = key.lstrip('inputs_')          # the reference's expression (heter_model_late.py:74)
    assert modality_of({key: {}, "anchor_box": None}) == expect == late.modality_of({key: {}})
    with pytest.raises(ValueError):
        modality_of({"inputs_m1": {}, "inputs_m2": {}})


class _Recorder:
    """A stand-in for a model's batched per-modality forward: records each call's modality and batch, returns a fake heads map
    whose image j carries the index of the cav it was computed for."""

    def __init__(self):
        self.calls = []

    def __call__(self, data, m, ext, out=None):
        inp = data[f"inputs_{m}"]
        ids = inp["ids"].tolist()
        self.calls.append((m, ids, out is not None))
        ext["depth_items_probe"] = (inp["ids"].float().view(-1, 1),)
        y = torch.tensor(ids, dtype=torch.float32).view(-1, 1, 1, 1).expand(-1, 2, 2, 3)
        if out is not None:
            out.t.copy_(y)
            return out
        return _FakeAct(y.contiguous())


class _FakeAct:
    def __init__(self, t):
        self.t, self.N, self.H, self.W, self.C = t, *t.shape
        self.device = t.device

    def images(self, a, b):
        return _FakeAct(self.t[a:b])


def test_forward_late_groups_by_modality_and_keeps_batch_order(monkeypatch):
    from heal_b200 import ops
    from heal_b200.models import heter_model_late as hml
    rec = _Recorder()

    class Model(hml.LateForward):
        training = False
        _heads_act = staticmethod(rec)

        def _any_heads(self):
            return None

        def _split(self, y):
            return {"heads": y}

    monkeypatch.setattr(ops, "act_empty", lambda n, h, w, c, fmt, dev: _FakeAct(torch.full((n, h, w, c), -1.0)))
    batch = OrderedDict((c, {f"inputs_{m}": {"ids": torch.tensor([i])}, "transformation_matrix": None})
                        for i, (c, m) in enumerate([("ego", "m2"), ("a", "m1"), ("b", "m2"), ("c", "m1"), ("d", "m1")]))
    out = Model().forward_late(batch)
    assert list(out) == ["ego", "a", "b", "c", "d"]
    # one call per modality, in order of first appearance, each with all of its cavs in batch order
    assert [(m, ids) for m, ids, _ in rec.calls] == [("m2", [0, 2]), ("m1", [1, 3, 4])]
    for i, (c, o) in enumerate(out.items()):
        assert torch.equal(o["heads"], torch.full((1, 2, 2, 3), float(i))), c
        assert o["depth_items_probe"][0].item() == i
    # a modality whose cavs are one contiguous run is written straight into the shared buffer
    rec.calls.clear()
    batch2 = OrderedDict((c, {f"inputs_{m}": {"ids": torch.tensor([i])}})
                         for i, (c, m) in enumerate([("ego", "m1"), ("a", "m2"), ("b", "m2")]))
    out = Model().forward_late(batch2)
    assert rec.calls == [("m1", [0], False), ("m2", [1, 2], True)]
    assert [o["heads"].flatten()[0].item() for o in out.values()] == [0.0, 1.0, 2.0]


def test_batch_inputs_layouts():
    from heal_b200.models.heter_model_late import batch_inputs
    a, b = late.lidar_cav(31), late.lidar_cav(32)
    v = batch_inputs([a, b])
    assert v["batch_size"] == 2 and v["voxel_features"].shape[0] == a["voxel_features"].shape[0] + b["voxel_features"].shape[0]
    na = a["voxel_coords"].shape[0]
    assert (v["voxel_coords"][:na, 0] == 0).all() and (v["voxel_coords"][na:, 0] == 1).all()
    assert torch.equal(v["voxel_coords"][na:, 1:], b["voxel_coords"][:, 1:]) and (b["voxel_coords"][:, 0] == 0).all()
    p = [torch.zeros(5, 4), torch.ones(7, 4), torch.ones(2, 4)]
    r = batch_inputs([{"points": x, "agent_offsets": torch.tensor([0, x.shape[0]], dtype=torch.int32)} for x in p])
    assert r["agent_offsets"].tolist() == [0, 5, 12, 14] and r["points"].shape == (14, 4)
    c = batch_inputs([oe.cam_inputs(1), oe.cam_inputs(2)])
    assert c["imgs"].shape[0] == 2 and c["rots"].shape[:2] == (2, 2)
    assert torch.equal(c["imgs"][1:], oe.cam_inputs(2)["imgs"])
