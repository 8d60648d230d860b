"""CPU checks of a captured scene's host logic (heal_b200.graph): the capacity spec and the validation `SceneGraph.load`
runs on the collated ego batch before it copies anything."""
import pytest
import torch

from heal_b200.graph import check_scene, scene_spec

SENSORS = {"m1": "lidar", "m2": "camera", "m3": "lidar", "m4": "camera"}
AML = ["m1", "m2", "m3", "m4", "m1"]
CAPS = {"m1": 5000, "m2": (2, 64, 128), "m3": 3000, "m4": (2, 90, 160, torch.uint8)}
LIMITS = {"m1": {"max_points_per_voxel": 32, "max_voxels": 70000}, "m3": {"max_points_per_voxel": 5, "max_voxels": 70000}}


def test_scene_spec_counts_agents_in_order_of_first_appearance():
    spec = scene_spec(SENSORS, AML, CAPS)
    assert list(spec) == ["m1", "m2", "m3", "m4"]
    assert spec["m1"] == {"agents": 2, "lidar": 5000}
    assert spec["m2"] == {"agents": 1, "camera": (2, 64, 128), "raw": False}
    assert spec["m4"] == {"agents": 1, "camera": (2, 90, 160), "raw": True}


@pytest.mark.parametrize("caps,aml,match", [
    ({**CAPS, "m2": (2, 64, 128, torch.float16)}, AML, "camera capacity"),
    ({**CAPS, "m2": (2, 64)}, AML, "camera capacity"),
    ({**CAPS, "m2": 5000}, AML, "camera capacity"),
    ({**CAPS, "m1": (2, 64, 128)}, AML, "lidar capacity"),
    ({**CAPS, "m1": 0}, AML, "lidar capacity"),
    ({**CAPS, "m1": True}, AML, "lidar capacity"),
    ({k: v for k, v in CAPS.items() if k != "m3"}, AML, "m3: no capacity"),
    (CAPS, AML + ["m5"], "agent modality 'm5'"),
])
def test_scene_spec_refuses_bad_capacities(caps, aml, match):
    with pytest.raises(ValueError, match=match):
        scene_spec(SENSORS, aml, caps)


def _batch(points=(1500, 900), m3_points=2000, raw_m4=True, m2_channels=3):
    cam = lambda k, raw, h, w: {"imgs": torch.zeros((k, 2, h, w, 3), dtype=torch.uint8) if raw else
                                torch.zeros((k, 2, m2_channels, h, w)),
                                **{key: torch.zeros((k, 2, 3, 3) if key.endswith("rots") or key == "intrins" else (k, 2, 3))
                                   for key in ("rots", "trans", "intrins", "post_rots", "post_trans")}}
    return {"agent_modality_list": list(AML), "record_len": torch.tensor([5]),
            "pairwise_t_matrix": torch.zeros((1, 5, 5, 4, 4), dtype=torch.float64),
            "inputs_m1": {"points": torch.zeros((sum(points), 4)), "agent_offsets": torch.zeros(3, dtype=torch.int32),
                          "max_points_per_voxel": 32, "max_voxels": 70000},
            "inputs_m2": cam(1, False, 64, 128),
            "inputs_m3": {"points": torch.zeros((m3_points, 4)), "agent_offsets": torch.zeros(2, dtype=torch.int32)},
            "inputs_m4": cam(1, raw_m4, 90, 160) if raw_m4 else cam(1, False, 90, 160)}


def test_check_scene_accepts_the_captured_scene_and_counts_bytes():
    spec = scene_spec(SENSORS, AML, CAPS)
    n = check_scene(spec, AML, LIMITS, _batch())
    images = 2 * 64 * 128 * 3 * 4 + 2 * 90 * 160 * 3                  # fp32 m2, uint8 m4: one agent of two cameras each
    matrices = 2 * 2 * (9 + 3 + 9 + 9 + 3) * 4                           # rots, trans, intrins, post_rots, post_trans
    assert n == 5 * 5 * 16 * 8 + (2400 + 2000) * 16 + (3 + 2) * 4 + images + matrices
    check_scene(spec, AML, LIMITS, _batch(m2_channels=4))         # a depth plane after RGB is left out of the copy


@pytest.mark.parametrize("change,match", [
    (lambda b: b.update(agent_modality_list=["m1", "m2", "m3", "m1", "m4"]), "captured for"),
    (lambda b: b.update(inputs_m1={**b["inputs_m1"], "points": torch.zeros((5001, 4))}), "capacity is 5000"),
    (lambda b: b.update(inputs_m3={**b["inputs_m3"], "points": torch.zeros((3001, 4))}), "capacity is 3000"),
    (lambda b: b.update(inputs_m1={**b["inputs_m1"], "agent_offsets": torch.zeros(2, dtype=torch.int32)}), "for 2 agents"),
    (lambda b: b.update(inputs_m1={**b["inputs_m1"], "max_voxels": 32000}), "captured with 70000"),
    (lambda b: b.update(inputs_m1={**b["inputs_m1"], "filter_points": True}), "filter_on_gpu"),
    (lambda b: b.update(inputs_m1={"voxel_features": torch.zeros(1)}), "raw clouds"),
    (lambda b: b.update(inputs_m4=_batch(raw_m4=False)["inputs_m4"]), "fp32 images for a graph captured with raw uint8"),
    (lambda b: b["inputs_m2"].update(imgs=torch.zeros((1, 2, 64, 128, 3), dtype=torch.uint8)), "raw uint8 frames for a graph"),
    (lambda b: b["inputs_m2"].update(imgs=torch.zeros((1, 2, 3, 64, 96))), "captured for"),
    (lambda b: b["inputs_m2"].update(imgs=torch.zeros((1, 3, 3, 64, 128))), "captured for"),
])
def test_check_scene_refusals(change, match):
    spec = scene_spec(SENSORS, AML, CAPS)
    b = _batch()
    change(b)
    with pytest.raises(ValueError, match=match):
        check_scene(spec, AML, LIMITS, b)
