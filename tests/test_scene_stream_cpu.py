"""CPU checks of SceneStream's host logic (heal_b200.graph.SceneGraphCache): the key of a frame, the least-recently-used graphs
of each pipeline slot and their eviction, and the refusals a frame meets before anything is copied.  A stub stands in for the
capture, so no device is needed.  Also the leading-slice views a SceneGraph takes of a slot's shared input buffers."""
import pytest
import torch

from heal_b200.graph import SceneGraphCache, _input_buffers, _input_views, scene_spec

SENSORS = {"m1": "lidar", "m2": "camera", "m3": "lidar", "m4": "camera"}
CAPS = {"m1": 5000, "m2": (2, 64, 128), "m3": 3000, "m4": (2, 90, 160, torch.uint8)}
LIMITS = {"m1": {"max_points_per_voxel": 32, "max_voxels": 70000}, "m3": {"max_points_per_voxel": 5, "max_voxels": 70000}}


def _cache(max_graphs=16, slots=2, caps=CAPS, max_cav=5):
    made = []

    def capture(slot, key):
        made.append((slot, key))
        return {"slot": slot, "key": key}
    return SceneGraphCache(SENSORS, caps, max_cav, LIMITS, slots, max_graphs, capture), made


def _batch(aml, points=1000):
    """A collated ego batch of the agent list `aml` (host tensors; only shapes matter)."""
    b = {"agent_modality_list": list(aml), "record_len": torch.tensor([len(aml)]),
         "pairwise_t_matrix": torch.zeros((1, 5, 5, 4, 4), dtype=torch.float64)}
    for m in dict.fromkeys(aml):
        k = aml.count(m)
        if SENSORS[m] == "lidar":
            b[f"inputs_{m}"] = {"points": torch.zeros((points, 4)), "agent_offsets": torch.zeros(k + 1, dtype=torch.int32)}
        else:
            raw = len(CAPS[m]) == 4
            cams, h, w = CAPS[m][:3]
            b[f"inputs_{m}"] = {"imgs": torch.zeros((k, cams, h, w, 3), dtype=torch.uint8) if raw else torch.zeros((k, cams, 3, h, w)),
                                **{key: torch.zeros((k, cams, 3, 3) if key.endswith("rots") or key == "intrins" else (k, cams, 3))
                                   for key in ("rots", "trans", "intrins", "post_rots", "post_trans")}}
    return b


def test_the_key_is_the_ordered_agent_list():
    c, made = _cache()
    assert c.check(_batch(["m1", "m3"])) == ("m1", "m3")
    assert c.check(_batch(["m3", "m1"])) == ("m3", "m1")
    assert c.key(["m1", "m2", "m1"]) == ("m1", "m2", "m1")
    a, b = c.graph(0, ("m1", "m3")), c.graph(0, ("m3", "m1"))     # another fusion order is another graph
    assert a is not b and made == [(0, ("m1", "m3")), (0, ("m3", "m1"))]
    assert c.graph(0, ("m1", "m3")) is a and c.captures == 2
    assert c.graph(1, ("m1", "m3")) is not a and c.captures == 3  # every slot captures its own
    assert c.graphs_captured == 3
    assert made == [(0, ("m1", "m3")), (0, ("m3", "m1")), (1, ("m1", "m3"))]


def test_least_recently_used_graph_is_evicted_at_max_graphs():
    c, made = _cache(max_graphs=3, slots=1)
    A, B, C, D = ("m1",), ("m1", "m3"), ("m1", "m2"), ("m1", "m4")
    for k in (A, B, C):
        c.graph(0, k)
    assert list(c.slots[0]) == [A, B, C]
    c.graph(0, A)                                                  # A becomes the most recent
    assert list(c.slots[0]) == [B, C, A] and c.captures == 3
    c.graph(0, D)                                                  # above max_graphs: B, the least recently used, goes
    assert list(c.slots[0]) == [C, A, D] and c.captures == 4
    c.graph(0, B)                                                  # B comes back: recaptured, C goes
    assert list(c.slots[0]) == [A, D, B] and c.captures == 5
    assert made[-1] == (0, B) and c.graphs_captured == 3


def test_max_graphs_one_keeps_the_last_list():
    c, _ = _cache(max_graphs=1, slots=1)
    for k in (("m1",), ("m1", "m3"), ("m1",)):
        c.graph(0, k)
    assert list(c.slots[0]) == [("m1",)] and c.captures == 3
    with pytest.raises(ValueError, match="at least one graph"):
        _cache(max_graphs=0)


@pytest.mark.parametrize("aml,caps,match", [
    (["m1", "m5"], CAPS, "agent modality 'm5'"),
    (["m1", "m3"], {k: v for k, v in CAPS.items() if k != "m3"}, "m3: no capacity"),
    (["m1", "m2", "m3", "m4", "m1", "m3"], CAPS, "6 agents .* max_cav = 5"),
    ([], CAPS, "0 agents"),
])
def test_refusals_of_the_list(aml, caps, match):
    c, made = _cache(caps=caps)
    with pytest.raises(ValueError, match=match):
        c.key(aml)
    with pytest.raises(ValueError, match=match):
        c.check({**_batch([m for m in aml if m in SENSORS]), "agent_modality_list": list(aml)})
    assert made == [] and c.captures == 0


def test_max_cav_is_the_stream_s():
    c, _ = _cache(max_cav=2)
    assert c.key(["m1", "m3"]) == ("m1", "m3")
    with pytest.raises(ValueError, match="3 agents .* max_cav = 2"):
        c.check(_batch(["m1", "m3", "m1"]))


@pytest.mark.parametrize("change,match", [
    (lambda b: b["inputs_m1"].update(points=torch.zeros((5001, 4))), "capacity is 5000"),
    (lambda b: b["inputs_m1"].update(agent_offsets=torch.zeros(4, dtype=torch.int32)), "for 2 agents"),
    (lambda b: b["inputs_m1"].update(max_voxels=32000), "captured with 70000"),
    (lambda b: b["inputs_m1"].update(filter_points=True), "filter_on_gpu"),
    (lambda b: b["inputs_m4"].update(imgs=torch.zeros((1, 2, 3, 90, 160))), "fp32 images for a graph captured with raw uint8"),
    (lambda b: b["inputs_m2"].update(imgs=torch.zeros((1, 2, 3, 64, 96))), "captured for"),
])
def test_check_scene_refusals_for_the_frame_s_own_list(change, match):
    """The frame's own list (two m1 agents here) is what check_scene measures the batch against."""
    c, made = _cache()
    b = _batch(["m1", "m4", "m2", "m1"])
    assert c.check(b) == ("m1", "m4", "m2", "m1")
    change(b)
    with pytest.raises(ValueError, match=match):
        c.check(b)
    assert made == []


def test_input_views_are_leading_slices_of_the_slot_buffers():
    full = {m: dict(sp, agents=5) for m, sp in scene_spec(SENSORS, list(CAPS), CAPS).items()}
    slot = _input_buffers(full, "cpu")
    views = _input_views(scene_spec(SENSORS, ["m1", "m4", "m1"], CAPS), slot)
    assert list(views) == ["m1", "m4"]
    assert views["m1"]["points"].shape == (5000, 4) and views["m1"]["points"].data_ptr() == slot["m1"]["points"].data_ptr()
    assert views["m1"]["agent_offsets"].shape == (3,) and views["m1"]["agent_offsets"].is_contiguous()
    assert views["m4"]["imgs"].shape == (1, 2, 90, 160, 3) and views["m4"]["imgs"].dtype == torch.uint8
    assert all(v.data_ptr() == slot["m4"][k].data_ptr() and v.is_contiguous() for k, v in views["m4"].items())
    with pytest.raises(ValueError, match=r"inputs\['m2'\]\['imgs'\]: missing"):
        _input_views(scene_spec(SENSORS, ["m2"], CAPS), {})
    small = _input_buffers({m: dict(sp, agents=1) for m, sp in full.items()}, "cpu")
    with pytest.raises(ValueError, match=r"inputs\['m1'\]\['agent_offsets'\]: \(2,\)"):
        _input_views(scene_spec(SENSORS, ["m1", "m1"], CAPS), small)
    with pytest.raises(ValueError, match=r"inputs\['m3'\]\['points'\]: \(3000, 4\).*\(4000, 4\)"):
        _input_views(scene_spec(SENSORS, ["m3"], {**CAPS, "m3": 4000}), slot)
