"""CPU checks of LateFusionStream's host logic (heal_b200.graph.late_cache, check_late_scene): the key of a late-fusion frame,
the least-recently-used graphs of each pipeline slot and their eviction, the cav limit, and every refusal a frame meets before
anything is copied.  A stub stands in for the capture and host tensors for the batch, so no device is needed.  Also the
box-decode buffers a stream slot shares: larger ones are taken, smaller ones refused."""
from collections import OrderedDict

import pytest
import torch

from heal_b200.graph import LateFusionStream, check_late_scene, late_cache

SENSORS = {"m1": "lidar", "m2": "camera", "m3": "lidar", "m4": "camera"}
CAPS = {"m1": 5000, "m2": (2, 64, 128), "m3": 3000, "m4": (2, 90, 160, torch.uint8)}
LIMITS = {"m1": {"max_points_per_voxel": 32, "max_voxels": 70000}, "m3": {"max_points_per_voxel": 5, "max_voxels": 70000}}


def _cache(max_graphs=16, slots=2, caps=CAPS, max_cav=5, gt_capacity=None):
    made = []

    def capture(slot, key):
        made.append((slot, key))
        return {"slot": slot, "key": key}
    return late_cache(SENSORS, caps, max_cav, LIMITS, slots, max_graphs, capture, gt_capacity), made


def _cav(m, points=1000):
    """One cav of a late batch (host tensors; only shapes matter)."""
    if SENSORS[m] == "lidar":
        inputs = {"points": torch.zeros((points, 4)), "agent_offsets": torch.tensor([0, points], dtype=torch.int32)}
    else:
        raw = len(CAPS[m]) == 4
        cams, h, w = CAPS[m][:3]
        inputs = {"imgs": torch.zeros((1, cams, h, w, 3), dtype=torch.uint8) if raw else torch.zeros((1, cams, 3, h, w)),
                  **{key: torch.zeros((1, cams, 3, 3) if key in ("rots", "intrins", "post_rots") else (1, cams, 3))
                     for key in ("rots", "trans", "intrins", "post_rots", "post_trans")}}
    return {f"inputs_{m}": inputs, "transformation_matrix": torch.eye(4)}


def _batch(mods, points=1000):
    return OrderedDict(("ego" if i == 0 else f"cav{i}", _cav(m, points)) for i, m in enumerate(mods))


def test_the_key_is_the_ordered_cav_modality_tuple():
    c, made = _cache()
    assert c.check(_batch(["m1", "m2", "m1"])) == ("m1", "m2", "m1")
    assert c.check(_batch(["m2", "m1", "m1"])) == ("m2", "m1", "m1")
    assert c.check(_batch(["m3"])) == ("m3",)
    assert c.key(["m1", "m4"]) == ("m1", "m4")
    a, b = c.graph(0, ("m1", "m2", "m1")), c.graph(0, ("m2", "m1", "m1"))     # another cav order is another graph
    assert a is not b and c.captures == 2
    assert c.graph(0, ("m1", "m2", "m1")) is a and c.captures == 2
    assert c.graph(1, ("m1", "m2", "m1")) is not a and c.captures == 3         # every slot captures its own
    assert made == [(0, ("m1", "m2", "m1")), (0, ("m2", "m1", "m1")), (1, ("m1", "m2", "m1"))]


def test_least_recently_used_graph_is_evicted_at_max_graphs():
    c, made = _cache(max_graphs=2, slots=1)
    A, B, C = ("m1",), ("m1", "m2"), ("m2", "m1")
    c.graph(0, A)
    c.graph(0, B)
    c.graph(0, A)                                                  # A becomes the most recent
    assert list(c.slots[0]) == [B, A] and c.captures == 2
    c.graph(0, C)                                                  # above max_graphs: B goes
    assert list(c.slots[0]) == [A, C] and c.captures == 3
    c.graph(0, B)                                                  # B comes back: recaptured, A goes
    assert list(c.slots[0]) == [C, B] and c.captures == 4 and made[-1] == (0, B)


def test_max_graphs_one_keeps_the_last_list():
    c, _ = _cache(max_graphs=1, slots=1)
    for k in (("m1",), ("m1", "m2"), ("m1",), ("m1",)):
        c.graph(0, k)
    assert list(c.slots[0]) == [("m1",)] and c.captures == 3
    with pytest.raises(ValueError, match="at least one graph"):
        _cache(max_graphs=0)


def test_max_cav_is_enforced():
    c, made = _cache(max_cav=2)
    assert c.check(_batch(["m1", "m2"])) == ("m1", "m2")
    with pytest.raises(ValueError, match=r"3 cavs .* max_cav = 2"):
        c.check(_batch(["m1", "m2", "m1"]))
    with pytest.raises(ValueError, match="max_cav = 2"):
        c.key(["m1", "m1", "m1"])
    assert made == []
    for bad in (17, 0, 2.0, True):
        with pytest.raises(ValueError, match="1 to 16 cavs"):
            LateFusionStream(object(), CAPS, bad, {})


def _gt(n):
    return torch.zeros((n, 8, 3))


def _voxels(b):
    b["ego"]["inputs_m1"] = {"voxel_features": torch.zeros((10, 32, 4)), "voxel_coords": torch.zeros((10, 4), dtype=torch.int32),
                             "voxel_num_points": torch.zeros(10, dtype=torch.int32)}


@pytest.mark.parametrize("mods,change,kw,match", [
    (["m1", "m5"], None, {}, "agent modality 'm5'"),
    (["m1", "m3"], None, {"caps": {k: v for k, v in CAPS.items() if k != "m3"}}, "m3: no capacity"),
    (["m1", "m2", "m3", "m4", "m1", "m3"], None, {}, r"6 cavs .* max_cav = 5"),
    ([], None, {}, r"0 cavs .* 1 to max_cav"),
    (["m1", "m2"], _voxels, {}, "raw cloud .* not voxels"),
    (["m1", "m2"], lambda b: b["ego"]["inputs_m1"].update(agent_offsets=torch.zeros(3, dtype=torch.int32)), {},
     "carries one cloud"),
    (["m1", "m2"], lambda b: b["ego"]["inputs_m1"].pop("agent_offsets"), {}, "raw cloud"),
    (["m1", "m2"], lambda b: b["ego"]["inputs_m1"].update(filter_points=True), {}, "filter_on_gpu"),
    (["m1", "m2"], lambda b: b["ego"]["inputs_m1"].update(max_voxels=32000), {}, "max_voxels 32000, .* captured with 70000"),
    (["m3"], lambda b: b["ego"]["inputs_m3"].update(max_points_per_voxel=32), {}, "captured with 5"),
    (["m1", "m1", "m1"], None, {"points": 1700}, "m1: the scene's 3 cavs have more points than the capacity 5000"),
    (["m1"], lambda b: b["ego"]["inputs_m1"].update(points=torch.zeros((10, 3))), {}, r"\(P, 4\) expected"),
    (["m1", "m2"], lambda b: b["cav1"]["inputs_m2"].update(imgs=torch.zeros((1, 2, 3, 64, 96))), {}, "captured for"),
    (["m1", "m2"], lambda b: b["cav1"]["inputs_m2"].update(imgs=torch.zeros((2, 2, 3, 64, 128))), {}, "captured for"),
    (["m4"], lambda b: b["ego"]["inputs_m4"].update(imgs=torch.zeros((1, 2, 3, 90, 160))), {},
     "fp32 images for a graph captured with raw uint8 frames"),
    (["m2"], lambda b: b["ego"]["inputs_m2"].update(imgs=torch.zeros((1, 2, 64, 128, 3), dtype=torch.uint8)), {},
     "raw uint8 frames for a graph captured with normalised fp32 images"),
    (["m2"], lambda b: b["ego"]["inputs_m2"].update(rots=torch.zeros((1, 3, 3, 3))), {}, r"rots of shape \(1, 3, 3, 3\)"),
    (["m1", "m2"], lambda b: b["cav1"].pop("transformation_matrix"), {}, "'cav1': no transformation_matrix"),
    (["m1"], lambda b: b["ego"].update(inputs_m2=_cav("m2")["inputs_m2"]), {}, "exactly one inputs_"),
    (["m1", "m2"], None, {"gt": _gt(3)}, "without eval_thresholds"),
    (["m1", "m2"], None, {"gt_capacity": 4}, r"gt_boxes \(G, 8, 3\) fp32 required"),
    (["m1", "m2"], None, {"gt_capacity": 4, "gt": _gt(5)}, "gt_capacity is 4"),
    (["m1", "m2"], None, {"gt_capacity": 4, "gt": _gt(2).double()}, "float32 corners expected"),
])
def test_check_late_scene_refusals(mods, change, kw, match):
    """Each refusal raises ValueError from the stream's check, before a graph is captured or a slot buffer written; the
    same batch without the fault passes."""
    c, made = _cache(caps=kw.get("caps", CAPS), gt_capacity=kw.get("gt_capacity"))
    b = _batch([m for m in mods if m in SENSORS], kw.get("points", 1000))
    if "m5" in mods:
        b["cav1"] = {"inputs_m5": {}, "transformation_matrix": torch.eye(4)}
    if change is not None:
        change(b)
    with pytest.raises(ValueError, match=match):
        c.check(b, kw.get("gt"))
    assert made == [] and c.captures == 0
    with pytest.raises(ValueError, match=match):
        check_late_scene(SENSORS, kw.get("caps", CAPS), 5, LIMITS, b, kw.get("gt"), kw.get("gt_capacity"))


def test_check_late_scene_counts_the_bytes_load_copies():
    b = _batch(["m1", "m4", "m1", "m2"], points=1200)
    per_cam = 2 * 3 * 3 * 4 * 3 + 2 * 3 * 4 * 2
    want = 2 * 1200 * 16 + 3 * 4 + 2 * 90 * 160 * 3 + 2 * 3 * 64 * 128 * 4 + 2 * per_cam + 4 * 64 + 5 * 96 + 4
    assert check_late_scene(SENSORS, CAPS, 5, LIMITS, b, _gt(5), 10) == want
    assert check_late_scene(SENSORS, CAPS, 5, LIMITS, _batch(["m1"] * 5), None, None) > 0        # 5 x 1000 = the capacity


class _OnDevice(torch.Tensor):
    """A host tensor that passes the wrapper's `is_cuda` test: validation reads only its shape, dtype and layout."""

    @property
    def is_cuda(self):
        return True


def _buffers(H, W, A, top=1000):
    from heal_b200 import ops
    b = object.__new__(ops.PostprocessBuffers)
    b.H, b.W, b.A, b.top = H, W, A, top
    b.workspace = b.boxes = b.scores = b.count = b.stats = torch.zeros(0)
    return b


def test_late_decode_takes_buffers_for_more_cavs_and_refuses_smaller_ones(monkeypatch):
    from heal_b200 import ops
    launched = []
    monkeypatch.setattr(ops, "_need_cuda", lambda *t: None)
    monkeypatch.setattr(ops, "_p", lambda t: 0)
    monkeypatch.setattr(ops, "_call", lambda name, *a: launched.append(a[5]))
    n, H, W, A = 3, 4, 5, 2
    heads = ops.Act(torch.zeros((n, H, W, 10 * A)), "f32")
    args = (heads, heads, heads, torch.zeros((H, W, A, 7)), torch.zeros((n, 4, 4)).as_subclass(_OnDevice), 0.2, 0.15)
    for rows in (H * n, H * 16):                                      # exactly the call's cavs, or a stream slot's max_cav
        ops.box_decode_nms_late(*args, buffers=_buffers(rows, W, A), coffsets=(0, A, 8 * A))
    assert launched == [n, n]
    for bad in (_buffers(H * n - 1, W, A), _buffers(H * n, W + 1, A), _buffers(H * n, W, A + 1), _buffers(H * n, W, A, 500)):
        with pytest.raises(ValueError, match="buffers were made for another geometry"):
            ops.box_decode_nms_late(*args, buffers=bad, coffsets=(0, A, 8 * A))
    assert launched == [n, n]
