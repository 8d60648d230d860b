"""LateFusionStream (heal_b200.graph): late, no and single fusion over a stream whose cav list changes from frame to frame, one
captured LateFusionGraph per ordered cav-modality list and pipeline slot, the graphs of a slot sharing its memory pool and
buffers.  Every frame's boxes must be, bit for bit, what a LateFusionGraph captured for its list alone gives on the same batch,
and what the eager forward_late + box_decode_nms_multi gives; with evaluation, `result_stat` must equal the one built frame by
frame through the eval_utils drop-in on those boxes."""
import copy
import gc
import os
from collections import OrderedDict

import numpy as np
import pytest
import torch

from oracle import eval as oev
from oracle import efficientnet as oe
from oracle import golden, late
from oracle.make_golden_eval import rect
from test_gpu_camera_input import _cam_batch
from test_gpu_eval_stream import THR3, _calculate_ap, _drop_in_stat, _gt_near
from test_gpu_late import _anchors_dev, _cuda, _eager_boxes, _mixed_late_args

pytestmark = pytest.mark.gpu

M1, M2 = "m1", "m2"
FRAMES = [[M1, M2, M1], [M1], [M2, M1], [M1, M1, M2, M2, M1], [M1, M2, M1], [M1]]
LISTS = list(dict.fromkeys(tuple(f) for f in FRAMES))
FAR = 5                                   # the last frame's ego pose lies 1 km away: every box leaves the range, none is kept
CAPS = {M1: 3 * 2000, M2: (2, 64, 128)}
RAW_CAPS = {M1: 3 * 2000, M2: (2, 90, 160, torch.uint8)}


@pytest.fixture(scope="module", autouse=True)
def _tc32():
    from heal_b200 import engine
    old = engine.PRECISION
    engine.set_precision("tc32")
    yield
    engine.set_precision(old)


def _model():
    """HeterModelLate with a PointPillars m1 and an LSS-EfficientNet m2 that also takes 90 x 160 uint8 frames; procedural weights
    with the class biases raised so that both modalities keep boxes."""
    from heal_b200.models.heter_model_late import HeterModelLate
    args = _mixed_late_args()
    args["m2"]["encoder_args"]["data_aug_conf"].update({"H": 90, "W": 160, "bot_pct_lim": [0.0, 0.05]})
    m = HeterModelLate(copy.deepcopy(args)).eval()
    sd = oe.state_dict_of({k: tuple(v.shape) for k, v in m.state_dict().items()})
    for k in [k for k in sd if k.startswith("cls_head") and k.endswith("bias")]:
        sd[k] = sd[k] + 3.0
    m.load_state_dict(sd, strict=True)
    return m.cuda()


def late_batch(model, mods, seed, raw=False, far=False):
    """A late batch `{cav_id: cav_content}` of the cav list `mods`, ego first: raw clouds of 1200-2000 points, two-camera rigs
    (fp32 64 x 128 images, or with `raw` uint8 90 x 160 frames), seeded poses as host fp32 4 x 4 matrices."""
    rng = np.random.default_rng(700 + seed)
    out = OrderedDict()
    for i, m in enumerate(mods):
        if m == M1:
            pts = torch.from_numpy(late.scene_points(1000 * seed + i, int(rng.integers(1200, 2000)))).cuda()
            inputs = {"points": pts, "agent_offsets": torch.tensor([0, pts.shape[0]], dtype=torch.int32, device="cuda")}
        elif raw:
            inputs = _cuda(_cam_batch(1, 2, 90, 160, model.encoder_m2.camera_plan(90, 160), 1000 * seed + i)[0])
        else:
            inputs = _cuda(oe.cam_inputs(1000 * seed + i))
        pose = (0.0, 0.0, 0.0) if i == 0 else (rng.uniform(-5, 5), rng.uniform(-5, 5), rng.uniform(-180, 180))
        if far and i == 0:
            pose = (1000.0, 0.0, 0.0)
        out["ego" if i == 0 else f"cav{i}"] = {f"inputs_{m}": inputs, "transformation_matrix": late.pose(*pose).float()}
    return out


def _stand_alone(m, caps, frames, batches, params):
    """Per frame, what a LateFusionGraph captured for that list alone gives: (boxes[:count], scores[:count], count)."""
    from heal_b200.graph import LateFusionGraph
    graphs, want = {}, []
    for mods, b in zip(frames, batches):
        g = graphs.get(tuple(mods))
        if g is None:
            g = graphs[tuple(mods)] = LateFusionGraph(m, mods, caps, params)
        g.load(b)
        out = g.replay()
        torch.cuda.synchronize()
        n = int(out.count.item())
        want.append((out.boxes[:n].cpu(), out.scores[:n].cpu(), n))
    return want


@pytest.fixture(scope="module")
def scene(golden_dir):
    m = _model()
    params = golden.load(os.path.join(golden_dir, "late_fusion_scene_small.pt"))["params"]
    batches = [late_batch(m, mods, i, far=i == FAR) for i, mods in enumerate(FRAMES)]
    return m, params, batches, _stand_alone(m, CAPS, FRAMES, batches, params)


def _copy(r):
    return {k: (v.clone() if torch.is_tensor(v) else v) for k, v in r.items()}


def _run(stream, batches, gts=None):
    got = []
    for i, b in enumerate(batches):
        r = stream.submit(b, None if gts is None else gts[i])
        if r is not None:
            got.append(_copy(r))
    return got + [_copy(r) for r in stream.drain()]


def _same(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(a, b)


def _check(got, want, frames):
    assert len(got) == len(frames)
    for i, (r, (boxes, scores, n), mods) in enumerate(zip(got, want, frames)):
        assert r["modality_list"] == list(mods), i                        # results come back in submission order
        assert {"boxes", "scores", "count", "modality_list"} <= set(r)
        assert int(r["count"][0]) == n, (i, mods)
        assert _same(r["boxes"][:n], boxes) and _same(r["scores"][:n], scores), (i, mods)


def test_stand_alone_graphs_equal_the_eager_late_path(scene):
    m, params, batches, want = scene
    anchors = _anchors_dev(params)
    for i, (b, (boxes, scores, n)) in enumerate(zip(batches, want)):
        eb, es = _eager_boxes(m, b, params, anchors)
        assert _same(boxes, eb.cpu()) and _same(scores, es.cpu()), i
        assert (n == 0) == (i == FAR), (i, n)                        # only the far frame has no box


@pytest.mark.parametrize("depth", [1, 2, 3])
def test_stream_of_changing_cav_lists_equals_stand_alone_graphs(scene, depth):
    from heal_b200.graph import LateFusionStream
    m, params, batches, want = scene
    stream = LateFusionStream(m, CAPS, 5, params, depth=depth)
    _check(_run(stream, batches), want, FRAMES)
    caps_per_slot = [len({tuple(FRAMES[i]) for i in range(k, len(FRAMES), depth)}) for k in range(depth)]
    assert stream.captures == sum(caps_per_slot) == stream.graphs_captured
    again = _run(stream, batches)             # every list replayed after the others; the first depth - 1 results are the tail
    _check(again[depth - 1:], want, FRAMES)
    assert stream.captures == sum(caps_per_slot)


def test_a_list_replays_its_own_bits_after_other_lists_in_its_slot(scene):
    from heal_b200.graph import LateFusionStream
    m, params, batches, want = scene
    stream = LateFusionStream(m, CAPS, 5, params, depth=1)
    for mods in reversed(LISTS):                                          # captured ahead: the first list last
        stream.capture(mods)
    assert stream.captures == len(LISTS)
    order = [3, 0, 1, 2, 4, 5, 0, 3]
    got = [_copy(stream.submit(batches[i])) for i in order]
    _check(got, [want[i] for i in order], [FRAMES[i] for i in order])
    assert stream.captures == len(LISTS)


def test_eviction_at_max_graphs_recaptures_and_still_matches(scene):
    from heal_b200.graph import LateFusionStream
    m, params, batches, want = scene
    stream = LateFusionStream(m, CAPS, 5, params, depth=1, max_graphs=2)
    order = [0, 1, 0, 2, 1, 3, 4]                     # L0 L1 L0 L2 (drops L1) L1 (drops L0) L3 (drops L2) L0 (drops L1)
    _check(_run(stream, [batches[i] for i in order]), [want[i] for i in order], [FRAMES[i] for i in order])
    assert stream.captures == 6 and stream.graphs_captured == 2
    assert list(stream.cache.slots[0]) == [tuple(FRAMES[3]), tuple(FRAMES[0])]
    one = LateFusionStream(m, CAPS, 5, params, depth=1, max_graphs=1)
    _check(_run(one, batches[:3]), want[:3], FRAMES[:3])
    assert one.captures == 3 and one.graphs_captured == 1


def _gts(want, params):
    """GT per frame: near every third box plus a few elsewhere; frame 1's GT is padded past `max_num` with far boxes."""
    gts = [_gt_near(boxes, 90 + i, 400) for i, (boxes, _, _) in enumerate(want)]
    extra = params["max_num"] + 10 - gts[1].shape[0]
    if extra > 0:
        far = np.stack([rect(40 + 5 * j, 44 + 5 * j, 40, 41.8) for j in range(extra)]).astype(np.float32)
        gts[1] = torch.cat([gts[1], torch.from_numpy(far)])
    assert gts[1].shape[0] > params["max_num"] and want[FAR][2] == 0 and gts[FAR].shape[0] > 0
    return gts


def _want_stat(want, gts):
    from heal_b200.utils import eval_utils as ev
    stat = oev.new_result_stat(THR3)
    for (boxes, scores, n), gt in zip(want, gts):
        if n == 0:                                   # the reference's caluclate_tp_fp with det_boxes None: the GT count only
            for t in THR3:
                ev.append_frame(stat, t, torch.zeros(0), torch.zeros(0), gt.shape[0])
        else:
            _drop_in_stat(boxes, scores, gt, THR3, stat)
    return stat


@pytest.fixture
def _isolate_opencood_modules():
    import sys
    before = {k: v for k, v in sys.modules.items() if k.startswith(("opencood", "shapely"))}
    yield
    for k in [k for k in sys.modules if k.startswith(("opencood", "shapely"))]:
        del sys.modules[k]
    sys.modules.update(before)


@pytest.mark.parametrize("depth", [1, 2])
def test_stream_result_stat_equals_the_drop_in_on_stand_alone_boxes(scene, depth, _isolate_opencood_modules):
    from heal_b200.graph import LateFusionStream
    m, params, batches, want = scene
    gts = _gts(want, params)
    expect = _want_stat(want, gts)
    with pytest.raises(ValueError, match=f"gt_capacity is {params['max_num']}"):
        LateFusionStream(m, CAPS, 5, params, depth=depth, eval_thresholds=THR3).submit(batches[1], gts[1])
    stream = LateFusionStream(m, CAPS, 5, params, depth=depth, eval_thresholds=THR3, gt_capacity=400)
    got = _run(stream, batches, [g.cuda() if i % 2 else g for i, g in enumerate(gts)])      # device or host GT
    _check(got, want, FRAMES)
    stream.drain()
    assert stream.result_stat == expect                                    # each frame once, in frame order
    assert sum(expect[0.5]["tp"]) > 0 and sum(expect[0.5]["fp"]) > 0
    calculate_ap = _calculate_ap()
    for t in THR3:
        assert calculate_ap(copy.deepcopy(stream.result_stat), t) == calculate_ap(copy.deepcopy(expect), t)


def test_refusals_leave_the_stream_untouched(scene):
    from heal_b200.graph import LateFusionStream
    m, params, batches, want = scene
    gts = _gts(want, params)
    stream = LateFusionStream(m, CAPS, 5, params, depth=2, eval_thresholds=THR3, gt_capacity=400)
    stream.submit(batches[0], gts[0])
    state = (stream.count, stream.captures, copy.deepcopy(stream.result_stat))
    six = OrderedDict(list(batches[3].items()) + [("cav5", batches[1]["ego"])])
    big = late_batch(m, [M1, M1, M1, M1], 3)                                 # four clouds of 1700 points, capacity 6000
    for cav in big.values():
        cav["inputs_m1"]["points"] = torch.zeros((1700, 4), device="cuda")
    wrong_cam = copy.copy(batches[2])
    wrong_cam["ego"] = {"inputs_m2": {**batches[2]["ego"]["inputs_m2"], "imgs": torch.zeros((1, 2, 3, 64, 96), device="cuda")},
                        "transformation_matrix": torch.eye(4)}
    for b, gt, match in ((six, gts[3], "6 cavs"), (big, gts[0], "more points than the capacity"),
                         (wrong_cam, gts[2], "captured for"), (batches[1], torch.zeros((401, 8, 3)), "gt_capacity is 400"),
                         (batches[1], None, "required")):
        with pytest.raises(ValueError, match=match):
            stream.submit(b, gt)
        assert (stream.count, stream.captures, stream.result_stat) == state
    got = _run(stream, batches[1:], gts[1:])                               # the first result is frame 0's
    _check(got, want, FRAMES)
    assert stream.result_stat == _want_stat(want, gts)


def test_no_and_single_fusion_are_ego_only_frames(scene):
    """inference_no_fusion / single: `{'ego': batch_data['ego']}` gives the ego's boxes of `forward` + box_decode_nms; the GT is
    the union of every cav's objects (no fusion) or the ego's own (single)."""
    from heal_b200 import ops
    from heal_b200.data_utils.post_processor.voxel_postprocessor import decode_kwargs
    from heal_b200.graph import LateFusionStream
    m, params, batches, want = scene
    union = _gts(want, params)
    anchors = _anchors_dev(params)
    egos, ego_want = [], []
    for b in batches:
        ego = {"ego": b["ego"]}
        with torch.no_grad():
            out = m(b["ego"])
        post = ops.box_decode_nms(out["cls_preds"], out["reg_preds"], out["dir_preds"], anchors, b["ego"]["transformation_matrix"],
                                  **decode_kwargs(params, True))
        n = int(post.count.item())
        egos.append(ego)
        ego_want.append((post.boxes[:n].cpu(), post.scores[:n].cpu(), n))
    own = [_gt_near(boxes, 150 + i, 60) for i, (boxes, _, _) in enumerate(ego_want)]
    for gts in (union, own):                                                 # no fusion, then single
        stream = LateFusionStream(m, CAPS, 5, params, depth=2, eval_thresholds=THR3, gt_capacity=400)
        _check(_run(stream, egos, gts), ego_want, [[f[0]] for f in FRAMES])
        assert stream.result_stat == _want_stat(ego_want, gts)
        assert stream.captures == 3                                          # slot 0: [m1], [m2]; slot 1: [m1]


def test_raw_camera_frames_match_the_stand_alone_graph(scene):
    from heal_b200.graph import LateFusionStream
    m, params, _, _ = scene
    frames = [[M2, M1], [M1, M2, M2], [M2, M1], [M2]]
    batches = [late_batch(m, mods, 40 + i, raw=True) for i, mods in enumerate(frames)]
    want = _stand_alone(m, RAW_CAPS, frames, batches, params)
    assert all(n > 0 for _, _, n in want)
    stream = LateFusionStream(m, RAW_CAPS, 4, params, depth=2)
    _check(_run(stream, batches), want, frames)
    with pytest.raises(ValueError, match="fp32 images for a graph captured with raw uint8 frames"):
        stream.submit(late_batch(m, [M2], 9))


def test_shared_pool_needs_less_memory_than_a_graph_per_list(scene):
    """Reserved memory of capturing the four lists into one slot against four stand-alone LateFusionGraphs."""
    from heal_b200.graph import LateFusionGraph, LateFusionStream
    m, params, batches, _ = scene
    with torch.no_grad():                       # lazily built weight caches exist before either arm is measured
        for b in batches:
            m.forward_late(b)

    def settled():
        torch.cuda.synchronize()
        gc.collect()
        torch.cuda.empty_cache()
        return torch.cuda.memory_reserved()

    r0 = settled()
    stream = LateFusionStream(m, CAPS, 5, params, depth=1, eval_thresholds=THR3, gt_capacity=400)
    for mods in LISTS:
        stream.capture(mods)
    shared = settled() - r0
    assert stream.captures == len(LISTS)
    del stream
    r1 = settled()
    graphs = [LateFusionGraph(m, mods, CAPS, params, eval_thresholds=THR3, gt_capacity=400) for mods in LISTS]
    alone = settled() - r1
    del graphs
    print(f"reserved for {len(LISTS)} lists: one shared slot {shared / 2**20:.1f} MiB, a graph per list {alone / 2**20:.1f} MiB")
    assert shared < alone, f"one shared slot {shared} B, {len(LISTS)} stand-alone LateFusionGraphs {alone} B"


def test_submit_does_not_synchronise_for_captured_lists(scene):
    from heal_b200.graph import LateFusionStream
    m, params, batches, want = scene
    gts = [g.cuda() for g in _gts(want, params)]
    stream = LateFusionStream(m, CAPS, 5, params, depth=2, eval_thresholds=THR3, gt_capacity=400)
    for mods in LISTS:
        stream.capture(mods)
    torch.cuda.synchronize()
    got = []
    torch.cuda.set_sync_debug_mode("error")
    try:
        for b, gt in zip(batches, gts):                          # host poses go through the slots' pinned staging
            r = stream.submit(b, gt)
            if r is not None:
                got.append(_copy(r))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    got += [_copy(r) for r in stream.drain()]
    _check(got, want, FRAMES)
    assert stream.result_stat == _want_stat(want, [g.cpu() for g in gts])
