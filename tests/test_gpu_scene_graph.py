"""SceneGraph and the scene pipelines (heal_b200.graph): a mixed-modality intermediate-fusion frame captured once and replayed
for scenes of other point counts, poses and camera frames, against the eager model and the GPU post-processor, bit for bit."""
import pytest
import torch

import scene_fixtures as sf

pytestmark = pytest.mark.gpu

HEADS = ("cls_preds", "reg_preds", "dir_preds")


def _eager(m, batch, params=None):
    """The eager heads and, with `params`, the GPU post-processor's (boxes, scores) of the ego."""
    from heal_b200.data_utils.post_processor.voxel_postprocessor import VoxelPostprocessor
    with torch.no_grad():
        out = m(batch)
        heads = {k: out[k].clone() for k in HEADS}
        boxes = None
        if params is not None:
            pp = VoxelPostprocessor(params, False)
            b, s = pp.post_process({"ego": {"anchor_box": pp.generate_anchor_box(), "transformation_matrix": torch.eye(4)}},
                                   {"ego": out})
            boxes = (b.clone(), s.clone()) if b is not None else (torch.zeros((0, 8, 3)), torch.zeros((0,)))
    torch.cuda.synchronize()
    return heads, boxes


def _same(a, b):
    return a.shape == b.shape and torch.equal(a.cpu(), b.cpu())


def _check_boxes(got_boxes, got_scores, count, want):
    k = int(count)
    assert k == want[0].shape[0]
    assert _same(got_boxes[:k], want[0]) and _same(got_scores[:k], want[1])


@pytest.mark.parametrize("kind", ["c4", "four"])
def test_scene_graph_replays_equal_eager(kind):
    from heal_b200.graph import SceneGraph
    m, params = sf.model(kind), sf.postprocess_params()
    scenes = [sf.scene_batch(kind, s) for s in (1, 2, 3)]
    assert len({int(sc["inputs_m1"]["agent_offsets"][-1]) for sc in scenes}) == 3       # different point counts
    want = [_eager(m, sc, params) for sc in scenes]
    g = SceneGraph(m, sf.AML[kind], sf.capacities(kind), sf.PAIRWISE_SHAPE, params)
    print(f"SceneGraph {kind}: {g.kernels_per_replay} kernels per replay")
    for i in (2, 0, 1, 2, 1):                                                           # out of order, repeated
        g.load(scenes[i])
        out = g.replay()
        torch.cuda.synchronize()
        for k in HEADS:
            assert _same(out[k], want[i][0][k]), (kind, i, k)
        buf = out["postprocess"]
        _check_boxes(buf.boxes, buf.scores, buf.count.item(), want[i][1])


@pytest.mark.parametrize("kind", ["c4", "four"])
def test_raw_frames_give_the_bits_of_the_fp32_images(kind):
    """A graph fed uint8 frames equals the eager model fed the fp32 images heal_camera_input makes of them."""
    from heal_b200 import ops
    from heal_b200.graph import SceneGraph
    m = sf.model(kind)
    raw = [sf.scene_batch(kind, s, raw=True) for s in (4, 5)]
    g = SceneGraph(m, sf.AML[kind], sf.capacities(kind, raw=True), sf.PAIRWISE_SHAPE)
    for sc in raw:
        fp32 = {k: (dict(v) if isinstance(v, dict) else v) for k, v in sc.items()}
        for mod in dict.fromkeys(sf.AML[kind]):
            imgs = sc[f"inputs_{mod}"].get("imgs")
            if imgs is None:
                continue
            k, n, H0, W0, _ = imgs.shape
            plan = getattr(m, f"encoder_{mod}").camera_plan(H0, W0)
            fp32[f"inputs_{mod}"]["imgs"] = ops.camera_input(imgs.reshape(k * n, H0, W0, 3), plan, "nchw").reshape(
                k, n, 3, sf.IMG_H, sf.IMG_W)
        want, _ = _eager(m, fp32)
        g.load(sc)
        out = g.replay()
        torch.cuda.synchronize()
        for key in HEADS:
            assert _same(out[key], want[key]), (kind, key)


@pytest.mark.parametrize("depth,boxes", [(2, True), (3, False)])
def test_frame_pipeline_over_a_scene(depth, boxes):
    from heal_b200.graph import FramePipeline
    m = sf.model("four")
    params = sf.postprocess_params() if boxes else None
    scenes = [sf.scene_batch("four", s) for s in (1, 2, 3, 6, 7)]
    want = [_eager(m, sc, params) for sc in scenes]
    pipe = FramePipeline.for_scene(m, sf.AML["four"], sf.capacities("four"), sf.PAIRWISE_SHAPE, postprocess_params=params,
                                   depth=depth)
    got = []
    for sc in scenes:
        r = pipe.submit(sc)
        if r is not None:
            got.append({k: v.clone() for k, v in r.items()})
    got += [{k: v.clone() for k, v in r.items()} for r in pipe.drain()]
    assert len(got) == len(scenes)
    for i, (r, (heads, bx)) in enumerate(zip(got, want)):
        if boxes:
            assert set(r) == {"boxes", "scores", "count"}
            _check_boxes(r["boxes"], r["scores"], r["count"][0], bx)
        else:
            for k in HEADS:
                assert _same(r[k], heads[k]), (i, k)
    per_frame = sum(t.numel() * t.element_size() for t in pipe.host_out[0].values())
    assert pipe.d2h_bytes == per_frame
    print(f"FramePipeline depth {depth}: {per_frame} bytes back per frame ({'boxes' if boxes else 'heads'})")


def test_frame_interleaver_over_a_scene():
    from heal_b200.graph import FrameInterleaver
    m = sf.model("c4")
    scenes = [sf.scene_batch("c4", s) for s in (1, 2, 3)]
    want = [_eager(m, sc)[0] for sc in scenes]
    il = FrameInterleaver.for_scene(m, sf.AML["c4"], sf.capacities("c4"), sf.PAIRWISE_SHAPE, n=2)
    for i, sc in enumerate(scenes):
        out = il.submit(sc)
        il.join(begin=False)
        torch.cuda.synchronize()
        for k in HEADS:
            assert _same(out[k], want[i][k]), (i, k)


def test_scene_graph_on_heter_model_baseline_att():
    from heal_b200.graph import SceneGraph
    m, params = sf.model("baseline"), sf.postprocess_params()
    scenes = [sf.scene_batch("baseline", s) for s in (1, 2, 3)]
    want = [_eager(m, sc, params) for sc in scenes]
    g = SceneGraph(m, sf.AML["baseline"], sf.capacities("baseline"), sf.PAIRWISE_SHAPE, params)
    for i in (1, 2, 0):
        g.load(scenes[i])
        out = g.replay()
        torch.cuda.synchronize()
        for k in HEADS:
            assert _same(out[k], want[i][0][k]), (i, k)
        _check_boxes(out["postprocess"].boxes, out["postprocess"].scores, out["postprocess"].count.item(), want[i][1])


def test_scene_graph_load_refusals():
    from heal_b200.graph import SceneGraph
    m = sf.model("c4")
    g = SceneGraph(m, sf.AML["c4"], sf.capacities("c4"), sf.PAIRWISE_SHAPE)
    sc = sf.scene_batch("c4", 1)
    with pytest.raises(ValueError, match="captured for"):
        g.load({**sc, "agent_modality_list": ["m1", "m2", "m1"]})
    big = {**sc, "inputs_m1": {"points": torch.zeros((sf.LIDAR_CAPACITY + 1, 4), device="cuda"),
                               "agent_offsets": sc["inputs_m1"]["agent_offsets"]}}
    with pytest.raises(ValueError, match="capacity"):
        g.load(big)
    raw = sf.scene_batch("c4", 1, raw=True)
    with pytest.raises(ValueError, match="raw uint8 frames for a graph captured with normalised fp32 images"):
        g.load(raw)
