"""SceneStream (heal_b200.graph): a stream of mixed-modality scenes whose agent list changes from frame to frame, one captured
graph per list and pipeline slot, the graphs of a slot sharing its memory pool and buffers.  Every frame's result must be, bit
for bit, what a SceneGraph captured for its list alone gives on the same batch."""
import copy
import gc

import numpy as np
import pytest
import torch

import scene_fixtures as sf

pytestmark = pytest.mark.gpu

HEADS = ("cls_preds", "reg_preds", "dir_preds")
A, B, C, D = ["m1", "m2", "m3", "m4", "m1"], ["m1", "m3"], ["m1"], ["m1", "m4", "m2"]
FRAMES = [A, B, C, D, A, B]                         # back to the first list, then B again
FIVE = [A, B, C, D, ["m2", "m1"]]


def stream_batch(model, aml, seed):
    """The collated ego batch of a scene of any agent list over `model`'s modalities, as scene_fixtures.scene_batch makes them:
    raw clouds (a 32-ring cloud for SECOND), two-camera rigs with fp32 images, poses padded to max_cav 5."""
    from workloads import synth
    rng = np.random.default_rng(300 + seed)
    batch = {"agent_modality_list": list(aml), "record_len": torch.tensor([len(aml)])}
    for m in dict.fromkeys(aml):
        k = aml.count(m)
        if model.sensor_type_dict[m] == "lidar":
            clouds = [synth.lidar_cloud(rng, 32, 256) if m == "m3" else sf._cloud(rng, int(rng.integers(1200, 2200)))
                      for _ in range(k)]
            offs = np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds])]).astype(np.int32)
            batch[f"inputs_{m}"] = {"points": torch.from_numpy(np.concatenate(clouds)).cuda(),
                                    "agent_offsets": torch.from_numpy(offs).cuda()}
        else:
            rots, trans, intr, post_rots, post_trans = [torch.from_numpy(a).cuda() for a in synth.camera_rig(k, sf.CAMS, sf.IMG_H, sf.IMG_W)]
            trans = trans + torch.from_numpy(rng.uniform(-0.3, 0.3, tuple(trans.shape)).astype(np.float32)).cuda()
            imgs = torch.randn(k, sf.CAMS, 3, sf.IMG_H, sf.IMG_W, generator=torch.Generator().manual_seed(2000 + seed))
            batch[f"inputs_{m}"] = {"imgs": imgs.cuda(), "rots": rots, "trans": trans, "intrins": intr, "post_rots": post_rots,
                                    "post_trans": post_trans}
    poses = [[0, 0, 0, 0, 0, 0]] + [[rng.uniform(-5, 5), rng.uniform(-5, 5), 0, 0, rng.uniform(-180, 180), 0]
                                    for _ in range(len(aml) - 1)]
    batch["pairwise_t_matrix"] = torch.from_numpy(synth.pairwise_t_matrix(poses, 5)[None]).cuda()
    return batch


def _stand_alone(m, caps, frames, batches, params):
    """Per frame, what a SceneGraph captured for that list alone gives on the same batch: heads, and with `params` the ego's
    boxes[:count], scores[:count] and count."""
    from heal_b200.graph import SceneGraph
    graphs, want = {}, []
    for aml, batch in zip(frames, batches):
        g = graphs.get(tuple(aml))
        if g is None:
            g = graphs[tuple(aml)] = SceneGraph(m, aml, caps, sf.PAIRWISE_SHAPE, params)
        g.load(batch)
        out = g.replay()
        torch.cuda.synchronize()
        w = {k: out[k].cpu() for k in HEADS}
        if params is not None:
            n = int(out["postprocess"].count.item())
            w.update(boxes=out["postprocess"].boxes[:n].cpu(), scores=out["postprocess"].scores[:n].cpu(), count=n)
        want.append(w)
    return want


def _run(stream, batches):
    got = []
    for b in batches:
        r = stream.submit(b)
        if r is not None:
            got.append(_copy(r))
    return got + [_copy(r) for r in stream.drain()]


def _copy(r):
    return {k: (v.clone() if torch.is_tensor(v) else v) for k, v in r.items()}


def _same(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(a, b)


def _check(got, want, frames, boxes):
    assert len(got) == len(frames)
    for i, (r, w, aml) in enumerate(zip(got, want, frames)):
        assert r["agent_modality_list"] == aml, i                         # results come back in submission order
        if boxes:
            assert set(r) == {"boxes", "scores", "count", "agent_modality_list"}
            n = int(r["count"][0])
            assert n == w["count"], (i, aml)
            assert _same(r["boxes"][:n], w["boxes"]) and _same(r["scores"][:n], w["scores"]), (i, aml)
        else:
            assert set(r) == set(HEADS) | {"agent_modality_list"}
            for k in HEADS:
                assert _same(r[k], w[k]), (i, aml, k)


@pytest.fixture(scope="module")
def four():
    m, params = sf.model("four"), sf.postprocess_params()
    batches = [stream_batch(m, aml, i) for i, aml in enumerate(FRAMES)]
    return m, params, batches, _stand_alone(m, sf.capacities("four"), FRAMES, batches, params)


@pytest.mark.parametrize("depth", [1, 2])
@pytest.mark.parametrize("boxes", [True, False])
def test_stream_of_changing_agent_lists_equals_stand_alone_graphs(four, depth, boxes):
    from heal_b200.graph import SceneStream
    m, params, batches, want = four
    stream = SceneStream(m, sf.capacities("four"), sf.PAIRWISE_SHAPE, postprocess_params=params if boxes else None, depth=depth)
    got = _run(stream, batches)
    _check(got, want, FRAMES, boxes)
    # each slot captured each of its lists once: depth 1 sees A B C D, depth 2 slot 0 sees A C A and slot 1 B D B
    assert stream.captures == 4 and stream.graphs_captured == 4
    again = _run(stream, batches)               # every list replayed after the others; at depth 2 the first result is frame 5
    _check(again[depth - 1:], want, FRAMES, boxes)
    assert stream.captures == 4


def test_a_list_replays_its_own_bits_after_other_lists_in_its_slot(four):
    """Slot 0 alone (depth 1): A after B, C and D have replayed out of the same pool, and B after A again."""
    from heal_b200.graph import SceneStream
    m, params, batches, want = four
    stream = SceneStream(m, sf.capacities("four"), sf.PAIRWISE_SHAPE, postprocess_params=params, depth=1)
    for aml in reversed(FIVE[:4]):                                          # captured ahead: A last, over the others' scratch
        stream.capture(aml)
    assert stream.captures == 4
    order = [4, 0, 1, 2, 3, 5, 0, 4]
    got = [_copy(stream.submit(batches[i])) for i in order]
    _check(got, [want[i] for i in order], [FRAMES[i] for i in order], True)
    assert stream.captures == 4


def test_eviction_at_max_graphs_recaptures_and_still_matches(four):
    from heal_b200.graph import SceneStream
    m, params, batches, want = four
    stream = SceneStream(m, sf.capacities("four"), sf.PAIRWISE_SHAPE, postprocess_params=params, depth=1, max_graphs=2)
    order = [0, 1, 0, 2, 1, 4]                                             # A B A C (drops B) B (drops A) A (drops C)
    got = _run(stream, [batches[i] for i in order])
    _check(got, [want[i] for i in order], [FRAMES[i] for i in order], True)
    assert stream.captures == 5 and stream.graphs_captured == 2
    assert list(stream.cache.slots[0]) == [tuple(B), tuple(A)]


def test_refusals_leave_the_stream_untouched(four):
    from heal_b200.graph import SceneStream
    m, params, batches, _ = four
    stream = SceneStream(m, sf.capacities("four"), sf.PAIRWISE_SHAPE, postprocess_params=params, depth=2)
    six = {**batches[0], "agent_modality_list": A + ["m1"]}
    with pytest.raises(ValueError, match="6 agents"):
        stream.submit(six)
    with pytest.raises(ValueError, match="agent modality 'm5'"):
        stream.submit({**batches[1], "agent_modality_list": ["m1", "m5"]})
    big = {**batches[1], "inputs_m1": {**batches[1]["inputs_m1"], "points": torch.zeros((sf.LIDAR_CAPACITY + 1, 4), device="cuda")}}
    with pytest.raises(ValueError, match="capacity"):
        stream.submit(big)
    assert stream.count == 0 and stream.captures == 0
    no_m3 = {k: v for k, v in sf.capacities("four").items() if k != "m3"}
    s2 = SceneStream(m, no_m3, sf.PAIRWISE_SHAPE, depth=1)
    with pytest.raises(ValueError, match="m3: no capacity"):
        s2.submit(batches[1])
    assert s2.captures == 0


def test_shared_pool_needs_less_memory_than_a_graph_per_list(four):
    """Reserved memory of capturing five lists into one slot against five stand-alone SceneGraphs."""
    from heal_b200.graph import SceneGraph, SceneStream
    m, params, _, _ = four
    caps = sf.capacities("four")
    with torch.no_grad():                       # lazily built weight caches exist before either arm is measured
        for i, aml in enumerate(FIVE):
            m(stream_batch(m, aml, 50 + i))

    def settled():
        torch.cuda.synchronize()
        gc.collect()
        torch.cuda.empty_cache()
        return torch.cuda.memory_reserved()

    r0 = settled()
    stream = SceneStream(m, caps, sf.PAIRWISE_SHAPE, postprocess_params=params, depth=1)
    for aml in FIVE:
        stream.capture(aml)
    shared = settled() - r0
    assert stream.captures == 5
    del stream
    r1 = settled()
    graphs = [SceneGraph(m, aml, caps, sf.PAIRWISE_SHAPE, params) for aml in FIVE]
    alone = settled() - r1
    del graphs
    print(f"reserved for five lists: one shared slot {shared / 2**20:.1f} MiB, a SceneGraph per list {alone / 2**20:.1f} MiB")
    assert shared < alone, f"one shared slot {shared} B, five stand-alone SceneGraphs {alone} B"


def _ms_model():
    from heal_b200.models.heter_model_baseline_ms import HeterModelBaselineMs
    from oracle import coalign, procedural
    from oracle import efficientnet as oe
    m = HeterModelBaselineMs(copy.deepcopy(coalign.hetero_args())).eval()
    m.load_state_dict(oe.state_dict_of(procedural.shapes_of(m)), strict=True)
    return m.cuda()


@pytest.mark.parametrize("kind", ["baseline", "baseline_ms"])
def test_heter_model_baseline_streams(kind):
    """HeterModelBaseline (att) with boxes back and HeterModelBaselineMs with heads back, one list change each."""
    from heal_b200.graph import SceneStream
    if kind == "baseline":
        m, params, caps = sf.model("baseline"), sf.postprocess_params(), sf.capacities("baseline")
        lists = [["m2", "m1", "m2"], ["m2", "m1", "m2"], ["m1", "m2"], ["m1", "m2"]]
    else:
        m, params, caps = _ms_model(), None, {"m1": sf.LIDAR_CAPACITY, "m4": (sf.CAMS, sf.IMG_H, sf.IMG_W)}
        lists = [["m1", "m4", "m1"], ["m1", "m4", "m1"], ["m1", "m4"], ["m1", "m4"]]
    batches = [stream_batch(m, aml, 20 + i) for i, aml in enumerate(lists)]
    want = _stand_alone(m, caps, lists, batches, params)
    stream = SceneStream(m, caps, sf.PAIRWISE_SHAPE, postprocess_params=params, depth=2)
    _check(_run(stream, batches), want, lists, params is not None)
    assert stream.captures == 4
