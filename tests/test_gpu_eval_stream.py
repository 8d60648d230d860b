"""Evaluation inside the captured scene path: heal_eval_tp_fp_counted (counts on the device, sizes from capacities) against
heal_eval_tp_fp bit for bit, alone and replayed in a captured graph with new counts; SceneGraph, FramePipeline.for_scene and
LateFusionGraph with `eval_thresholds` against the eval_utils drop-in (what install_gpu_eval() binds) on the graphs' own boxes;
and SceneStream's `result_stat` over the changing-list stream against the one built frame by frame from stand-alone graphs."""
import copy
import os

import numpy as np
import pytest
import torch

import scene_fixtures as sf
from oracle import eval as oev
from oracle import ref_shim
from oracle.make_golden_eval import random_frame, rect
from test_gpu_scene_stream import FRAMES, stream_batch

pytestmark = pytest.mark.gpu

THR3 = (0.3, 0.5, 0.7)
THR8 = (0.3, 0.5, 0.7, 0.1, 0.25, 0.45, 0.6, 0.85)
K_CAP, G_CAP = 1000, 300
SENTINEL = 0xA5


def _bits(t):
    return t.contiguous().view(torch.int32).cpu()


def _plain(det, score, gt, thresholds):
    """heal_eval_tp_fp on the live rows: (status, scores (K,), tp (n_thr, K)) on the host."""
    from heal_b200 import ops
    buf = ops.eval_tp_fp(det.contiguous(), score.contiguous(), gt.contiguous(), thresholds)
    return ops.EvalBuffers.unpack(buf.packed.cpu(), det.shape[0], len(thresholds))


class Counted:
    """Static capacity buffers for heal_eval_tp_fp_counted; `put` writes a frame's live rows over garbage."""

    def __init__(self, thresholds, k_cap=K_CAP, g_cap=G_CAP):
        from heal_b200 import ops
        self.thr, self.k_cap, self.g_cap = thresholds, k_cap, g_cap
        self.det = torch.zeros((k_cap, 8, 3), device="cuda")
        self.score = torch.zeros((k_cap,), device="cuda")
        self.gt = torch.zeros((g_cap, 8, 3), device="cuda")
        self.k = torch.zeros((1,), dtype=torch.int32, device="cuda")
        self.g = torch.zeros((1,), dtype=torch.int32, device="cuda")
        self.buf = ops.EvalBuffers(k_cap, g_cap, "cuda")

    def put(self, det, score, gt, seed, k=None, g=None):
        gen = torch.Generator(device="cuda").manual_seed(seed)
        self.det.copy_(torch.randn(self.det.shape, generator=gen, device="cuda") * 20)        # garbage past the live rows
        self.score.copy_(torch.randn(self.score.shape, generator=gen, device="cuda"))
        self.score[::7] = float("nan")
        self.gt.copy_(torch.randn(self.gt.shape, generator=gen, device="cuda") * 20)
        self.det[:det.shape[0]] = det
        self.score[:det.shape[0]] = score
        self.gt[:gt.shape[0]] = gt
        self.k.fill_(det.shape[0] if k is None else k)
        self.g.fill_(gt.shape[0] if g is None else g)
        self.buf.out.fill_(SENTINEL)

    def run(self):
        from heal_b200 import ops
        return ops.eval_tp_fp_counted(self.det, self.score, self.k, self.gt, self.g, self.thr, self.buf)

    def result(self, K):
        from heal_b200 import ops
        packed = self.buf.packed.cpu()
        assert packed.numel() == 4 + 4 * self.k_cap + len(self.thr) * self.k_cap
        status, s, tp = ops.EvalBuffers.unpack(packed, self.k_cap, len(self.thr))
        # nothing is written past the live count
        assert (s[K:].view(torch.uint8) == SENTINEL).all() and (tp[:, K:] == SENTINEL).all()
        return status, s[:K], tp[:, :K]


def _same(got, want, what):
    assert got[0] == want[0], (what, got[0], want[0])
    assert torch.equal(_bits(got[1]), _bits(want[1])), what
    if want[0] == 0:
        assert torch.equal(got[2], want[2]), (what, (got[2] != want[2]).nonzero()[:5])


def _cuda(a):
    return torch.as_tensor(np.asarray(a, dtype=np.float32)).cuda()


def _frames():
    """(name, det (K,8,3), score (K,), gt (G,8,3)) on the GPU: K in {0, 1, 37, 1000}, G in {0, 1, 57, G_CAP}, with tied and NaN
    scores in some; a zero-union frame."""
    out = []
    for i, K in enumerate((0, 1, 37, 1000)):
        for j, G in enumerate((0, 1, 57, G_CAP)):
            seed = 10 * i + j
            det, score, gt = random_frame(seed, max(K, 1), max(G, 1), "hwl" if seed % 2 else "lwh", bool(seed % 3 == 0))
            det, score, gt = det[:K], np.asarray(score, np.float32)[:K].copy(), gt[:G]
            if seed % 2 and K > 1:
                score = np.float32([0.9, 0.6, 0.3])[np.arange(K) % 3]                       # ties
                score[::11] = np.nan
            out.append((f"k{K}_g{G}", _cuda(det).reshape(-1, 8, 3), _cuda(score).reshape(-1), _cuda(gt).reshape(-1, 8, 3)))
    point, segment = np.zeros((1, 8, 3), np.float32), rect(0, 4, 0, 0)[None]
    out.append(("zero_union", _cuda(np.concatenate([point, rect(0, 1, 0, 1)[None]])), _cuda([0.5, 0.7]),
                _cuda(np.concatenate([segment, rect(0, 1, 0, 1)[None]]))))
    return out


@pytest.fixture(scope="module")
def golden(golden_dir):
    return torch.load(os.path.join(golden_dir, "eval_tp_fp.pt"), weights_only=False)


@pytest.mark.parametrize("thresholds", [THR3, THR8], ids=["3thr", "8thr"])
def test_counted_equals_the_host_count_entry(golden, thresholds):
    c = Counted(thresholds)
    frames = [(f["name"], f["det"].cuda(), f["score"].cuda(), f["gt"].cuda()) for f in golden["frames"] if f["det"] is not None]
    statuses = set()
    for n, (name, det, score, gt) in enumerate(frames + _frames()):
        want = _plain(det, score, gt, thresholds)
        c.put(det, score, gt, seed=n)
        c.run()
        got = c.result(det.shape[0])
        _same(got, want, name)
        statuses.add(got[0])
    assert statuses == {0, 1}


def test_counted_replays_in_a_captured_graph_with_new_counts():
    c = Counted(THR3)
    frames = _frames()
    name, det, score, gt = frames[-2]                        # K = 1000, G = G_CAP for the warm-up and the capture
    c.put(det, score, gt, seed=0)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        c.run()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        c.run()
    for n in (5, 0, 9, 15, 3, 16, 12, 15):                  # new counts every replay, one frame twice
        name, det, score, gt = frames[n]
        c.put(det, score, gt, seed=100 + n)
        graph.replay()
        torch.cuda.synchronize()
        _same(c.result(det.shape[0]), _plain(det, score, gt, THR3), name)


def test_over_capacity_sets_its_bit_and_writes_no_flag():
    from heal_b200 import ops
    c = Counted(THR3, k_cap=64, g_cap=32)
    _, det, score, gt = _frames()[10]                        # K = 37, G = 57
    for k, g in ((37, 32), (65, 5), (37, 33), (-1, 5), (37, -1)):
        c.put(det[:min(max(k, 0), 64)], score[:min(max(k, 0), 64)], gt[:min(max(g, 0), 32)], seed=1, k=k, g=g)
        c.run()
        over = not (0 <= k <= 64 and 0 <= g <= 32)
        status, s, tp = ops.EvalBuffers.unpack(c.buf.packed.cpu(), 64, 3)
        assert status == (2 if over else 0), (k, g, status)
        if over:
            assert (s.view(torch.uint8) == SENTINEL).all() and (tp == SENTINEL).all()
    with pytest.raises(ValueError, match="buffers for K=64"):
        ops.eval_tp_fp_counted(torch.zeros((65, 8, 3), device="cuda"), torch.zeros(65, device="cuda"), c.k, c.gt, c.g, THR3, c.buf)
    with pytest.raises(RuntimeError):
        ops.eval_tp_fp_counted(torch.zeros((4097, 8, 3), device="cuda"), torch.zeros(4097, device="cuda"), c.k, c.gt, c.g, THR3)


# ---- captured frames that evaluate their boxes ------------------------------------------------------------------------------

def _gt_near(boxes, seed, cap):
    """GT corners for a frame: every third detection moved by up to ~0.6 m (some stay matches at 0.3 / 0.5 / 0.7, some do not)
    and a few boxes elsewhere, at most `cap`."""
    rng = np.random.default_rng(seed)
    near = boxes[::3].cpu().numpy()
    near = near + rng.uniform(-0.6, 0.6, (near.shape[0], 1, 3)).astype(np.float32) * np.float32([1, 1, 0])
    far = [rect(x, x + 4, y, y + 1.8) for x, y in rng.uniform(-12, 8, (5, 2))]
    gt = np.concatenate([near.reshape(-1, 8, 3), np.stack(far)]).astype(np.float32)[:cap]
    return torch.from_numpy(gt)


def _drop_in_stat(boxes, scores, gt, thresholds, stat=None):
    """The frame through the eval_utils drop-in (the function install_gpu_eval() puts into opencood.utils.eval_utils)."""
    from heal_b200.utils import eval_utils as ev
    stat = oev.new_result_stat(thresholds) if stat is None else stat
    for t in thresholds:
        ev.caluclate_tp_fp(boxes.cuda().contiguous(), scores.cuda().contiguous(), gt.cuda(), stat, t)
    return stat


def test_scene_graph_and_pipeline_evaluate_their_own_boxes():
    from heal_b200.graph import FramePipeline, SceneGraph
    from heal_b200.utils import eval_utils as ev
    m, params = sf.model("four"), sf.postprocess_params()
    caps = sf.capacities("four")
    scenes = [sf.scene_batch("four", s) for s in (1, 2, 3, 6)]
    plain = SceneGraph(m, sf.AML["four"], caps, sf.PAIRWISE_SHAPE, params)
    boxes = []
    for sc in scenes:
        plain.load(sc)
        out = plain.replay()["postprocess"]
        n = int(out.count.item())
        boxes.append((out.boxes[:n].clone(), out.scores[:n].clone()))
    gts = [_gt_near(b, i, 150) for i, (b, _) in enumerate(boxes)]
    gts[2] = gts[2][:0]                                                    # a frame without GT
    g = SceneGraph(m, sf.AML["four"], caps, sf.PAIRWISE_SHAPE, params, eval_thresholds=THR3)     # gt_capacity: max_num
    assert g.gt_capacity == params["max_num"]
    print(f"SceneGraph with evaluation: {g.kernels_per_replay} kernels per replay (without: {plain.kernels_per_replay})")
    assert g.kernels_per_replay == plain.kernels_per_replay + 4
    want_total = oev.new_result_stat(THR3)
    for i in (0, 1, 2, 3, 1):
        g.load(scenes[i], gt_boxes=gts[i].cuda() if i % 2 else gts[i])     # device or host GT
        out = g.replay()
        torch.cuda.synchronize()
        n = int(out["postprocess"].count.item())
        assert n == boxes[i][0].shape[0] and torch.equal(out["postprocess"].boxes[:n], boxes[i][0])
        got = oev.new_result_stat(THR3)
        r = g.results()
        ev.append_packed(got, THR3, r["eval"].cpu(), n, r["scores"].shape[0], int(r["gt_count"].item()))
        want = _drop_in_stat(*boxes[i], gts[i], THR3)
        assert got == want, i
        assert sum(want[0.3]["tp"]) > 0 or n == 0 or gts[i].shape[0] == 0
    with pytest.raises(ValueError, match="gt_boxes .* required"):
        g.load(scenes[0])
    with pytest.raises(ValueError, match="gt_capacity is 150"):
        g.load(scenes[0], gt_boxes=torch.zeros((151, 8, 3)))
    with pytest.raises(ValueError, match="without eval_thresholds"):
        plain.load(scenes[0], gt_boxes=gts[0])
    with pytest.raises(ValueError, match="needs postprocess_params"):
        SceneGraph(m, sf.AML["four"], caps, sf.PAIRWISE_SHAPE, None, eval_thresholds=THR3, gt_capacity=10)
    # the pipeline over the same scenes: result_stat in frame order, each frame once (flush after drain adds nothing)
    pipe = FramePipeline.for_scene(m, sf.AML["four"], caps, sf.PAIRWISE_SHAPE, postprocess_params=params, depth=2,
                                   eval_thresholds=THR3, gt_capacity=200)
    for i in range(4):
        r = pipe.submit(scenes[i], gts[i])
        assert set(r or {}) <= {"boxes", "scores", "count", "eval", "gt_count"}
        _drop_in_stat(*boxes[i], gts[i], THR3, want_total)
    pipe.drain()
    pipe.flush()
    assert pipe.result_stat == want_total
    assert pipe.d2h_bytes == 1000 * 8 * 3 * 4 + 1000 * 4 + 4 + (4 + 1000 * 4 + 3 * 1000) + 4


def test_late_fusion_graph_evaluates_its_own_boxes(golden_dir):
    from heal_b200 import engine
    from heal_b200.graph import LateFusionGraph
    from heal_b200.utils import eval_utils as ev
    from oracle import golden, late
    from test_gpu_late import _raw_scene, _scene_model
    old = engine.PRECISION
    engine.set_precision("tc32")
    try:
        g = golden.load(os.path.join(golden_dir, "late_fusion_scene_small.pt"))
        m, _ = _scene_model(g)
        params = {k: v for k, v in g["params"].items() if k != "max_num"}
        with pytest.raises(ValueError, match="no 'max_num'"):
            LateFusionGraph(m, ["m1"] * 3, {"m1": 3 * 1500}, params, eval_thresholds=THR3)
        plain = LateFusionGraph(m, ["m1"] * 3, {"m1": 3 * 1500}, params)
        lg = LateFusionGraph(m, ["m1"] * 3, {"m1": 3 * 1500}, params, eval_thresholds=THR3, gt_capacity=400)
        poses_b = ((0.0, 0.0, 0.0), (-6.0, 1.0, 80.0), (3.0, 5.0, 170.0))
        for i, poses in enumerate((late.SCENE_POSES, poses_b, late.SCENE_POSES)):
            scene = _raw_scene(poses)
            plain.load(scene)
            out = plain.replay()
            k = int(out.count.item())
            boxes, scores = out.boxes[:k].clone(), out.scores[:k].clone()
            gt = _gt_near(boxes, 40 + i, 400)
            lg.load(scene, gt)
            out = lg.replay()
            torch.cuda.synchronize()
            assert int(out.count.item()) == k > 0 and torch.equal(out.boxes[:k], boxes)
            got = oev.new_result_stat(THR3)
            ev.append_packed(got, THR3, lg.eval.buffers.packed.cpu(), k, 1000, gt.shape[0])
            want = _drop_in_stat(boxes, scores, gt, THR3)
            assert got == want, i
            assert sum(want[0.5]["tp"]) > 0
    finally:
        engine.set_precision(old)


# ---- SceneStream over the changing-list stream ------------------------------------------------------------------------------

def _calculate_ap():
    """The reference's calculate_ap when its package is built, else the restatement pinned to it (oracle/eval.py)."""
    if ref_shim.available():
        from oracle.make_golden_eval import install_reference
        return install_reference().calculate_ap
    return oev.calculate_ap


@pytest.fixture(scope="module")
def four_eval():
    from heal_b200.graph import SceneGraph
    m, params = sf.model("four"), sf.postprocess_params()
    caps = sf.capacities("four")
    batches = [stream_batch(m, aml, i) for i, aml in enumerate(FRAMES)]
    graphs, want, gts = {}, oev.new_result_stat(THR3), []
    for i, (aml, b) in enumerate(zip(FRAMES, batches)):
        g = graphs.get(tuple(aml))
        if g is None:
            g = graphs[tuple(aml)] = SceneGraph(m, aml, caps, sf.PAIRWISE_SHAPE, params)
        g.load(b)
        out = g.replay()["postprocess"]
        n = int(out.count.item())
        gts.append(_gt_near(out.boxes[:n], 70 + i, 120))
        _drop_in_stat(out.boxes[:n].clone(), out.scores[:n].clone(), gts[-1], THR3, want)
    return m, params, caps, batches, gts, want


@pytest.fixture
def _isolate_opencood_modules():
    import sys
    before = {k: v for k, v in sys.modules.items() if k.startswith(("opencood", "shapely"))}
    yield
    for k in [k for k in sys.modules if k.startswith(("opencood", "shapely"))]:
        del sys.modules[k]
    sys.modules.update(before)


@pytest.mark.parametrize("depth", [1, 2])
def test_stream_result_stat_equals_stand_alone_graphs(four_eval, depth, _isolate_opencood_modules):
    from heal_b200.graph import SceneStream
    m, params, caps, batches, gts, want = four_eval
    stream = SceneStream(m, caps, sf.PAIRWISE_SHAPE, postprocess_params=params, depth=depth, eval_thresholds=THR3,
                         gt_capacity=120)
    got = []
    for b, gt in zip(batches, gts):
        r = stream.submit(b, gt)
        if r is not None:
            got.append(r["agent_modality_list"])
    got += [r["agent_modality_list"] for r in stream.drain()]
    assert got == FRAMES
    stream.drain()
    assert stream.result_stat == want                                       # a second drain appends nothing
    assert sum(want[0.5]["tp"]) > 0 and sum(want[0.5]["fp"]) > 0
    calculate_ap = _calculate_ap()
    for t in THR3:
        assert calculate_ap(copy.deepcopy(stream.result_stat), t) == calculate_ap(copy.deepcopy(want), t)
    with pytest.raises(ValueError, match="gt_capacity is 120"):
        stream.submit(batches[0], torch.zeros((121, 8, 3)))
    with pytest.raises(ValueError, match="gt_boxes .* required"):
        stream.submit(batches[0])
    assert stream.count == len(FRAMES) and stream.result_stat == want
