"""CUDA-graph capture of one frame.  The per-frame path issues ~80-150 short kernels; replaying them as one graph
removes the Python / launch overhead (SURVEY.md 7.1 step 10).  Everything on the raw-points path is capture-safe: no host
syncs (voxel counts stay on the device), caller-independent workspaces, TMA descriptors baked against graph-pool buffers.

The scene shape (number of agents, point-buffer capacity, pairwise matrix shape) is fixed per graph; the live point count
travels in `agent_offsets[-1]` on the device, so clouds of different sizes reuse the same graph.
"""
from __future__ import annotations

import collections
import numbers

import torch

from . import ops
from ._lib import lib
from .data_utils.post_processor.voxel_postprocessor import TOP, VoxelPostprocessor, decode_kwargs


def warm_up(run, device):
    """Two eager calls of `run` on a side stream under no_grad, then a device synchronise: the first launches load modules and
    build lazy caches outside any capture, and outside a capture's private memory pool."""
    side = torch.cuda.Stream(device=device)
    side.wait_stream(torch.cuda.current_stream(device))
    with torch.cuda.stream(side), torch.no_grad():
        for _ in range(2):
            run()
    torch.cuda.current_stream(device).wait_stream(side)
    torch.cuda.synchronize(device)


def record(run, pool=None):
    """Capture one call of `run` into a CUDA graph, in the private memory pool `pool` (torch.cuda.graph_pool_handle()) when
    given.  Returns (graph, the output of `run`, kernels launched per replay)."""
    graph = torch.cuda.CUDAGraph()
    l0 = lib.heal_launch_count()
    with torch.no_grad(), torch.cuda.graph(graph, pool=pool, capture_error_mode="thread_local"):
        out = run()
    return graph, out, int(lib.heal_launch_count() - l0)


def capture(run, device, pool=None):
    """`warm_up` then `record`: (graph, output, kernels per replay) of `run`."""
    warm_up(run, device)
    return record(run, pool)


def _heads(out):
    """The heads of a model's output dict, by name."""
    return {k: out[k] for k in ("cls_preds", "reg_preds", "dir_preds") if k in out}


def _anchors(postprocess_params, device):
    """VoxelPostprocessor's anchor grid (H, W, A, 7) for `postprocess_params`, fp32 on `device`."""
    grid = VoxelPostprocessor(postprocess_params, False).generate_anchor_box()
    return torch.from_numpy(grid).to(device=device, dtype=torch.float32).contiguous()


def _join(device, streams, begin: bool):
    """Order `streams` after (begin) / before (end) the current stream of `device`, e.g. around timing events."""
    cur = torch.cuda.current_stream(device)
    for s in streams:
        if begin:
            s.wait_stream(cur)
        else:
            cur.wait_stream(s)


class GraphedCall:
    """Generic capture: `fn(build(buffers))` over named static input buffers.  `spec` maps a name to (shape, dtype);
    names in `varlen` may be loaded with fewer rows than their capacity (prefix copy; the live length travels in another input,
    e.g. `agent_offsets[-1]`); `init` is loaded before the capture.  Used by bench.py for the single-agent / SECOND / camera
    workloads."""

    def __init__(self, fn, spec, build, device, varlen=(), init=None):
        self.bufs = {k: torch.zeros(tuple(shape), dtype=dt, device=device) for k, (shape, dt) in spec.items()}
        self.varlen = set(varlen)
        if init is not None:
            GraphedCall.load(self, **init)          # by name, whatever a subclass's `load` takes
        self.data = build(self.bufs)
        self.graph, self.out, self.kernels_per_replay = capture(lambda: fn(self.data), device)

    def load(self, **tensors):
        nbytes = 0
        for k, t in tensors.items():
            b = self.bufs[k]
            if k in self.varlen:
                if t.shape[0] > b.shape[0]:
                    raise ValueError(f"{k}: {t.shape[0]} rows, graph capacity is {b.shape[0]}")
                b[:t.shape[0]].copy_(t, non_blocking=True)
            else:
                b.copy_(t, non_blocking=True)
            nbytes += t.numel() * t.element_size()
        return nbytes

    def replay(self):
        self.graph.replay()
        return self.out


class FrameGraph(GraphedCall):
    """One frame of `n_agents` agents of one lidar modality: `model` over the static inputs `points` (up to `point_capacity`
    rows; the live count travels in `agent_offsets[-1]`), `agent_offsets` and `pairwise` (identities until the first load)."""

    def __init__(self, model, n_agents: int, point_capacity: int, pairwise_shape, modality: str = "m1", device=None):
        dev = device or next(model.parameters()).device
        spec = {"points": ((point_capacity, 4), torch.float32), "agent_offsets": ((n_agents + 1,), torch.int32),
                "pairwise": (tuple(pairwise_shape), torch.float64)}

        def build(b):
            return {f"inputs_{modality}": {"points": b["points"], "agent_offsets": b["agent_offsets"]},
                    "agent_modality_list": [modality] * n_agents, "record_len": [n_agents], "pairwise_t_matrix": b["pairwise"]}
        self.capacity = point_capacity
        super().__init__(model, spec, build, dev, varlen=("points",),
                         init={"pairwise": torch.eye(4, dtype=torch.float64, device=dev).expand(tuple(pairwise_shape))})

    def load(self, points: torch.Tensor, offsets: torch.Tensor, pairwise: torch.Tensor):
        """points (P,4) f32, offsets (A+1) i32, pairwise f64 — device or pinned-host tensors (async copies on the current stream).
        Returns the bytes copied."""
        if points.shape[0] > self.capacity:
            raise ValueError(f"scene has {points.shape[0]} points, graph capacity is {self.capacity}")
        return super().load(points=points, agent_offsets=offsets, pairwise=pairwise)

    def results(self):
        """The device tensors a frame's consumer reads: the heads."""
        return _heads(self.out)


class FrameInterleaver:
    """N captured frames, each on its own stream: consecutive frames overlap on the GPU (the small latency-bound kernels at the
    head of frame i+1 -- voxeliser, VFE, stem -- and the tails / prologues of its convolutions run in the gaps of frame i).  A
    throughput device for streams of independent frames; the latency of one frame is that of a single FrameGraph or worse.

        il = FrameInterleaver(model, n_agents, point_capacity, pairwise_shape, n=2)
        out = il.submit(points, offsets, pairwise)     # device tensors of frame i; `out` is complete after il.wait(slot)
    """

    def __init__(self, model, n_agents: int, point_capacity: int, pairwise_shape, n: int = 2, modality: str = "m1", device=None):
        dev = device or next(model.parameters()).device
        self._start([FrameGraph(model, n_agents, point_capacity, pairwise_shape, modality, device=dev) for _ in range(n)], dev)

    @staticmethod
    def for_scene(*args, **kwargs):
        """N captured SceneGraphs of a mixed-modality scene: SceneInterleaver(model, agent_modality_list, capacities,
        pairwise_shape, postprocess_params=None, n=2, device=None, **graph_kwargs)."""
        return SceneInterleaver(*args, **kwargs)

    def _start(self, graphs, dev):
        self.dev, self.n = dev, len(graphs)
        self.graphs = graphs
        self.streams = [torch.cuda.Stream(device=dev) for _ in range(self.n)]
        self.count = 0
        self.join(begin=True)

    @property
    def kernels_per_replay(self):
        return self.graphs[0].kernels_per_replay

    def submit(self, points, offsets, pairwise):
        return self._submit(points, offsets, pairwise)

    def _submit(self, *inputs):
        k = self.count % self.n
        with torch.cuda.stream(self.streams[k]):        # the previous use of slot k is earlier on the same stream
            self.graphs[k].load(*inputs)
            out = self.graphs[k].replay()
        self.count += 1
        return out

    def join(self, begin: bool):
        """Order the interleaver's streams after (begin) / before (end) the caller's current stream."""
        _join(self.dev, self.streams, begin)


class FramePipeline:
    """Two captured frames on four streams: while frame i computes, frame i+1's inputs are copied in (pinned host -> HBM), frame
    i-1's predictions are copied out (HBM -> pinned host), and -- each frame slot replays on its OWN compute stream -- the head of
    frame i+1 (voxeliser, VFE, stem: small latency-bound kernels) runs in the gaps of frame i's convolutions
    (`compute_streams=1` restores strict frame-after-frame execution).  The serving loop's
    public entry point:

        pipe = FramePipeline(model, n_agents, point_capacity, pairwise_shape)
        preds = pipe.submit(points_pinned, offsets_pinned, pairwise_pinned)   # dict of pinned host tensors of frame i - 1 (or None)
        last = pipe.flush()                                                      # waits for the frame in flight

    Each frame's result is complete on the host before its buffers are reused (events, no host sync inside submit).
    """

    def __init__(self, model, n_agents: int, point_capacity: int, pairwise_shape, modality: str = "m1", device=None,
                 compute_streams: int = 2, depth: int = 2):
        """`depth` = captured frames (slots) in flight: `submit` of frame i returns the predictions of frame i - (depth - 1).
        depth 2 keeps one frame queued behind the running one; deeper pipelines keep both compute streams fed while the host
        waits for a result (on C2 depths 2-4 measure the same within run-to-run noise, 290-305 frames/s end to end)."""
        dev = device or next(model.parameters()).device
        self._start([FrameGraph(model, n_agents, point_capacity, pairwise_shape, modality, device=dev)
                     for _ in range(max(2, int(depth)))], dev, compute_streams)

    @staticmethod
    def for_scene(*args, **kwargs):
        """The pipeline over a mixed-modality scene: ScenePipeline(model, agent_modality_list, capacities, pairwise_shape,
        postprocess_params=None, device=None, compute_streams=2, depth=2, **graph_kwargs), e.g. `eval_thresholds`."""
        return ScenePipeline(*args, **kwargs)

    def _start(self, graphs, dev, compute_streams, eval_thresholds=None):
        """Slot k replays `graphs[k]` and copies its `results()` (device tensors by name) back to the host after each replay; a
        None slot is bound by `_bind` when a frame gives it a graph.  With `eval_thresholds` the results carry each frame's
        evaluation (SceneGraph.results), which goes into `result_stat` as the frame is handed back."""
        self.dev, self.depth = dev, len(graphs)
        self.eval_thresholds = eval_thresholds
        self.result_stat = None if eval_thresholds is None else \
            {t: {'tp': [], 'fp': [], 'score': [], 'gt': 0} for t in eval_thresholds}
        self.evaluated = 0                                     # frames appended to result_stat (or refused by it) so far
        self.graphs = graphs
        self.s_in, self.s_out = (torch.cuda.Stream(device=dev) for _ in range(2))
        comp = [torch.cuda.Stream(device=dev) for _ in range(2 if compute_streams >= 2 else 1)]
        self.s_comp = comp                                     # consecutive frames alternate between the compute streams
        self.ev_in = [torch.cuda.Event() for _ in range(self.depth)]
        self.ev_comp = [torch.cuda.Event() for _ in range(self.depth)]
        self.ev_out = [torch.cuda.Event() for _ in range(self.depth)]
        self.dev_out, self.host_out = [None] * self.depth, [None] * self.depth
        self.count = 0
        self.h2d_bytes = 0
        self.d2h_bytes = 0
        for k, g in enumerate(graphs):
            if g is not None:
                self._bind(k, g.results())
        self.join(begin=True)

    def _bind(self, k, results):
        """Slot k copies `results` (device tensors by name) into its pinned host tensors after each replay."""
        self.dev_out[k] = results
        if self.host_out[k] is None:
            self.host_out[k] = {n: torch.empty(t.shape, dtype=t.dtype).pin_memory() for n, t in results.items()}
            self.d2h_bytes = sum(t.numel() * t.element_size() for t in self.host_out[k].values())

    def _slot(self, k, *inputs):
        """The graph slot k replays for this frame."""
        return self.graphs[k]

    def _result(self, k):
        """What `submit` / `drain` hand back for the frame that last used slot k."""
        return self.host_out[k]

    def _returned(self, c):
        """The result of frame c (complete on the host).  With evaluation, the first time frame c is handed back its flags go
        into `result_stat`, in frame order; a frame whose evaluation failed raises here and is not appended again."""
        r = self._result(c % self.depth)
        if self.result_stat is not None and c >= self.evaluated:
            from .utils.eval_utils import append_packed
            self.evaluated = c + 1
            append_packed(self.result_stat, self.eval_thresholds, r["eval"], int(r["count"][0]), r["scores"].shape[0],
                          int(r["gt_count"][0]))
        return r

    def submit(self, points: torch.Tensor, offsets: torch.Tensor, pairwise: torch.Tensor):
        return self._submit(points, offsets, pairwise)

    def _submit(self, *inputs):
        d = self.depth
        k = self.count % d
        g = self._slot(k, *inputs)
        with torch.cuda.stream(self.s_in):
            if self.count >= d:
                self.s_in.wait_event(self.ev_comp[k])          # frame count-depth has consumed these input buffers
            h2d = g.load(*inputs)
            self.ev_in[k].record(self.s_in)
        sc = self.s_comp[self.count % len(self.s_comp)]        # slot reuse is ordered through ev_comp -> ev_in, whatever the stream
        with torch.cuda.stream(sc):
            sc.wait_event(self.ev_in[k])
            if self.count >= d:
                sc.wait_event(self.ev_out[k])                  # its predictions have left the output buffers
            g.replay()
            self.ev_comp[k].record(sc)
        with torch.cuda.stream(self.s_out):
            self.s_out.wait_event(self.ev_comp[k])
            for name, h in self.host_out[k].items():
                h.copy_(self.dev_out[k][name], non_blocking=True)
            self.ev_out[k].record(self.s_out)
        frame = self.count - (d - 1)
        if frame >= 0:
            self.ev_out[frame % d].synchronize()               # frame count-(depth-1) is complete on the host
        self.h2d_bytes = h2d
        self.count += 1
        return self._returned(frame) if frame >= 0 else None

    def drain(self):
        """Predictions of the frames still in flight, oldest first (the results `submit` has not returned yet)."""
        out = []
        for c in range(max(self.count - (self.depth - 1), 0), self.count):
            self.ev_out[c % self.depth].synchronize()
            out.append(self._returned(c))
        return out

    def flush(self):
        """Wait for everything in flight; returns the LAST frame's predictions."""
        if self.count == 0:
            return None
        res = self.drain()
        return res[-1]

    def join(self, begin: bool):
        """Order the pipeline's streams after (begin) / before (end) the caller's current stream, e.g. around timing events."""
        _join(self.dev, (self.s_in, *self.s_comp, self.s_out), begin)


def _count(v):
    return isinstance(v, numbers.Integral) and not isinstance(v, bool) and v > 0


def scene_spec(sensor_type_dict, agent_modality_list, capacities):
    """The static input buffers of a captured scene, from `capacities` (see LateFusionGraph / SceneGraph), checked on the host:
    {m: {"agents": k, "lidar": point capacity} or {"agents": k, "camera": (cams, h, w), "raw": bool}} in order of first
    appearance.  Raises ValueError for a modality the model does not have or a capacity that is missing or malformed."""
    spec = {}
    for m in agent_modality_list:
        if m not in sensor_type_dict:
            raise ValueError(f"agent modality {m!r}: the model has {list(sensor_type_dict)}")
        if m in spec:
            spec[m]["agents"] += 1
            continue
        if m not in capacities:
            raise ValueError(f"{m}: no capacity given")
        cap = capacities[m]
        if sensor_type_dict[m] == "camera":
            ok = isinstance(cap, (tuple, list)) and len(cap) in (3, 4) and all(_count(v) for v in cap[:3]) \
                and (len(cap) == 3 or cap[3] is torch.uint8)
            if not ok:
                raise ValueError(f"{m}: camera capacity {cap}; (cams, h, w) takes normalised fp32 images and "
                                 "(cams, H0, W0, torch.uint8) raw frames")
            spec[m] = {"agents": 1, "camera": tuple(int(v) for v in cap[:3]), "raw": len(cap) == 4}
        else:
            if not _count(cap):
                raise ValueError(f"{m}: lidar capacity {cap!r}; the point capacity of all its agents is a positive int")
            spec[m] = {"agents": 1, "lidar": int(cap)}
    return spec


def _input_buffers(spec, dev):
    inputs = {}
    for m, sp in spec.items():
        k = sp["agents"]
        if "camera" in sp:
            cams, h, w = sp["camera"]
            imgs = torch.zeros((k, cams, h, w, 3), dtype=torch.uint8, device=dev) if sp["raw"] else \
                torch.zeros((k, cams, 3, h, w), dtype=torch.float32, device=dev)
            inputs[m] = {"imgs": imgs,
                         "rots": torch.eye(3, device=dev).repeat(k, cams, 1, 1),
                         "trans": torch.zeros((k, cams, 3), dtype=torch.float32, device=dev),
                         "intrins": torch.eye(3, device=dev).repeat(k, cams, 1, 1),
                         "post_rots": torch.eye(3, device=dev).repeat(k, cams, 1, 1),
                         "post_trans": torch.zeros((k, cams, 3), dtype=torch.float32, device=dev)}
        else:
            inputs[m] = {"points": torch.zeros((sp["lidar"], 4), dtype=torch.float32, device=dev),
                         "agent_offsets": torch.zeros((k + 1,), dtype=torch.int32, device=dev)}
    return inputs


def _input_views(spec, inputs):
    """The input buffers of `spec` as leading slices of caller-owned ones (`_input_buffers` of the same capacities for as many or
    more agents), so that the graphs of several agent lists can read one set.  Raises ValueError for a buffer that cannot hold
    the spec's."""
    views = {}
    for m, want in _input_buffers(spec, "meta").items():
        views[m] = {}
        for key, w in want.items():
            b = inputs.get(m, {}).get(key)
            if b is None or b.dtype != w.dtype or b.shape[1:] != w.shape[1:] or b.shape[0] < w.shape[0]:
                got = "missing" if b is None else f"{tuple(b.shape)} {b.dtype}"
                raise ValueError(f"inputs[{m!r}][{key!r}]: {got}, the scene needs {tuple(w.shape)} {w.dtype}")
            views[m][key] = b[:w.shape[0]]
    return views


def _voxel_limits(model, spec, voxel_limits):
    """{m: {max_points_per_voxel, max_voxels}} of every lidar modality of `spec`: the encoder's defaults unless `voxel_limits[m]`
    gives them."""
    out = {}
    for m, sp in spec.items():
        if "lidar" in sp:
            lim = dict(getattr(model, f"encoder_{m}").voxelize_args)
            lim.update((voxel_limits or {}).get(m, {}))
            out[m] = {k: int(lim[k]) for k in ("max_points_per_voxel", "max_voxels")}
    return out


def eval_setup(postprocess_params, eval_thresholds, gt_capacity):
    """(thresholds, GT capacity) of a captured frame that evaluates its boxes, or (None, None) when `eval_thresholds` is None.
    Checked on the host: evaluation needs `postprocess_params`; 1 to 8 thresholds, each > 0; the GT capacity is `gt_capacity`,
    by default `postprocess_params['max_num']` (100 in the shipped yamls), and lies in [1, 4096].  Raises ValueError."""
    if eval_thresholds is None:
        if gt_capacity is not None:
            raise ValueError("gt_capacity without eval_thresholds: the frame does not evaluate its boxes")
        return None, None
    if postprocess_params is None:
        raise ValueError("evaluation matches the post-processed boxes: eval_thresholds needs postprocess_params")
    thr = tuple(float(v) for v in eval_thresholds)
    if not 1 <= len(thr) <= 8 or not all(v > 0 for v in thr):
        raise ValueError(f"eval_thresholds {eval_thresholds}: 1 to 8 IoU thresholds, each > 0")
    if gt_capacity is None:
        if 'max_num' not in postprocess_params:
            raise ValueError("gt_capacity: postprocess_params has no 'max_num'; give the most GT boxes a frame may have")
        gt_capacity = postprocess_params['max_num']
    if not _count(gt_capacity) or gt_capacity > 4096:
        raise ValueError(f"gt_capacity {gt_capacity!r}: an int in [1, 4096]")
    return thr, int(gt_capacity)


def check_gt(gt_boxes, gt_capacity):
    """Host-side checks of a frame's GT against a captured frame's GT capacity (None: the frame does not evaluate): GT
    (G, 8, 3) fp32 corners, as the reference's post_processor.generate_gt_bbx returns them, with G <= capacity, required when the
    frame evaluates and refused when it does not.  Raises ValueError; returns the bytes the load copies."""
    if gt_capacity is None:
        if gt_boxes is not None:
            raise ValueError("gt_boxes given to a frame captured without eval_thresholds")
        return 0
    if gt_boxes is None:
        raise ValueError("the frame evaluates its boxes (eval_thresholds): gt_boxes (G, 8, 3) fp32 required")
    if not isinstance(gt_boxes, torch.Tensor) or gt_boxes.dim() != 3 or tuple(gt_boxes.shape[1:]) != (8, 3):
        raise ValueError(f"gt_boxes of shape {tuple(getattr(gt_boxes, 'shape', ()))}, (G, 8, 3) corners expected")
    if gt_boxes.dtype != torch.float32:
        raise ValueError(f"gt_boxes of dtype {gt_boxes.dtype}, float32 corners expected")
    if gt_boxes.shape[0] > gt_capacity:
        raise ValueError(f"the frame has {gt_boxes.shape[0]} GT boxes, the graph's gt_capacity is {gt_capacity}")
    return gt_boxes.shape[0] * 96 + 4


class FrameEval:
    """The evaluation of a captured frame: its static GT input (`gt` (capacity, 8, 3) fp32 corners, `gt_count` (1,) int32) and
    the ops.EvalBuffers heal_eval_tp_fp_counted writes, for up to `det_capacity` boxes (the decode capacity TOP).  Caller-owned
    so that several graphs can share one (SceneStream: one per pipeline slot, outside the graph pool)."""

    def __init__(self, det_capacity: int, gt_capacity: int, device):
        self.gt = torch.zeros((gt_capacity, 8, 3), dtype=torch.float32, device=device)
        self.gt_count = torch.zeros((1,), dtype=torch.int32, device=device)
        self.buffers = ops.EvalBuffers(det_capacity, gt_capacity, device)

    def run(self, post, thresholds):
        """Match the post-processed boxes (ops.PostprocessBuffers: boxes, scores, count on the device) to the GT; capture-safe."""
        return ops.eval_tp_fp_counted(post.boxes, post.scores, post.count, self.gt, self.gt_count, thresholds, self.buffers)

    def load(self, gt_boxes):
        """Copy a frame's GT (checked by check_gt) into the static buffers, asynchronously on the current stream."""
        n = gt_boxes.shape[0]
        if n:
            self.gt[:n].copy_(gt_boxes, non_blocking=True)
        self.gt_count.fill_(n)


class LateFusionGraph:
    """Late fusion of one scene as ONE captured graph: a single-agent model's `grouped_heads` (one batched forward per modality,
    every cav's heads in one (n_cav, H, W, S) buffer) and heal_box_decode_nms_late (decode with the transforms read on the device,
    sort, rotated NMS, range mask).  The reference runs one model call per cav, then the post-processor on the host.

        g = LateFusionGraph(model, ["m1", "m1", "m2"], {"m1": 200000, "m2": (4, 256, 704)}, hypes["postprocess"])
        g.load(batch_data)            # {cav_id: {inputs_<m>: ..., transformation_matrix: 4x4}} in the captured modality order
        out = g.replay()              # out.boxes[:out.count], out.scores[:out.count] on the device, no host sync

    With `eval_thresholds` (e.g. inference.py's (0.3, 0.5, 0.7)) the graph ends in heal_eval_tp_fp_counted, which matches the
    boxes to the GT given to `load(batch_data, gt_boxes)`: `g.eval.buffers.packed` holds the frame's status, sorted scores and
    flags at the decode capacity TOP (eval_utils.append_packed turns a host copy into `result_stat` entries).  Late fusion's GT
    is the union of every cav's objects, so `gt_capacity` (default `postprocess_params['max_num']`) may need to be larger than
    an intermediate-fusion frame's.
    `capacities[m]`: for a lidar modality the point capacity of ALL its cavs together (raw clouds, `points` + `agent_offsets`; the
    live counts travel in the offsets), for a camera modality (cameras, image height, image width) per cav for normalised fp32
    images, or (cameras, frame height, frame width, torch.uint8) for raw uint8 (H0, W0, 3) frames, which the encoder resizes, crops
    and normalises on the GPU.  The poses are inputs: replaying the graph for another scene uses that scene's transforms.

    Several graphs can share memory (LateFusionStream does so per pipeline slot), as SceneGraph's do: `inputs` are caller-owned
    input buffers (`_input_buffers` of these capacities for as many or more cavs; the graph reads leading slices), `transforms` a
    caller-owned (max_cav, 4, 4) fp32 device buffer of which the graph reads the leading (n, 4, 4), `postprocess_buffers`
    caller-owned ops.PostprocessBuffers for (H * n or more, W, A, TOP), `eval_buffers` a caller-owned FrameEval, and `pool` the
    private memory pool of the capture.  `voxel_limits[m]` overrides the encoder's {max_points_per_voxel, max_voxels} of a lidar
    modality.  `staging`: pinned host tensors (`late_staging`) through which `load` sends the per-cav point offsets and poses
    instead of pageable ones; the caller keeps them unwritten until the last load's copies are done."""

    CAMERA_KEYS = ("rots", "trans", "intrins", "post_rots", "post_trans")

    def __init__(self, model, modality_of_each_cav, capacities, postprocess_params, device=None, eval_thresholds=None,
                 gt_capacity=None, inputs=None, pool=None, postprocess_buffers=None, eval_buffers=None, transforms=None,
                 voxel_limits=None, staging=None):
        dev = device or next(model.parameters()).device
        self.eval_thresholds, self.gt_capacity = eval_setup(postprocess_params, eval_thresholds, gt_capacity)
        self.eval = None
        if self.eval_thresholds is not None:
            self.eval = FrameEval(TOP, self.gt_capacity, dev) if eval_buffers is None else eval_buffers
        self.modalities = list(modality_of_each_cav)
        n = len(self.modalities)
        self.groups = {}
        for i, m in enumerate(self.modalities):
            self.groups.setdefault(m, []).append(i)
        self.spec = scene_spec(model.sensor_type_dict, self.modalities, capacities)
        self.inputs = _input_buffers(self.spec, dev) if inputs is None else _input_views(self.spec, inputs)
        self.voxel_limits = _voxel_limits(model, self.spec, voxel_limits)
        for m, lim in self.voxel_limits.items():
            self.inputs[m].update(lim)
        if transforms is None:
            self.transforms = torch.eye(4, dtype=torch.float32, device=dev).repeat(n, 1, 1).contiguous()
        elif not isinstance(transforms, torch.Tensor) or transforms.dtype != torch.float32 or transforms.dim() != 3 \
                or tuple(transforms.shape[1:]) != (4, 4) or transforms.shape[0] < n or not transforms.is_contiguous():
            raise ValueError(f"transforms: a contiguous (max_cav >= {n}, 4, 4) fp32 buffer expected, got "
                             f"{tuple(getattr(transforms, 'shape', ()))} {getattr(transforms, 'dtype', None)}")
        else:
            self.transforms = transforms[:n]
        self.staging = staging
        self.anchors = _anchors(postprocess_params, dev)
        A = self.anchors.shape[2]
        self.buffers = ops.PostprocessBuffers(self.anchors.shape[0] * n, self.anchors.shape[1], A, TOP, dev) \
            if postprocess_buffers is None else postprocess_buffers
        decode = decode_kwargs(postprocess_params, True)       # the grouped heads always carry the dir channels

        def run():
            y, _ = model.grouped_heads(self.groups, self.inputs, n)
            post = ops.box_decode_nms_late(y, y, y, self.anchors, self.transforms, **decode, buffers=self.buffers,
                                           coffsets=(0, A, 8 * A))
            if self.eval is not None:
                self.eval.run(post, self.eval_thresholds)
            return post

        self.graph, self.out, self.kernels_per_replay = capture(run, dev, pool)

    def load(self, batch_data, gt_boxes=None):
        """Copy a scene's inputs and cav -> ego transforms into the captured buffers (asynchronous copies on the current stream).
        The cavs must come in the captured modality order; each lidar cav carries one raw cloud (`points`, `agent_offsets`).
        `gt_boxes`: the scene's GT corners (G, 8, 3) fp32, required with evaluation and refused without (check_gt)."""
        from .models.heter_model_late import modality_of
        cavs = list(batch_data.keys())
        mods = [modality_of(batch_data[c]) for c in cavs]
        if mods != self.modalities:
            raise ValueError(f"scene modalities {mods}, the graph was captured for {self.modalities}")
        check_gt(gt_boxes, self.gt_capacity)
        for m, idx in self.groups.items():
            buf = self.inputs[m]
            if "points" in buf:
                offs, total = [0], 0
                for j, i in enumerate(idx):
                    pts = batch_data[cavs[i]][f"inputs_{m}"]["points"]
                    if total + pts.shape[0] > buf["points"].shape[0]:
                        raise ValueError(f"{m}: the scene has more points than the graph's capacity {buf['points'].shape[0]}")
                    buf["points"][total:total + pts.shape[0]].copy_(pts, non_blocking=True)
                    total += pts.shape[0]
                    offs.append(total)
                if self.staging is None:
                    buf["agent_offsets"].copy_(torch.tensor(offs, dtype=torch.int32), non_blocking=True)
                else:
                    host = self.staging["offsets"][m][:len(offs)]
                    host.copy_(torch.tensor(offs, dtype=torch.int32))
                    buf["agent_offsets"].copy_(host, non_blocking=True)
            else:
                for j, i in enumerate(idx):
                    src = batch_data[cavs[i]][f"inputs_{m}"]
                    for k in ("imgs",) + self.CAMERA_KEYS:
                        raw = k == "imgs" and buf[k].dtype == torch.uint8         # raw frames (cams, H0, W0, 3) go in whole
                        buf[k][j].copy_(src[k][0][:, :3] if k == "imgs" and not raw else src[k][0], non_blocking=True)
        mats = [torch.as_tensor(batch_data[c]['transformation_matrix']) for c in cavs]
        if self.staging is None:
            T = torch.stack([t.reshape(4, 4).to(torch.float32) for t in mats])
            self.transforms.copy_(T, non_blocking=True)
        else:
            host = self.staging["transforms"][:len(cavs)]
            for i, t in enumerate(mats):
                if not t.is_cuda:
                    host[i].copy_(t.reshape(4, 4))
            self.transforms.copy_(host, non_blocking=True)
            for i, t in enumerate(mats):                  # poses already on the device are copied there, after the staged ones
                if t.is_cuda:
                    self.transforms[i].copy_(t.reshape(4, 4), non_blocking=True)
        if self.eval is not None:
            self.eval.load(gt_boxes)

    def replay(self):
        self.graph.replay()
        return self.out

    def results(self):
        """The device tensors a frame's consumer reads, named as SceneGraph.results(): the boxes, scores and box count, with
        evaluation also `eval` (EvalBuffers.packed at capacity TOP) and `gt_count`."""
        out = {"boxes": self.buffers.boxes, "scores": self.buffers.scores, "count": self.buffers.count}
        if self.eval is not None:
            out.update(eval=self.eval.buffers.packed, gt_count=self.eval.gt_count)
        return out


def late_staging(capacities, sensor_type_dict, max_cav: int):
    """Pinned host tensors through which LateFusionGraph.load sends a frame's per-cav point offsets ({m: (max_cav + 1,) int32} for
    every lidar modality of `capacities`) and cav -> ego poses ((max_cav, 4, 4) fp32)."""
    offsets = {m: torch.zeros((max_cav + 1,), dtype=torch.int32).pin_memory()
               for m in capacities if sensor_type_dict.get(m) != "camera"}
    return {"offsets": offsets, "transforms": torch.eye(4).repeat(max_cav, 1, 1).pin_memory()}


def late_modalities(batch_data):
    """The ordered modality of every cav of a late batch `{cav_id: cav_content}` (modality_of: its one `inputs_*` key)."""
    from .models.heter_model_late import modality_of
    return [modality_of(cav) for cav in batch_data.values()]


def check_late_scene(sensor_type_dict, capacities, max_cav: int, voxel_limits, batch_data, gt_boxes=None, gt_capacity=None):
    """Host-side checks of a late-fusion batch `{cav_id: cav_content}` (dataset order, ego first) against the captured graphs of
    a LateFusionStream, before anything is copied and without reading the device: 1 to `max_cav` cavs, each of a modality the
    model has (`sensor_type_dict`) and `capacities` gives; a lidar cav carries one raw cloud (`points` (P, 4) and `agent_offsets`
    of length 2), not left for GPU filtering (`filter_points`), with the voxelisation limits `voxel_limits[m]` the graphs were
    captured with when it names them, and the clouds of one modality fit its point capacity together; a camera cav's images
    have the captured shape and kind (uint8 frames or fp32 images); every cav has a `transformation_matrix`; the GT passes
    check_gt.  Raises ValueError; returns the bytes LateFusionGraph.load copies."""
    mods = late_modalities(batch_data)
    if not 0 < len(mods) <= max_cav:
        raise ValueError(f"{len(mods)} cavs {mods}: the stream serves 1 to max_cav = {max_cav}")
    spec = scene_spec(sensor_type_dict, mods, capacities)
    nbytes = check_gt(gt_boxes, gt_capacity) + len(mods) * 64
    points = dict.fromkeys(spec, 0)
    for cav, m in zip(batch_data, mods):
        content, sp = batch_data[cav], spec[m]
        src = content[f"inputs_{m}"]
        if "transformation_matrix" not in content:
            raise ValueError(f"cav {cav!r}: no transformation_matrix")
        if torch.as_tensor(content["transformation_matrix"]).numel() != 16:
            raise ValueError(f"cav {cav!r}: transformation_matrix of {torch.as_tensor(content['transformation_matrix']).numel()} "
                             "values, a 4 x 4 matrix expected")
        if "lidar" in sp:
            if "points" not in src or "agent_offsets" not in src:
                raise ValueError(f"cav {cav!r} inputs_{m}: a raw cloud (points, agent_offsets) expected, not voxels")
            if tuple(src["agent_offsets"].shape) != (2,):
                raise ValueError(f"cav {cav!r} inputs_{m}: agent_offsets of shape {tuple(src['agent_offsets'].shape)}, a late-"
                                 "fusion cav carries one cloud (2,)")
            if src.get("filter_points"):
                raise ValueError(f"cav {cav!r} inputs_{m}: clouds left for heal_mask_points (filter_on_gpu) are not served by a "
                                 "captured frame; filter them in the dataset")
            for key, v in voxel_limits[m].items():
                if key in src and int(src[key]) != v:
                    raise ValueError(f"cav {cav!r} inputs_{m}: {key} {int(src[key])}, the graph was captured with {v}")
            pts = src["points"]
            if pts.dim() != 2 or pts.shape[1] != 4:
                raise ValueError(f"cav {cav!r} inputs_{m}: points of shape {tuple(pts.shape)}, (P, 4) expected")
            points[m] += pts.shape[0]
            if points[m] > sp["lidar"]:
                raise ValueError(f"{m}: the scene's {sp['agents']} cavs have more points than the capacity {sp['lidar']}")
            nbytes += pts.shape[0] * 16
        else:
            imgs = src["imgs"]
            cams, h, w = sp["camera"]
            if sp["raw"] != (imgs.dtype == torch.uint8):
                raise ValueError(f"cav {cav!r} inputs_{m}: {'fp32 images' if sp['raw'] else 'raw uint8 frames'} for a graph "
                                 f"captured with {'raw uint8 frames' if sp['raw'] else 'normalised fp32 images'}")
            want = (1, cams, h, w, 3) if sp["raw"] else (1, cams, 3, h, w)
            got = tuple(imgs.shape) if sp["raw"] else tuple(imgs.shape[:2]) + (3,) + tuple(imgs.shape[3:])
            if imgs.dim() != 5 or got != want or (not sp["raw"] and imgs.shape[2] < 3):
                raise ValueError(f"cav {cav!r} inputs_{m}: images of shape {tuple(imgs.shape)}, the graph was captured for {want}")
            nbytes += cams * h * w * 3 * (1 if sp["raw"] else 4)
            for key in LateFusionGraph.CAMERA_KEYS:
                shape = (1, cams, 3, 3) if key in ("rots", "intrins", "post_rots") else (1, cams, 3)
                v = src.get(key)
                if v is None or tuple(v.shape) != shape:
                    got = "missing" if v is None else f"of shape {tuple(v.shape)}"
                    raise ValueError(f"cav {cav!r} inputs_{m}: {key} {got}, {shape} expected")
                nbytes += v.numel() * 4
    return nbytes + sum(4 * (sp["agents"] + 1) for sp in spec.values() if "lidar" in sp)


def check_scene(spec, agent_modality_list, voxel_limits, ego_batch, gt_boxes=None, gt_capacity=None):
    """Host-side checks of a collated `batch_data['ego']` against a captured scene (no device read): the agent modalities, every
    input's shape against its buffer, the lidar voxelisation limits the graph was captured with, uint8 frames against fp32
    images, and the frame's GT against the graph's `gt_capacity` (check_gt; None: the graph does not evaluate).  Raises
    ValueError; returns the bytes `SceneGraph.load` copies."""
    aml = list(ego_batch["agent_modality_list"])
    if aml != list(agent_modality_list):
        raise ValueError(f"scene modalities {aml}, the graph was captured for {list(agent_modality_list)}")
    nbytes = ego_batch["pairwise_t_matrix"].numel() * 8 + check_gt(gt_boxes, gt_capacity)
    for m, sp in spec.items():
        src = ego_batch[f"inputs_{m}"]
        k = sp["agents"]
        if "lidar" in sp:
            if "points" not in src:
                raise ValueError(f"inputs_{m}: raw clouds (points, agent_offsets) expected, not voxels")
            if src.get("filter_points"):
                raise ValueError(f"inputs_{m}: clouds left for heal_mask_points (filter_on_gpu) are not served by a captured "
                                 "scene; filter them in the dataset")
            for key, v in voxel_limits[m].items():
                if key in src and int(src[key]) != v:
                    raise ValueError(f"inputs_{m}: {key} {int(src[key])}, the graph was captured with {v}")
            pts, offs = src["points"], src["agent_offsets"]
            if pts.dim() != 2 or pts.shape[1] != 4:
                raise ValueError(f"inputs_{m}: points of shape {tuple(pts.shape)}, (P, 4) expected")
            if pts.shape[0] > sp["lidar"]:
                raise ValueError(f"inputs_{m}: the scene has {pts.shape[0]} points, the graph's capacity is {sp['lidar']}")
            if tuple(offs.shape) != (k + 1,):
                raise ValueError(f"inputs_{m}: agent_offsets of shape {tuple(offs.shape)} for {k} agents")
            nbytes += pts.numel() * 4 + offs.numel() * 4
        else:
            imgs = src["imgs"]
            cams, h, w = sp["camera"]
            if sp["raw"] != (imgs.dtype == torch.uint8):
                raise ValueError(f"inputs_{m}: {'fp32 images' if sp['raw'] else 'raw uint8 frames'} for a graph captured with "
                                 f"{'raw uint8 frames' if sp['raw'] else 'normalised fp32 images'}")
            want = (k, cams, h, w, 3) if sp["raw"] else (k, cams, 3, h, w)
            got = tuple(imgs.shape) if sp["raw"] else tuple(imgs.shape[:2]) + (3,) + tuple(imgs.shape[3:])
            if got != want or (not sp["raw"] and imgs.shape[2] < 3):
                raise ValueError(f"inputs_{m}: images of shape {tuple(imgs.shape)}, the graph was captured for {want}")
            nbytes += k * cams * h * w * 3 * (1 if sp["raw"] else 4)
            for key in LateFusionGraph.CAMERA_KEYS:
                nbytes += src[key].numel() * 4
    return nbytes


class SceneGraph:
    """One intermediate-fusion frame of a mixed-modality scene as ONE captured graph: every modality's encoder on its agents,
    the agent assembly (heal_agent_stack), fusion and heads, and - with `postprocess_params` - heal_box_decode_nms for the ego.
    Works for HeterPyramidCollab, HeterModelBaseline and HeterModelBaselineMs.

        g = SceneGraph(model, ["m1", "m2", "m3", "m4", "m1"], {"m1": 240000, "m2": (4, 256, 704), "m3": 120000,
                       "m4": (4, 600, 800, torch.uint8)}, pairwise_shape=(1, 5, 5, 4, 4), postprocess_params=hypes["postprocess"])
        g.load(batch_data["ego"])      # the reference's collated ego batch (GpuVoxelPreprocessor raw clouds)
        out = g.replay()               # the model's output dict; out["postprocess"].boxes[:count] etc. on the device, no host sync

    `capacities[m]` follows LateFusionGraph: for a lidar modality the point capacity of ALL its agents together (the live counts
    travel in `agent_offsets`), for a camera modality (cameras, image height, image width) for normalised fp32 images or
    (cameras, frame height, frame width, torch.uint8) for raw frames, which the encoder resizes, crops and normalises on the
    GPU.  The voxelisation limits of a lidar modality are the encoder's defaults unless `voxel_limits[m]` gives
    {max_points_per_voxel, max_voxels}; a batch that carries other values is refused.  The ego's boxes are decoded in the ego
    frame (intermediate fusion: the identity transform).

    Several graphs can share memory (SceneStream does so per pipeline slot): `inputs` are caller-owned input buffers, as
    `_input_buffers` makes them for these capacities and as many or more agents (the graph reads leading slices);
    `postprocess_buffers` are caller-owned ops.PostprocessBuffers for the box decode; `eval_buffers` a caller-owned FrameEval;
    `pool` is the private memory pool the frame is captured into (torch.cuda.graph_pool_handle()).  The warm-up frames run outside
    the pool, so weight caches built lazily land in the ordinary allocator.

    Evaluation: with `eval_thresholds` (inference.py's are (0.3, 0.5, 0.7)) the graph ends in heal_box_decode_nms ->
    heal_eval_tp_fp_counted, which matches the ego's boxes to the frame's GT on the device (the box count never leaves it).  The
    GT comes in with `load(ego_batch, gt_boxes)`: (G, 8, 3) fp32 corners, what the reference's
    `post_processor.generate_gt_bbx(batch_data)` returns on the host, copied into a static (gt_capacity, 8, 3) buffer and a
    device count.  `gt_capacity` defaults to `postprocess_params['max_num']` and must be given when that key is absent.
    `results()` then adds the packed evaluation (ops.EvalBuffers: status, sorted scores, flags at the decode capacity TOP)
    and G."""

    def __init__(self, model, agent_modality_list, capacities, pairwise_shape, postprocess_params=None, device=None,
                 voxel_limits=None, inputs=None, pool=None, postprocess_buffers=None, eval_thresholds=None, gt_capacity=None,
                 eval_buffers=None):
        dev = device or next(model.parameters()).device
        self.eval_thresholds, self.gt_capacity = eval_setup(postprocess_params, eval_thresholds, gt_capacity)
        self.modalities = list(agent_modality_list)
        n = len(self.modalities)
        self.spec = scene_spec(model.sensor_type_dict, self.modalities, capacities)
        self.inputs = _input_buffers(self.spec, dev) if inputs is None else _input_views(self.spec, inputs)
        self.voxel_limits = _voxel_limits(model, self.spec, voxel_limits)
        for m, lim in self.voxel_limits.items():
            self.inputs[m].update(lim)
        self.pairwise = torch.eye(4, dtype=torch.float64, device=dev).expand(tuple(pairwise_shape)).contiguous()
        self.data = {**{f"inputs_{m}": buf for m, buf in self.inputs.items()}, "agent_modality_list": list(self.modalities),
                     "record_len": [n], "pairwise_t_matrix": self.pairwise}
        self.postprocess = None
        if postprocess_params is not None:
            self.anchors = _anchors(postprocess_params, dev)
            H, W, A = self.anchors.shape[:3]
            self.postprocess = ops.PostprocessBuffers(H, W, A, TOP, dev) if postprocess_buffers is None else postprocess_buffers
        self.eval = None
        if self.eval_thresholds is not None:
            self.eval = FrameEval(TOP, self.gt_capacity, dev) if eval_buffers is None else eval_buffers
        pparams, eye = postprocess_params, torch.eye(4, dtype=torch.float64)

        def run():
            out = model(self.data)
            if pparams is not None:                     # VoxelPostprocessor._decode_one for the ego
                dirp = out.get('dir_preds')
                out['postprocess'] = ops.box_decode_nms(out['cls_preds'], out['reg_preds'], dirp, self.anchors, eye,
                                                        **decode_kwargs(pparams, dirp is not None), buffers=self.postprocess)
                if self.eval is not None:
                    self.eval.run(out['postprocess'], self.eval_thresholds)
            return out

        self.graph, self.out, self.kernels_per_replay = capture(run, dev, pool)

    def load(self, ego_batch, gt_boxes=None):
        """Copy a scene's inputs and pairwise transforms (and with evaluation its GT corners) into the captured buffers
        (asynchronous copies on the current stream, device or pinned-host sources).  Checks the batch on the host first
        (check_scene); returns the bytes copied."""
        nbytes = check_scene(self.spec, self.modalities, self.voxel_limits, ego_batch, gt_boxes, self.gt_capacity)
        for m, buf in self.inputs.items():
            src = ego_batch[f"inputs_{m}"]
            if "points" in buf:
                pts = src["points"]
                buf["points"][:pts.shape[0]].copy_(pts, non_blocking=True)
                buf["agent_offsets"].copy_(src["agent_offsets"], non_blocking=True)
            else:
                imgs = src["imgs"]
                buf["imgs"].copy_(imgs if imgs.dtype == torch.uint8 else imgs[:, :, :3], non_blocking=True)
                for k in LateFusionGraph.CAMERA_KEYS:
                    buf[k].copy_(src[k], non_blocking=True)
        self.pairwise.copy_(ego_batch["pairwise_t_matrix"], non_blocking=True)
        if self.eval is not None:
            self.eval.load(gt_boxes)
        return nbytes

    def replay(self):
        self.graph.replay()
        return self.out

    def results(self):
        """The device tensors a frame's consumer reads: the ego's boxes, scores and box count with `postprocess_params`, else
        the heads; with evaluation also `eval` (EvalBuffers.packed at capacity TOP) and `gt_count`."""
        if self.postprocess is not None:
            out = {"boxes": self.postprocess.boxes, "scores": self.postprocess.scores, "count": self.postprocess.count}
            if self.eval is not None:
                out.update(eval=self.eval.buffers.packed, gt_count=self.eval.gt_count)
            return out
        return _heads(self.out)


class SceneInterleaver(FrameInterleaver):
    """N captured SceneGraphs of a mixed-modality scene on N streams (FrameInterleaver.for_scene): `submit(ego_batch)`
    (`submit(ego_batch, gt_boxes)` with `eval_thresholds`) loads and replays one."""

    def __init__(self, model, agent_modality_list, capacities, pairwise_shape, postprocess_params=None, n: int = 2,
                 device=None, **graph_kwargs):
        dev = device or next(model.parameters()).device
        self._start([SceneGraph(model, agent_modality_list, capacities, pairwise_shape, postprocess_params, device=dev,
                                **graph_kwargs) for _ in range(n)], dev)

    def submit(self, ego_batch, gt_boxes=None):
        return self._submit(ego_batch, gt_boxes)


class ScenePipeline(FramePipeline):
    """The pipeline over a mixed-modality scene, SceneGraph slots (FramePipeline.for_scene): `submit(ego_batch)` takes the
    reference's collated `batch_data['ego']` and returns, pinned on the host, the boxes, scores and box count of frame
    i - (depth - 1) when `postprocess_params` is given (`boxes[:count[0]]`), else its heads.  With `eval_thresholds` (and
    `gt_capacity`, see SceneGraph) `submit(ego_batch, gt_boxes)` also takes the frame's GT, each frame is evaluated in its
    graph, and `pipe.result_stat` collects the frames in the reference's format as they come back."""

    def __init__(self, model, agent_modality_list, capacities, pairwise_shape, postprocess_params=None, device=None,
                 compute_streams: int = 2, depth: int = 2, **graph_kwargs):
        dev = device or next(model.parameters()).device
        graphs = [SceneGraph(model, agent_modality_list, capacities, pairwise_shape, postprocess_params, device=dev,
                             **graph_kwargs) for _ in range(max(2, int(depth)))]
        self._start(graphs, dev, compute_streams, graphs[0].eval_thresholds)

    def submit(self, ego_batch, gt_boxes=None):
        return self._submit(ego_batch, gt_boxes)


class SceneGraphCache:
    """The host side of SceneStream and LateFusionStream: a frame's key and its refusals, and per pipeline slot the captured
    graphs by key, least recently used first.  The key is an ordered modality list as a tuple: SceneStream's is the
    `agent_modality_list` (the ego first; the order is the fusion order), LateFusionStream's every cav's modality in batch order
    (the order decides NMS ties), which its `frame(batch, gt_boxes)` returns after check_late_scene.  `capture(slot, key)`
    makes slot `slot`'s graph for `key`."""

    def __init__(self, sensor_type_dict, capacities, max_cav: int, voxel_limits, slots: int, max_graphs: int, capture,
                 gt_capacity=None, frame=None):
        if int(max_graphs) < 1:
            raise ValueError(f"max_graphs {max_graphs}: a slot keeps at least one graph")
        self.sensors, self.capacities = dict(sensor_type_dict), dict(capacities)
        self.max_cav, self.voxel_limits, self.max_graphs = int(max_cav), voxel_limits, int(max_graphs)
        self.slots = [collections.OrderedDict() for _ in range(slots)]
        self.capture = capture
        self.gt_capacity = gt_capacity                          # None: the graphs do not evaluate
        self.frame = self._scene_frame if frame is None else frame
        self.captures = 0

    def _spec(self, key):
        if not 0 < len(key) <= self.max_cav:
            raise ValueError(f"{len(key)} agents {list(key)}: the stream serves 1 to max_cav = {self.max_cav}")
        return scene_spec(self.sensors, key, self.capacities)

    def key(self, agent_modality_list):
        """The key of an agent list.  Raises ValueError for an empty list, more agents than `max_cav`, a modality the model
        does not have or one without a capacity."""
        key = tuple(agent_modality_list)
        self._spec(key)
        return key

    def check(self, batch, gt_boxes=None):
        """The key of a frame after its host checks (nothing is copied): `frame(batch, gt_boxes)` when the cache was made with
        one (LateFusionStream), else those of a collated `batch_data['ego']`: the checks of `key` and of `check_scene` for the
        frame's own list and GT."""
        return self.frame(batch, gt_boxes)

    def _scene_frame(self, ego_batch, gt_boxes):
        key = tuple(ego_batch["agent_modality_list"])
        check_scene(self._spec(key), key, self.voxel_limits, ego_batch, gt_boxes, self.gt_capacity)
        return key

    def graph(self, slot: int, key):
        """Slot `slot`'s graph for `key`, captured on a miss.  Above `max_graphs` the least recently used graph of the slot is
        dropped, after the new one is captured, so the slot's memory pool always has a graph that holds it."""
        graphs = self.slots[slot]
        if key in graphs:
            graphs.move_to_end(key)
            return graphs[key]
        g = graphs[key] = self.capture(slot, key)
        self.captures += 1
        while len(graphs) > self.max_graphs:
            graphs.popitem(last=False)
        return g

    @property
    def graphs_captured(self):
        """Graphs held over all slots."""
        return sum(len(s) for s in self.slots)


class SceneStream(FramePipeline):
    """A stream of mixed-modality scenes whose agent list changes from frame to frame (the CAVs in range and their modalities,
    as in a dataset's test split), served through FramePipeline's slots: copy-in stream, compute stream, copy-out stream, events
    and no host sync.  `submit(ego_batch)` returns, pinned on the host, frame i - (depth - 1): the ego's boxes, scores and box
    count with `postprocess_params` (`boxes[:count[0]]`), else its heads, and the frame's `agent_modality_list`.

        stream = SceneStream(model, {"m1": 240_000, "m2": (4, 600, 800, torch.uint8), "m3": 120_000, "m4": (4, 600, 800,
                             torch.uint8)}, pairwise_shape=(1, 5, 5, 4, 4), postprocess_params=hypes["postprocess"])
        for batch_data in data_loader:
            res = stream.submit(batch_data["ego"])      # None while the pipeline fills
        rest = stream.drain()

    With `eval_thresholds` (and `gt_capacity`, see SceneGraph) every graph ends in the evaluation of its boxes:
    `submit(ego_batch, gt_boxes)` takes the frame's GT from the reference's `post_processor.generate_gt_bbx(batch_data)`, and
    `stream.result_stat` ({thr: {'tp', 'fp', 'score', 'gt'}}, the reference's format) gains each frame once, in frame order, when
    `submit` / `drain` / `flush` hands it back.  A frame with no box adds its GT count only.  A frame with a union of area 0
    raises ZeroDivisionError from that call, as the reference does, and is not appended.  The reference's
    `eval_utils.eval_final_results(stream.result_stat, ...)` then gives the AP.

    `capacities` follows SceneGraph for every modality the stream may see; `pairwise_shape[1]` is max_cav.  Each slot keeps one
    captured SceneGraph per agent list, so a 2-agent frame runs a 2-agent graph and its result is bit for bit that of a
    SceneGraph captured for its list alone.  A list new to a slot is captured inside `submit` (a device synchronise and two eager
    warm-up frames); `capture(agent_modality_list)` does it ahead.  Above `max_graphs` graphs in a slot the least recently used
    one is dropped (and recaptured if its list comes back).  A frame that cannot be served raises ValueError on the host before
    anything is copied: a modality the model does not have or without a capacity, more agents than max_cav, or any refusal of
    `check_scene` for its own list.

    Memory: the graphs of slot k are captured into one private pool, read slot k's one set of input buffers (every modality at
    its capacity, for max_cav agents) and write slot k's one set of post-processing (and evaluation) buffers, which lie outside
    the pool.  Graphs
    of one slot never run at once (slot k's next frame waits for its last one's replay and copy-out), so they share their
    scratch.  A graph's static outputs may lie in another graph's scratch: a frame's device results are valid only until its
    slot's next replay.  The copy-out to the host happens before that; the host results are valid until the slot's next
    copy-out, `depth` submits later, as in FramePipeline."""

    def __init__(self, model, capacities, pairwise_shape, postprocess_params=None, depth: int = 2, max_graphs: int = 16,
                 voxel_limits=None, device=None, eval_thresholds=None, gt_capacity=None):
        dev = device or next(model.parameters()).device
        depth = max(1, int(depth))
        self.model, self.capacities, self.pairwise_shape = model, dict(capacities), tuple(pairwise_shape)
        self.postprocess_params, self.voxel_limits = postprocess_params, voxel_limits
        thresholds, self.gt_capacity = eval_setup(postprocess_params, eval_thresholds, gt_capacity)
        spec = scene_spec(model.sensor_type_dict, list(self.capacities), self.capacities)
        max_cav = int(self.pairwise_shape[1])
        self.cache = SceneGraphCache(model.sensor_type_dict, self.capacities, max_cav, _voxel_limits(model, spec, voxel_limits),
                                     depth, max_graphs, self._capture, self.gt_capacity)
        self.inputs = [_input_buffers({m: dict(sp, agents=max_cav) for m, sp in spec.items()}, dev) for _ in range(depth)]
        self.pools = [torch.cuda.graph_pool_handle() for _ in range(depth)]
        self.postprocess = [None] * depth
        if postprocess_params is not None:
            H, W, A = _anchors(postprocess_params, "meta").shape[:3]
            self.postprocess = [ops.PostprocessBuffers(H, W, A, TOP, dev) for _ in range(depth)]
        self.evals = [None] * depth
        if thresholds is not None:
            self.evals = [FrameEval(TOP, self.gt_capacity, dev) for _ in range(depth)]
        self.lists = [None] * depth                             # the agent list of the frame that last used each slot
        self._start([None] * depth, dev, 2, thresholds)         # a slot's graphs are captured as frames need them

    def _capture(self, k, key):
        self.join(begin=False)          # the warm-up follows every frame in flight: slot k's last frame has left its buffers
        return SceneGraph(self.model, list(key), self.capacities, self.pairwise_shape, self.postprocess_params, device=self.dev,
                          voxel_limits=self.voxel_limits, inputs=self.inputs[k], pool=self.pools[k],
                          postprocess_buffers=self.postprocess[k], eval_thresholds=self.eval_thresholds,
                          gt_capacity=self.gt_capacity, eval_buffers=self.evals[k])

    def _slot(self, k, ego_batch, gt_boxes=None):
        key = self.cache.check(ego_batch, gt_boxes)
        g = self.cache.graph(k, key)
        self.lists[k] = key
        self._bind(k, g.results())
        return g

    def _result(self, k):
        return {**self.host_out[k], "agent_modality_list": list(self.lists[k])}

    def submit(self, ego_batch, gt_boxes=None):
        return self._submit(ego_batch, gt_boxes)

    def capture(self, agent_modality_list):
        """Capture the graphs of an agent list in every slot ahead of the stream (a list a slot already holds is kept)."""
        key = self.cache.key(agent_modality_list)
        for k in range(self.depth):
            self.cache.graph(k, key)

    @property
    def captures(self):
        """Graph captures so far, recaptures after eviction included."""
        return self.cache.captures

    @property
    def graphs_captured(self):
        """Graphs the stream holds over all slots."""
        return self.cache.graphs_captured


def late_cache(sensor_type_dict, capacities, max_cav: int, voxel_limits, slots: int, max_graphs: int, capture, gt_capacity=None):
    """LateFusionStream's SceneGraphCache: a frame is a late batch `{cav_id: cav_content}`, checked by check_late_scene and keyed
    by its ordered cav modalities."""
    def frame(batch_data, gt_boxes):
        check_late_scene(sensor_type_dict, capacities, max_cav, voxel_limits, batch_data, gt_boxes, gt_capacity)
        return tuple(late_modalities(batch_data))
    return SceneGraphCache(sensor_type_dict, capacities, max_cav, voxel_limits, slots, max_graphs, capture, gt_capacity,
                           frame=frame)


class LateFusionStream(FramePipeline):
    """A stream of late-fusion scenes whose cav list changes from frame to frame (the CAVs in range and their modalities, as
    in a dataset's test split), for the single-agent models (HeterModelLate, HeterPyramidSingle), served through FramePipeline's
    slots as SceneStream serves intermediate fusion.  `submit(batch_data)` takes what the late datasets collate
    (`{cav_id: cav_content}` in dataset order, ego first, what the reference's `inference_late_fusion` loops over) and returns,
    pinned on the host, frame i - (depth - 1): its boxes, scores and box count (`boxes[:count[0]]`) and its `modality_list`.

        stream = LateFusionStream(model, {"m1": 400_000, "m2": (4, 600, 800, torch.uint8)}, max_cav=5,
                                  postprocess_params=hypes["postprocess"], eval_thresholds=(0.3, 0.5, 0.7), gt_capacity=400)
        for batch_data in data_loader:
            gt = dataset.post_processor.generate_gt_bbx(batch_data)
            res = stream.submit(batch_data, gt)                    # late; None while the pipeline fills
            # no fusion: stream.submit({'ego': batch_data['ego']}, gt)
            # single:    stream.submit({'ego': batch_data['ego']}, dataset.post_processor.generate_gt_bbx({'ego': batch_data['ego']}))
        stream.drain()
        eval_utils.eval_final_results(stream.result_stat, save_path, infer_info)

    Each slot keeps one captured LateFusionGraph per ordered cav-modality list, so a frame's boxes are bit for bit those of a
    LateFusionGraph captured for its list alone.  A list new to a slot is captured inside `submit` (a device synchronise and two
    eager warm-up frames); `capture(modality_list)` does it ahead.  Above `max_graphs` graphs in a slot the least recently used
    one is dropped (and recaptured if its list comes back).  A frame that cannot be served raises ValueError on the host before
    anything is copied (check_late_scene).  `capacities` follows LateFusionGraph for every modality the stream may see; a lidar
    capacity holds the clouds of all its cavs in one frame.  `max_cav` is at most 16, the limit of heal_box_decode_nms_late.

    With `eval_thresholds` every graph ends in heal_eval_tp_fp_counted: `submit(batch_data, gt_boxes)` takes the frame's GT
    ((G, 8, 3) fp32 corners, the reference's `post_processor.generate_gt_bbx(batch_data)`: the union of every cav's objects, so
    `gt_capacity`, by default `postprocess_params['max_num']`, may need to be larger), and `stream.result_stat` gains each
    frame once, in frame order, in the reference's format, as in SceneStream.

    Inputs and GT are device or pinned host tensors; the per-cav point offsets and host-side poses go through the slot's pinned
    staging tensors, so `submit` issues no pageable copy and reads nothing back for a list its slot holds.  Memory: the graphs
    of slot k are captured into one private pool, read slot k's one set of input buffers (every modality at its capacity, for
    max_cav cavs) and one (max_cav, 4, 4) transforms buffer, and write slot k's one set of post-processing (sized for max_cav
    cavs) and evaluation buffers, which lie outside the pool.  Graphs of one slot never run at once, so they share their
    scratch: a frame's device results are valid only until its slot's next replay; the host results are valid until the slot's
    next copy-out, `depth` submits later, as in FramePipeline."""

    def __init__(self, model, capacities, max_cav: int, postprocess_params, depth: int = 2, max_graphs: int = 16,
                 voxel_limits=None, device=None, eval_thresholds=None, gt_capacity=None):
        if not _count(max_cav) or max_cav > 16:
            raise ValueError(f"max_cav {max_cav!r}: 1 to 16 cavs, the limit of heal_box_decode_nms_late")
        dev = device or next(model.parameters()).device
        depth = max(1, int(depth))
        self.model, self.capacities, self.max_cav = model, dict(capacities), int(max_cav)
        self.postprocess_params, self.voxel_limits = postprocess_params, voxel_limits
        thresholds, self.gt_capacity = eval_setup(postprocess_params, eval_thresholds, gt_capacity)
        spec = scene_spec(model.sensor_type_dict, list(self.capacities), self.capacities)
        self.cache = late_cache(model.sensor_type_dict, self.capacities, self.max_cav, _voxel_limits(model, spec, voxel_limits),
                                depth, max_graphs, self._capture, self.gt_capacity)
        self.inputs = [_input_buffers({m: dict(sp, agents=self.max_cav) for m, sp in spec.items()}, dev) for _ in range(depth)]
        self.transforms = [torch.eye(4, dtype=torch.float32, device=dev).repeat(self.max_cav, 1, 1) for _ in range(depth)]
        self.staging = [late_staging(self.capacities, model.sensor_type_dict, self.max_cav) for _ in range(depth)]
        self.pools = [torch.cuda.graph_pool_handle() for _ in range(depth)]
        H, W, A = _anchors(postprocess_params, "meta").shape[:3]
        self.postprocess = [ops.PostprocessBuffers(H * self.max_cav, W, A, TOP, dev) for _ in range(depth)]
        self.evals = [None] * depth
        if thresholds is not None:
            self.evals = [FrameEval(TOP, self.gt_capacity, dev) for _ in range(depth)]
        self.lists = [None] * depth                             # the modality list of the frame that last used each slot
        self._start([None] * depth, dev, 2, thresholds)

    def _capture(self, k, key):
        self.join(begin=False)          # the warm-up follows every frame in flight: slot k's last frame has left its buffers
        return LateFusionGraph(self.model, list(key), self.capacities, self.postprocess_params, device=self.dev,
                               eval_thresholds=self.eval_thresholds, gt_capacity=self.gt_capacity, inputs=self.inputs[k],
                               pool=self.pools[k], postprocess_buffers=self.postprocess[k], eval_buffers=self.evals[k],
                               transforms=self.transforms[k], voxel_limits=self.voxel_limits, staging=self.staging[k])

    def _slot(self, k, batch_data, gt_boxes=None):
        key = self.cache.check(batch_data, gt_boxes)
        g = self.cache.graph(k, key)
        self.lists[k] = key
        self._bind(k, g.results())
        return g

    def _result(self, k):
        return {**self.host_out[k], "modality_list": list(self.lists[k])}

    def submit(self, batch_data, gt_boxes=None):
        return self._submit(batch_data, gt_boxes)

    def capture(self, modality_list):
        """Capture the graphs of a cav-modality list in every slot ahead of the stream (a list a slot already holds is kept)."""
        key = self.cache.key(modality_list)
        for k in range(self.depth):
            self.cache.graph(k, key)

    @property
    def captures(self):
        """Graph captures so far, recaptures after eviction included."""
        return self.cache.captures

    @property
    def graphs_captured(self):
        """Graphs the stream holds over all slots."""
        return self.cache.graphs_captured
