"""CUDA-graph capture of one frame.  The per-frame path issues ~80-150 short kernels; replaying them as one graph
removes the Python / launch overhead (SURVEY.md 7.1 step 10).  Everything on the raw-points path is capture-safe: no host
syncs (voxel counts stay on the device), caller-independent workspaces, TMA descriptors baked against graph-pool buffers.

The scene shape (number of agents, point-buffer capacity, pairwise matrix shape) is fixed per graph; the live point count
travels in `agent_offsets[-1]` on the device, so clouds of different sizes reuse the same graph.
"""
from __future__ import annotations

import torch

from ._lib import lib


class GraphedCall:
    """Generic capture: `fn(build(buffers))` over named static input buffers.  `spec` maps a name to (shape, dtype);
    names in `varlen` may be loaded with fewer rows than their capacity (prefix copy; the live length travels in another input,
    e.g. `agent_offsets[-1]`).  Used by bench.py for the single-agent / SECOND / camera workloads."""

    def __init__(self, fn, spec, build, device, varlen=(), init=None, warmup=2):
        self.bufs = {k: torch.zeros(tuple(shape), dtype=dt, device=device) for k, (shape, dt) in spec.items()}
        self.varlen = set(varlen)
        if init is not None:
            self.load(**init)
        self.data = build(self.bufs)
        side = torch.cuda.Stream(device=device)
        side.wait_stream(torch.cuda.current_stream(device))
        with torch.cuda.stream(side), torch.no_grad():
            for _ in range(warmup):
                fn(self.data)
        torch.cuda.current_stream(device).wait_stream(side)
        torch.cuda.synchronize(device)
        self.graph = torch.cuda.CUDAGraph()
        l0 = lib.heal_launch_count()
        with torch.no_grad(), torch.cuda.graph(self.graph, capture_error_mode="thread_local"):
            self.out = fn(self.data)
        self.kernels_per_replay = int(lib.heal_launch_count() - l0)

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


class FrameGraph:
    def __init__(self, model, n_agents: int, point_capacity: int, pairwise_shape, modality: str = "m1", forward_fn=None,
                 device=None, warmup: int = 2):
        dev = device or next(model.parameters()).device
        self.points = torch.zeros((point_capacity, 4), dtype=torch.float32, device=dev)
        self.offsets = torch.zeros((n_agents + 1,), dtype=torch.int32, device=dev)
        self.pairwise = torch.zeros(tuple(pairwise_shape), dtype=torch.float64, device=dev)
        self.capacity = point_capacity
        self.data = {f"inputs_{modality}": {"points": self.points, "agent_offsets": self.offsets},
                     "agent_modality_list": [modality] * n_agents, "record_len": [n_agents],
                     "pairwise_t_matrix": self.pairwise}
        fn = forward_fn or model
        self.pairwise.copy_(torch.eye(4, dtype=torch.float64, device=dev).expand(self.pairwise.shape))
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side), torch.no_grad():
            for _ in range(warmup):
                fn(self.data)
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        self.graph = torch.cuda.CUDAGraph()
        l0 = lib.heal_launch_count()
        with torch.no_grad(), torch.cuda.graph(self.graph, capture_error_mode="thread_local"):
            self.out = fn(self.data)
        self.kernels_per_replay = int(lib.heal_launch_count() - l0)

    def load(self, points: torch.Tensor, offsets: torch.Tensor, pairwise: torch.Tensor):
        """points (P,4) f32, offsets (A+1) i32, pairwise f64 — device or pinned-host tensors (async copies on the current stream)."""
        n = points.shape[0]
        if n > self.capacity:
            raise ValueError(f"scene has {n} points, graph capacity is {self.capacity}")
        self.points[:n].copy_(points, non_blocking=True)
        self.offsets.copy_(offsets, non_blocking=True)
        self.pairwise.copy_(pairwise, non_blocking=True)

    def replay(self):
        self.graph.replay()
        return self.out


class FrameInterleaver:
    """N captured frames, each on its own stream: consecutive frames overlap on the GPU (the small latency-bound kernels at the
    head of frame i+1 -- voxeliser, VFE, stem -- and the tails / prologues of its convolutions run in the gaps of frame i).  A
    throughput device for streams of independent frames; the latency of one frame is that of a single FrameGraph or worse.

        il = FrameInterleaver(model, n_agents, point_capacity, pairwise_shape, n=2)
        out = il.submit(points, offsets, pairwise)     # device tensors of frame i; `out` is complete after il.wait(slot)
    """

    def __init__(self, model, n_agents: int, point_capacity: int, pairwise_shape, n: int = 2, modality: str = "m1", device=None):
        dev = device or next(model.parameters()).device
        self.dev, self.n = dev, n
        self.graphs = [FrameGraph(model, n_agents, point_capacity, pairwise_shape, modality, device=dev) for _ in range(n)]
        self.streams = [torch.cuda.Stream(device=dev) for _ in range(n)]
        self.count = 0
        self.join(begin=True)

    @property
    def kernels_per_replay(self):
        return self.graphs[0].kernels_per_replay

    def submit(self, points, offsets, pairwise):
        k = self.count % self.n
        with torch.cuda.stream(self.streams[k]):        # the previous use of slot k is earlier on the same stream
            self.graphs[k].load(points, offsets, pairwise)
            out = self.graphs[k].replay()
        self.count += 1
        return out

    def join(self, begin: bool):
        cur = torch.cuda.current_stream(self.dev)
        for s in self.streams:
            if begin:
                s.wait_stream(cur)
            else:
                cur.wait_stream(s)


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

    OUT_KEYS = ("cls_preds", "reg_preds", "dir_preds")

    def __init__(self, model, n_agents: int, point_capacity: int, pairwise_shape, modality: str = "m1", device=None,
                 compute_streams: int = 2, depth: int = 2):
        """`depth` = captured frames (slots) in flight: `submit` of frame i returns the predictions of frame i - (depth - 1).
        depth 2 keeps one frame queued behind the running one; deeper pipelines keep both compute streams fed while the host
        waits for a result (on C2 depths 2-4 measure the same within run-to-run noise, 290-305 frames/s end to end)."""
        dev = device or next(model.parameters()).device
        self.dev, self.depth = dev, max(2, int(depth))
        self.graphs = [FrameGraph(model, n_agents, point_capacity, pairwise_shape, modality, device=dev) for _ in range(self.depth)]
        self.s_in, self.s_out = (torch.cuda.Stream(device=dev) for _ in range(2))
        comp = [torch.cuda.Stream(device=dev) for _ in range(2 if compute_streams >= 2 else 1)]
        self.s_comp = comp                                     # consecutive frames alternate between the compute streams
        self.ev_in = [torch.cuda.Event() for _ in range(self.depth)]
        self.ev_comp = [torch.cuda.Event() for _ in range(self.depth)]
        self.ev_out = [torch.cuda.Event() for _ in range(self.depth)]
        self.host_out = [{k: torch.empty(g.out[k].shape, dtype=g.out[k].dtype).pin_memory() for k in self.OUT_KEYS if k in g.out}
                         for g in self.graphs]
        self.count = 0
        self.h2d_bytes = 0
        self.d2h_bytes = sum(t.numel() * t.element_size() for t in self.host_out[0].values())
        cur = torch.cuda.current_stream(dev)
        for s in (self.s_in, *set(self.s_comp), self.s_out):
            s.wait_stream(cur)

    def submit(self, points: torch.Tensor, offsets: torch.Tensor, pairwise: torch.Tensor):
        d = self.depth
        k = self.count % d
        g = self.graphs[k]
        prev = None
        with torch.cuda.stream(self.s_in):
            if self.count >= d:
                self.s_in.wait_event(self.ev_comp[k])          # frame count-depth has consumed these input buffers
            g.load(points, offsets, pairwise)
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
                h.copy_(g.out[name], non_blocking=True)
            self.ev_out[k].record(self.s_out)
        if self.count >= d - 1:
            j = (self.count - (d - 1)) % d
            self.ev_out[j].synchronize()                       # frame count-(depth-1) is complete on the host
            prev = self.host_out[j]
        self.h2d_bytes = points.numel() * points.element_size() + offsets.numel() * offsets.element_size() \
            + pairwise.numel() * pairwise.element_size()
        self.count += 1
        return prev

    def drain(self):
        """Predictions of the frames still in flight, oldest first (the results `submit` has not returned yet)."""
        out = []
        for c in range(max(self.count - (self.depth - 1), 0), self.count):
            self.ev_out[c % self.depth].synchronize()
            out.append(self.host_out[c % self.depth])
        return out

    def flush(self):
        """Wait for everything in flight; returns the LAST frame's predictions."""
        if self.count == 0:
            return None
        res = self.drain()
        return res[-1]

    def join(self, begin: bool):
        """Order the pipeline's streams after (begin) / before (end) the caller's current stream, e.g. around timing events."""
        cur = torch.cuda.current_stream(self.dev)
        for s in (self.s_in, *set(self.s_comp), self.s_out):
            if begin:
                s.wait_stream(cur)
            else:
                cur.wait_stream(s)


class LateFusionGraph:
    """Late fusion of one scene as ONE captured graph: a single-agent model's `grouped_heads` (one batched forward per modality,
    every cav's heads in one (n_cav, H, W, S) buffer) and heal_box_decode_nms_late (decode with the transforms read on the device,
    sort, rotated NMS, range mask).  The reference runs one model call per cav, then the post-processor on the host.

        g = LateFusionGraph(model, ["m1", "m1", "m2"], {"m1": 200000, "m2": (4, 256, 704)}, hypes["postprocess"])
        g.load(batch_data)            # {cav_id: {inputs_<m>: ..., transformation_matrix: 4x4}} in the captured modality order
        out = g.replay()              # out.boxes[:out.count], out.scores[:out.count] on the device, no host sync

    `capacities[m]`: for a lidar modality the point capacity of ALL its cavs together (raw clouds, `points` + `agent_offsets`; the
    live counts travel in the offsets), for a camera modality (cameras, image height, image width) per cav for normalised fp32
    images, or (cameras, frame height, frame width, torch.uint8) for raw uint8 (H0, W0, 3) frames, which the encoder resizes, crops
    and normalises on the GPU.  The poses are inputs: replaying the graph for another scene uses that scene's transforms."""

    CAMERA_KEYS = ("rots", "trans", "intrins", "post_rots", "post_trans")

    def __init__(self, model, modality_of_each_cav, capacities, postprocess_params, device=None, warmup: int = 2, top: int = 1000):
        from . import ops
        from .data_utils.post_processor.voxel_postprocessor import VoxelPostprocessor
        dev = device or next(model.parameters()).device
        self.modalities = list(modality_of_each_cav)
        n = len(self.modalities)
        self.groups = {}
        for i, m in enumerate(self.modalities):
            self.groups.setdefault(m, []).append(i)
        self.inputs = {}
        for m, idx in self.groups.items():
            k = len(idx)
            if model.sensor_type_dict[m] == "camera":
                cams, h, w, *dtype = capacities[m]
                if dtype and dtype != [torch.uint8]:
                    raise ValueError(f"{m}: camera capacity {capacities[m]}; (cams, h, w) takes normalised fp32 images and "
                                     "(cams, H0, W0, torch.uint8) raw frames")
                imgs = torch.zeros((k, cams, h, w, 3), dtype=torch.uint8, device=dev) if dtype else \
                    torch.zeros((k, cams, 3, h, w), dtype=torch.float32, device=dev)
                self.inputs[m] = {"imgs": imgs,
                                  "rots": torch.eye(3, device=dev).repeat(k, cams, 1, 1),
                                  "trans": torch.zeros((k, cams, 3), dtype=torch.float32, device=dev),
                                  "intrins": torch.eye(3, device=dev).repeat(k, cams, 1, 1),
                                  "post_rots": torch.eye(3, device=dev).repeat(k, cams, 1, 1),
                                  "post_trans": torch.zeros((k, cams, 3), dtype=torch.float32, device=dev)}
            else:
                self.inputs[m] = {"points": torch.zeros((int(capacities[m]), 4), dtype=torch.float32, device=dev),
                                  "agent_offsets": torch.zeros((k + 1,), dtype=torch.int32, device=dev)}
        self.transforms = torch.eye(4, dtype=torch.float32, device=dev).repeat(n, 1, 1).contiguous()
        pp = VoxelPostprocessor(postprocess_params, False)
        self.anchors = torch.from_numpy(pp.generate_anchor_box()).to(device=dev, dtype=torch.float32).contiguous()
        A = self.anchors.shape[2]
        dargs = postprocess_params.get('dir_args', {})
        bins = int(dargs.get('num_bins', 2))
        self.buffers = ops.PostprocessBuffers(self.anchors.shape[0] * n, self.anchors.shape[1], A, top, dev)

        def run():
            y, _ = model.grouped_heads(self.groups, self.inputs, n)
            return ops.box_decode_nms_late(y, y, y, self.anchors, self.transforms,
                                           postprocess_params['target_args']['score_threshold'], postprocess_params['nms_thresh'],
                                           dir_offset=dargs.get('dir_offset', 0.0), num_bins=bins, order=postprocess_params['order'],
                                           gt_range=postprocess_params['gt_range'], top=top, buffers=self.buffers,
                                           coffsets=(0, A, 8 * A))

        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side), torch.no_grad():
            for _ in range(warmup):
                run()
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        self.graph = torch.cuda.CUDAGraph()
        l0 = lib.heal_launch_count()
        with torch.no_grad(), torch.cuda.graph(self.graph, capture_error_mode="thread_local"):
            self.out = run()
        self.kernels_per_replay = int(lib.heal_launch_count() - l0)

    def load(self, batch_data):
        """Copy a scene's inputs and cav -> ego transforms into the captured buffers (asynchronous copies on the current stream).
        The cavs must come in the captured modality order; each lidar cav carries one raw cloud (`points`, `agent_offsets`)."""
        from .models.heter_model_late import modality_of
        cavs = list(batch_data.keys())
        mods = [modality_of(batch_data[c]) for c in cavs]
        if mods != self.modalities:
            raise ValueError(f"scene modalities {mods}, the graph was captured for {self.modalities}")
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
                buf["agent_offsets"].copy_(torch.tensor(offs, dtype=torch.int32), non_blocking=True)
            else:
                for j, i in enumerate(idx):
                    src = batch_data[cavs[i]][f"inputs_{m}"]
                    for k in ("imgs",) + self.CAMERA_KEYS:
                        raw = k == "imgs" and buf[k].dtype == torch.uint8         # raw frames (cams, H0, W0, 3) go in whole
                        buf[k][j].copy_(src[k][0][:, :3] if k == "imgs" and not raw else src[k][0], non_blocking=True)
        T = torch.stack([torch.as_tensor(batch_data[c]['transformation_matrix']).reshape(4, 4).to(torch.float32) for c in cavs])
        self.transforms.copy_(T, non_blocking=True)

    def replay(self):
        self.graph.replay()
        return self.out
