"""Scene-parallel inference over agents: one process per GPU, rank r owns a contiguous slice of the scene's agents
(voxelize -> encoder -> per-agent backbone -> ResNeXt pyramid levels + occupancy heads), ONE all-gather of the packed
per-agent pyramid (NCCL over NVLink 5 / NVSwitch; gloo in the CPU tests), then every rank runs the fusion, decode,
shrink and heads on the gathered maps (SURVEY.md 8e, variant B).  The reference has no counterpart: it stacks all
agents on one GPU (intermediate_heter_fusion_dataset.py:619,662) and DDP shards scenes, not agents.

Packed message per agent (bytes): [level0 | level1 | level2 | occ0 | occ1 | occ2] where a level is the agent's feature
map in the conv engine's storage format laid out (planes, H, W, C) and occ is fp32 (h, w).  For the HEAL pyramid at a
256x256 fusion map that is 64*256^2 + 128*128^2 + 256*64^2 (x4 bytes, split-bf16 or fp32) + 86016*4 = 29.7 MB.
"""
from __future__ import annotations

from typing import List, Sequence, Tuple

import torch
import torch.distributed as dist


def agent_plan(n_agents: int, world: int) -> List[List[int]]:
    """Contiguous, balanced assignment of agents to ranks: the first n % world ranks hold ceil(n/world) agents, the others
    floor(n/world) (5 agents on 4 ranks = 2+1+1+1); every rank's chunk of the gather buffer has ceil(n/world) slots."""
    base, extra = divmod(n_agents, world)
    plan, a = [], 0
    for r in range(world):
        k = base + (1 if r < extra else 0)
        plan.append(list(range(a, a + k)))
        a += k
    return plan


def message_layout(level_shapes: Sequence[Tuple[int, int, int, int]], occ_shapes: Sequence[Tuple[int, int]], elem_bytes: int = 2):
    """level_shapes: (planes, H, W, C) per level (bf16 elements; fp32 storage = planes 2 worth of bytes with elem_bytes 2);
    occ_shapes: (h, w) fp32.  Returns (offsets in bytes per segment, total bytes padded to 16)."""
    offs, o = [], 0
    for (p, h, w, c) in level_shapes:
        offs.append(o)
        o += p * h * w * c * elem_bytes
    for (h, w) in occ_shapes:
        offs.append(o)
        o += h * w * 4
    return offs, (o + 15) // 16 * 16


def pack_agents(levels: Sequence[torch.Tensor], occs: Sequence[torch.Tensor], slots: int) -> torch.Tensor:
    """levels[i]: (n_local, planes, H, W, C) any dtype; occs[i]: (n_local, h, w) fp32 -> uint8 (slots, msg_bytes), zero padded."""
    n_local = levels[0].shape[0] if len(levels) else 0
    parts = [l.contiguous().view(torch.uint8).reshape(n_local, -1) for l in levels] + \
            [o.contiguous().view(torch.uint8).reshape(n_local, -1) for o in occs]
    msg = torch.cat(parts, dim=1) if n_local > 0 else None
    nbytes = sum(int(p.shape[1]) for p in parts) if n_local > 0 else None
    if n_local == 0:
        raise ValueError("pack_agents needs at least one local agent (use zero-filled maps for an idle rank)")
    pad = (nbytes + 15) // 16 * 16
    out = torch.zeros((slots, pad), dtype=torch.uint8, device=levels[0].device)
    out[:n_local, :nbytes] = msg
    return out


def unpack_agents(buf: torch.Tensor, level_shapes, level_dtypes, occ_shapes, agent_slots: Sequence[int]):
    """buf: uint8 (total_slots, msg_bytes); agent_slots: slot index of each real agent in scene order.
    Returns (levels [(n, planes, H, W, C)], occs [(n, h, w) fp32])."""
    idx = torch.as_tensor(list(agent_slots), dtype=torch.long, device=buf.device)
    rows = buf.index_select(0, idx)
    levels, occs, o = [], [], 0
    for shp, dt in zip(level_shapes, level_dtypes):
        nb = int(torch.tensor([], dtype=dt).element_size())
        n = 1
        for v in shp:
            n *= v
        levels.append(rows[:, o:o + n * nb].contiguous().view(dt).view(len(agent_slots), *shp))
        o += n * nb
    for (h, w) in occ_shapes:
        occs.append(rows[:, o:o + h * w * 4].contiguous().view(torch.float32).view(len(agent_slots), h, w))
        o += h * w * 4
    return levels, occs


def all_gather_bytes(local: torch.Tensor, world: int) -> torch.Tensor:
    """(slots, B) uint8 per rank -> (world*slots, B): the single collective of the path."""
    out = torch.empty((world * local.shape[0], local.shape[1]), dtype=torch.uint8, device=local.device)
    dist.all_gather_into_tensor(out, local.contiguous())
    return out


def _refuse_compressor(model):
    if getattr(model, "compress", False):
        raise NotImplementedError(f"{type(model).__name__} with a `compressor:`: the agent-sharded path does not apply the "
                                  "compressor; run the model on one GPU")


def forward_agent_sharded(model, data_dict, rank: int, world: int):
    """HeterPyramidCollab.forward with the per-agent part sharded over `world` ranks (single lidar modality 'm1').
    data_dict carries the WHOLE scene on every rank (raw points + agent_offsets); each rank touches only its agents' points."""
    _refuse_compressor(model)
    from . import ops
    from .engine import act_fmt
    from .utils.transformation_utils import normalize_pairwise_tfm
    aml = data_dict['agent_modality_list']
    n_agents = len(aml)
    assert all(a == aml[0] for a in aml), "agent-sharded path is implemented for single-modality scenes"
    m = aml[0]
    plan = agent_plan(n_agents, world)
    mine = plan[rank]
    slots = len(plan[0])
    inp = data_dict[f'inputs_{m}']
    offs_host = inp.get('agent_offsets_host')
    if offs_host is None:
        offs_host = inp['agent_offsets'].cpu().tolist()           # one-time host copy when the caller did not provide it
    pb = model.pyramid_backbone
    fmt = act_fmt()
    # ---- local agents: encoder -> backbone -> aligner -> ResNeXt levels + occ heads ---------------------
    idle = len(mine) == 0
    use = mine if not idle else [0]                                # an idle rank computes agent 0 and discards it
    lo, hi = offs_host[use[0]], offs_host[use[-1] + 1]
    sub_offs = torch.tensor([o - lo for o in offs_host[use[0]:use[-1] + 2]], dtype=torch.int32, device=inp['points'].device)
    sub = {f'inputs_{m}': {'points': inp['points'][lo:hi], 'agent_offsets': sub_offs}}
    x = getattr(model, f"aligner_{m}").forward_nhwc(model._encode(sub, m))
    feats = pb.multiscale_nhwc(x)
    occs = [pb._occ_nhwc(f, i) for i, f in enumerate(feats)]
    def per_agent(a: "ops.Act"):
        t = a.t if a.fmt != "f32" else a.t.unsqueeze(0)
        return t.permute(1, 0, 2, 3, 4).contiguous()               # (n_local, planes|1, H, W, C)
    lv = [per_agent(f) for f in feats]
    oc = [o.t.view(o.N, o.H, o.W) for o in occs]
    level_shapes = [tuple(l.shape[1:]) for l in lv]
    level_dtypes = [l.dtype for l in lv]
    occ_shapes = [tuple(o.shape[1:]) for o in oc]
    if idle:
        lv = [torch.zeros_like(l) for l in lv]
        oc = [torch.zeros_like(o) for o in oc]
    local = pack_agents(lv, oc, slots)
    # ---- the one exchange step -------------------------------------------------------------------------------
    with ops._Prof("allgather_bev_pyramid"):
        gathered = all_gather_bytes(local, world) if world > 1 else local
    agent_slots = [r * slots + s for r in range(world) for s in range(len(plan[r]))]
    g_levels, g_occs = unpack_agents(gathered, level_shapes, level_dtypes, occ_shapes, agent_slots)
    # ---- replicated tail: fuse x3 -> decode -> shrink -> heads ------------------------------------------------
    rng = model.cav_range
    affine = normalize_pairwise_tfm(data_dict['pairwise_t_matrix'], model.H, model.W, model.fake_voxel_size)
    from .models.fuse_modules.pyramid_fuse import weighted_fuse_nhwc
    fused = []
    for lvl, occ in zip(g_levels, g_occs):
        t = lvl.permute(1, 0, 2, 3, 4).contiguous()                 # (planes, n, H, W, C)
        act = ops.Act(t if fmt != "f32" else t[0], fmt)
        fused.append(weighted_fuse_nhwc(act, occ.contiguous(), data_dict['record_len'], affine, pb.align_corners, None))
    f = pb.decode_nhwc(fused)
    if model.shrink_flag:
        f = model.shrink_conv.forward_nhwc(f)
    cls, reg, dirp = model._heads(f)
    return {'pyramid': 'collab', 'cls_preds': cls, 'reg_preds': reg, 'dir_preds': dirp,
            'occ_single_list': [o.unsqueeze(1) for o in g_occs]}


# ======================================================================================================================
# Graph-captured agent-per-GPU frame (SURVEY.md 8e, variant B) with a row-sharded fusion tail
# ======================================================================================================================
def rank_layout(level_shapes: Sequence[Tuple[int, int, int]], planes: int, slots: int):
    """Byte layout of ONE rank's chunk of the symmetric gather buffer: for every pyramid level a dense
    (planes, slots, H, W, C) bf16 block (fp32 storage: planes = 2 worth of bytes), then per level a (slots, H, W) fp32 occupancy
    block.  Level-major inside the chunk so that a rank's local agents form ordinary dense `Act`s the conv epilogues write into.
    Returns (feat byte offsets, occ byte offsets, chunk bytes padded to 256)."""
    foffs, ooffs, o = [], [], 0
    for (h, w, c) in level_shapes:
        foffs.append(o)
        o += planes * slots * h * w * c * 2
    for (h, w, c) in level_shapes:
        ooffs.append(o)
        o += slots * h * w * 4
    return foffs, ooffs, (o + 255) // 256 * 256


def agent_offsets_in_gather(plan, level_shapes, planes: int, slots: int, elem_bytes: int = 2):
    """For every level: (feature element offsets, occupancy float offsets) of each REAL agent, in scene order, from the base of
    the gathered (world, chunk) buffer -- the table heal_pyramid_fuse_level reads the agents through (no unpack copy)."""
    foffs, ooffs, chunk = rank_layout(level_shapes, planes, slots)
    table = []
    for li, (h, w, c) in enumerate(level_shapes):
        fo, oo = [], []
        for r, agents in enumerate(plan):
            for s in range(len(agents)):
                fo.append((r * chunk + foffs[li]) // elem_bytes + s * h * w * c)
                oo.append((r * chunk + ooffs[li]) // 4 + s * h * w)
        table.append((fo, oo))
    return table


def tail_rows(H: int, rank: int, world: int):
    """Row partition of the fused map for the replicated tail (deblocks -> shrink 3x3 x2 -> heads): rank r produces head rows
    [r0, r1); it needs the second 3x3's input rows [b0, b1) = [r0-1, r1+1) and the first 3x3's input (the 384-channel concat)
    rows [c0, c1) = [r0-2, r1+2) rounded out to multiples of 4 (the coarsest pyramid level is 4x smaller), all clamped to the map.
    Returns None when H does not split evenly (callers then run the tail replicated)."""
    if world < 2 or H % world or (H // world) % 4:
        return None
    per = H // world
    r0, r1 = rank * per, (rank + 1) * per
    c0, c1 = max(0, (r0 - 2) // 4 * 4), min(H, -(-(r1 + 2) // 4) * 4)
    b0, b1 = max(0, r0 - 1), min(H, r1 + 1)
    return {"r": (r0, r1), "b": (b0, b1), "c": (c0, c1)}


class SymmetricExchange:
    """A symmetric device buffer (same size on every rank, every peer's copy mapped into this process through
    torch.distributed._symmetric_memory = CUDA IPC / fabric handles over NVLink) + the two heal_p2p_* primitives on it:
    `push` (my slice -> the same offset of every peer's copy) and `signal_wait` (flag barrier, monotonically increasing
    sequence numbers kept in device memory so that CUDA-graph replays keep counting)."""

    N_BARRIERS = 4

    @staticmethod
    def usable(device, group=None) -> bool:
        """True when EVERY rank of the group can allocate symmetric memory (checked before the collective rendezvous, so a rank
        without support cannot leave the others waiting): the `comm="auto"` choice between the P2P push and NCCL."""
        ok = 1
        try:
            import torch.distributed._symmetric_memory as symm_mem
            g = group if group is not None else dist.group.WORLD
            try:
                symm_mem.enable_symm_mem_for_group(g.group_name)
            except Exception:
                pass
            symm_mem.empty(256, dtype=torch.uint8, device=device)
        except Exception:
            ok = 0
        t = torch.tensor([ok], dtype=torch.int32, device=device)
        dist.all_reduce(t, op=dist.ReduceOp.MIN, group=group)
        return int(t.item()) == 1

    def __init__(self, nbytes: int, device, group=None):
        import ctypes
        import torch.distributed._symmetric_memory as symm_mem
        self.group = group if group is not None else dist.group.WORLD
        self.rank, self.world = dist.get_rank(self.group), dist.get_world_size(self.group)
        name = self.group.group_name
        try:
            symm_mem.enable_symm_mem_for_group(name)
        except Exception:
            pass                                           # newer torch enables it implicitly
        nbytes = (int(nbytes) + 255) // 256 * 256
        self.buf = symm_mem.empty(nbytes, dtype=torch.uint8, device=device)
        self.flags = symm_mem.empty(4096, dtype=torch.uint8, device=device)
        self.buf.zero_()
        self.flags.zero_()
        self.hdl = symm_mem.rendezvous(self.buf, self.group)
        self.fhdl = symm_mem.rendezvous(self.flags, self.group)
        self.ptrs = [int(p) for p in self.hdl.buffer_ptrs]
        self.fptrs = [int(p) for p in self.fhdl.buffer_ptrs]
        assert self.ptrs[self.rank] == self.buf.data_ptr() and len(self.ptrs) == self.world
        self.seq = torch.zeros((self.N_BARRIERS,), dtype=torch.int32, device=device)
        torch.cuda.synchronize(device)
        dist.barrier(group=self.group)                     # everybody's zero-fill is done before anybody pushes
        self._vp, self._arr = ctypes.c_void_p, ctypes.c_void_p * self.world

    def push(self, byte_off: int, nbytes: int):
        """copy buf[byte_off : byte_off+nbytes] (16-byte aligned) to the same offset of every peer's buffer, on the current stream"""
        from ._lib import lib, check
        dst = self._arr(*[p + byte_off for p in self.ptrs])
        check(lib.heal_p2p_push(self._vp(self.ptrs[self.rank] + byte_off), dst, self.world, self.rank, int(nbytes),
                                self._vp(torch.cuda.current_stream().cuda_stream)), "heal_p2p_push")

    def signal_wait(self, which: int):
        """barrier `which`: everybody's earlier pushes (on their streams) are visible in my buffer when this kernel completes"""
        from ._lib import lib, check
        fl = self._arr(*[p + which * 256 for p in self.fptrs])
        check(lib.heal_p2p_signal_wait(fl, self.world, self.rank, self._vp(self.seq.data_ptr() + 4 * which),
                                       self._vp(torch.cuda.current_stream().cuda_stream)), "heal_p2p_signal_wait")


class AgentShardedFrame:
    """One scene, agents sharded over `world` ranks, captured as CUDA graphs on every rank:

        voxelize -> PillarVFE -> per-agent ResNet -> ResNeXt levels + occupancy heads      (my agents; the last conv of every
                                                                                             level and the occupancy heads write
                                                                                             straight into my chunk of the
                                                                                             symmetric gather buffer)
        exchange of the BEV pyramids                                                        comm='p2p' (default): each level's block
                                                                                             is PUSHED to every peer over NVLink by
                                                                                             heal_p2p_push on a side stream while the
                                                                                             next level computes, then one flag barrier;
                                                                                             comm='nccl': ONE in-place ncclAllGather
        warp + weighted fuse x3 -> deblocks -> shrink 3x3 x2 -> heads                      for MY slab of output rows only, read
                                                                                             straight from the gathered buffer
        exchange of the head rows (5 MB in total)                                           p2p push + flag barrier | ncclAllGather

    No torch.cat / index_select / permute copies on the data path.  `load_scene` copies only this rank's agents' points.
    p2p mode double-buffers the gather buffer (a fast rank may push frame k+1 while a slow one still fuses frame k), so two graphs
    are captured and replayed alternately; the flag barrier of frame k+1 cannot pass before every rank has finished frame k."""

    def __init__(self, model, n_agents: int, rank: int, world: int, point_capacity: int, pairwise_shape, device=None,
                 modality: str = "m1", shard_tail: bool = True, group=None, comm: str = "auto"):
        _refuse_compressor(model)
        from . import ops
        from .engine import act_fmt
        from .graph import record, warm_up
        dev = device or next(model.parameters()).device
        self.model, self.rank, self.world, self.dev, self.group = model, rank, world, dev, group
        self.n_agents, self.m = n_agents, modality
        self.plan = agent_plan(n_agents, world)
        self.slots = len(self.plan[0])
        self.mine = self.plan[rank]
        pb = model.pyramid_backbone
        fmt = act_fmt()
        self.fmt = fmt
        planes = 2 if fmt in ("split", "f32") else 1            # f32 storage = two bf16 planes worth of bytes
        H0 = int(round((model.cav_range[4] - model.cav_range[1]) / model.args[modality]['encoder_args']['voxel_size'][1])) // 2
        W0 = int(round((model.cav_range[3] - model.cav_range[0]) / model.args[modality]['encoder_args']['voxel_size'][0])) // 2
        nf = pb.model_cfg['num_filters']
        strides = pb.model_cfg['layer_strides']
        shapes, h, w = [], H0, W0
        for c, s in zip(nf, strides):
            h, w = (h - 1) // s + 1, (w - 1) // s + 1
            shapes.append((h, w, c))
        self.level_shapes, self.planes = shapes, planes
        self.foffs, self.ooffs, self.chunk = rank_layout(shapes, planes, self.slots)
        self.table = agent_offsets_in_gather(self.plan, shapes, planes, self.slots, 4 if fmt == "f32" else 2)
        self.Hf, self.Wf = shapes[0][0], shapes[0][1]
        self.rows = tail_rows(self.Hf, rank, world) if shard_tail else None
        self.n_head = model.cls_head.out_channels + model.reg_head.out_channels + model.dir_head.out_channels
        head_bytes = self.Hf * self.Wf * self.n_head * 4
        if comm == "auto":
            comm = "p2p" if (world > 1 and SymmetricExchange.usable(dev, group)) else "nccl"
        self.comm = comm
        nsides = 2 if (comm == "p2p" and world > 1) else 1
        gather_bytes = world * self.chunk
        if comm == "p2p" and world > 1:
            # one symmetric allocation: [gather side 0 | gather side 1 | heads]
            self.sym = SymmetricExchange(nsides * gather_bytes + head_bytes, dev, group)
            base = self.sym.buf
            gathers = [base[i * gather_bytes:(i + 1) * gather_bytes].view(world, self.chunk) for i in range(nsides)]
            self.gather_off = [i * gather_bytes for i in range(nsides)]
            self.heads_off = nsides * gather_bytes
            self.heads = base[self.heads_off:self.heads_off + head_bytes].view(torch.float32).view(1, self.Hf, self.Wf, self.n_head)
        else:
            self.sym = None
            gathers = [torch.zeros((world, self.chunk), dtype=torch.uint8, device=dev)]
            self.heads = torch.zeros((1, self.Hf, self.Wf, self.n_head), dtype=torch.float32, device=dev)
        S = self.slots
        self.sides = []
        for g in gathers:
            mychunk = g[rank]
            level_out, occ_out = [], []
            for (h, w, c), fo, oo in zip(shapes, self.foffs, self.ooffs):
                if fmt == "f32":
                    t = mychunk[fo:fo + S * h * w * c * 4].view(torch.float32).view(S, h, w, c)
                else:
                    t = mychunk[fo:fo + planes * S * h * w * c * 2].view(torch.bfloat16).view(planes, S, h, w, c)
                level_out.append(ops.Act(t, fmt))
                occ_out.append(ops.Act(mychunk[oo:oo + S * h * w * 4].view(torch.float32).view(S, h, w, 1), "f32"))
            self.sides.append({"i": len(self.sides), "gather": g, "level_out": level_out, "occ_out": occ_out})
        # static inputs: my agents' points (idle slots = empty clouds), their offsets, the scene's pairwise matrix
        self.cap = point_capacity
        self.points = torch.zeros((point_capacity, 4), dtype=torch.float32, device=dev)
        self.offsets = torch.zeros((S + 1,), dtype=torch.int32, device=dev)
        self.pairwise = torch.zeros(tuple(pairwise_shape), dtype=torch.float64, device=dev)
        self.pairwise.copy_(torch.eye(4, dtype=torch.float64, device=dev).expand(self.pairwise.shape))
        self._offs_ring = [torch.zeros((S + 1,), dtype=torch.int32).pin_memory() for _ in range(8)]
        self._ring_i = 0
        self.tail_mode = ("row-sharded (rows %d..%d of %d per rank) + exchange of the head rows" % (self.rows["r"][0], self.rows["r"][1], self.Hf)
                          if self.rows else "replicated on every rank")
        self.exchanges_per_frame = (2 if self.rows else 1) if world > 1 else 0          # pyramid (+ head rows)
        self.collectives_per_frame = self.exchanges_per_frame if comm == "nccl" else 0  # NCCL calls inside the frame
        self.side_stream = torch.cuda.Stream(device=dev)
        # warm-up (every side), then capture one graph per side
        warm_up(lambda: [self._frame(sd) for sd in self.sides], dev)
        if world > 1:
            dist.barrier(group=group)
        kernels = 0
        for sd in self.sides:
            sd["graph"], sd["out"], k = record(lambda: self._frame(sd))
            kernels += k
        self.kernels_per_replay = kernels // len(self.sides)
        self.count = 0
        self.out = self.sides[0]["out"]

    # ---- host side --------------------------------------------------------------------------------------------------
    def load_scene(self, points: torch.Tensor, offsets_host, pairwise: torch.Tensor):
        """points: the WHOLE scene's (P,4) clouds (device or pinned host), offsets_host: (n_agents+1) python/numpy ints.
        Only this rank's agents are copied; idle slots (and an idle rank) get empty clouds."""
        offs = [int(v) for v in offsets_host]
        S = self.slots
        if self.mine:
            lo, hi = offs[self.mine[0]], offs[self.mine[-1] + 1]
            local = [offs[a] - lo for a in self.mine] + [hi - lo]
        else:
            lo = hi = 0
            local = [0]
        local = local + [local[-1]] * (S + 1 - len(local))
        if hi - lo > self.cap:
            raise ValueError(f"{hi - lo} points for this rank, capacity {self.cap}")
        if hi > lo:
            self.points[:hi - lo].copy_(points[lo:hi], non_blocking=True)
        stage = self._offs_ring[self._ring_i]
        self._ring_i = (self._ring_i + 1) % len(self._offs_ring)
        stage.copy_(torch.tensor(local, dtype=torch.int32))
        self.offsets.copy_(stage, non_blocking=True)
        self.pairwise.copy_(pairwise, non_blocking=True)

    def replay(self):
        sd = self.sides[self.count % len(self.sides)]
        self.count += 1
        sd["graph"].replay()
        self.out = sd["out"]
        return self.out

    # ---- the frame (captured) ---------------------------------------------------------------------------------------
    def _exchange_pyramid_nccl(self, sd):
        if self.world > 1:
            dist.all_gather_into_tensor(sd["gather"].view(-1), sd["gather"][self.rank], group=self.group)

    def _push_on_side_stream(self, byte_off, nbytes):
        """fork: the side stream waits for everything issued so far on the current stream, then pushes"""
        cur = torch.cuda.current_stream(self.dev)
        self.side_stream.wait_stream(cur)
        with torch.cuda.stream(self.side_stream):
            self.sym.push(byte_off, nbytes)

    def _frame(self, sd):
        from . import ops
        from .engine import conv_bn_act, act_fmt
        from .utils.transformation_utils import normalize_pairwise_tfm
        from .models.sub_modules.base_bev_backbone_resnet import decode_levels
        model, m = self.model, self.m
        pb = model.pyramid_backbone
        p2p = self.sym is not None
        side_i = sd["i"]
        sub = {f'inputs_{m}': {'points': self.points, 'agent_offsets': self.offsets}}
        x = getattr(model, f"aligner_{m}").forward_nhwc(model._encode(sub, m))
        # ResNeXt levels: the last conv of each level writes into my chunk of the gather buffer; in p2p mode the level's block is
        # pushed to the peers on the side stream while the next level computes
        S = self.slots
        feats = []
        for li in range(pb.resnet.layernum):
            x = pb.resnet._run_level(getattr(pb.resnet, f"layer{li}"), x, out=sd["level_out"][li])
            feats.append(x)
            if p2p:
                h, w, c = self.level_shapes[li]
                self._push_on_side_stream(self.gather_off[side_i] + self.rank * self.chunk + self.foffs[li], self.planes * S * h * w * c * 2)
        for li, f in enumerate(feats):
            pb._occ_nhwc(f, li, out=sd["occ_out"][li])
        if p2p:
            occ_bytes = sum(S * h * w * 4 for (h, w, c) in self.level_shapes)
            self._push_on_side_stream(self.gather_off[side_i] + self.rank * self.chunk + self.ooffs[0], (occ_bytes + 15) // 16 * 16)
            torch.cuda.current_stream(self.dev).wait_stream(self.side_stream)      # join
            self.sym.signal_wait(0)                                                   # everybody's pyramid is in my buffer
        else:
            self._exchange_pyramid_nccl(sd)
        gather = sd["gather"]
        affine = normalize_pairwise_tfm(self.pairwise, model.H, model.W, model.fake_voxel_size)
        theta = affine[0, 0, :self.n_agents].contiguous()
        occ_base = gather.view(-1).view(torch.float32)
        fmt = self.fmt
        fused = []
        rows = self.rows
        for li, (h, w, c) in enumerate(self.level_shapes):
            base = gather.view(-1)
            if fmt == "f32":
                geo = ops.Act(base[:h * w * c * 4].view(torch.float32).view(1, h, w, c), "f32")
            else:
                planes = 2 if fmt == "split" else 1
                # geometry of ONE agent's map at the buffer base; plane stride = slots*h*w*c elements (level-major chunk layout)
                t = torch.as_strided(base.view(torch.bfloat16), (planes, 1, h, w, c), (S * h * w * c, h * w * c, w * c, c, 1))
                geo = ops.Act(t, fmt)
            sc = self.Hf // h
            rr = (rows["c"][0] // sc, (rows["c"][1] - rows["c"][0]) // sc) if rows else None
            fused.append(ops.pyramid_fuse_level(geo, occ_base, theta, pb.align_corners, None, out_fmt=fmt,
                                                agent_offsets=self.table[li], n_agents=self.n_agents, rows=rr))
        f = decode_levels(pb.deblocks, fused)                          # (1, c1-c0 | H, W, 384)
        dc = model.shrink_conv.layers[0].double_conv if model.shrink_flag else None
        if rows is None:
            if model.shrink_flag:
                f = model.shrink_conv.forward_nhwc(f)
            self._head_conv(f, self.heads_act())
        else:
            assert model.shrink_flag and len(model.shrink_conv.layers) == 1, "row-sharded tail expects the single DoubleConv shrink header"
            (r0, r1), (b0, b1), (c0, c1) = rows["r"], rows["b"], rows["c"]
            a = conv_bn_act(f, dc[0], None, relu=True)                 # rows [c0, c1); valid on [c0+1, c1-1) (or to the map border)
            b = conv_bn_act(a.rows(b0 - c0, b1 - c0), dc[2], None, relu=True)   # rows [b0, b1); valid on [r0, r1)
            self._head_conv(b.rows(r0 - b0, r1 - b0), self.heads_act().rows(r0, r1))
            row_bytes = self.Wf * self.n_head * 4
            if p2p:
                self.sym.push(self.heads_off + r0 * row_bytes, (r1 - r0) * row_bytes)
                self.sym.signal_wait(1)
            elif self.world > 1:
                dist.all_gather_into_tensor(self.heads.view(-1), self.heads[0, r0:r1].reshape(-1), group=self.group)
        o, outs = 0, {}
        for name, head in (("cls_preds", model.cls_head), ("reg_preds", model.reg_head), ("dir_preds", model.dir_head)):
            outs[name] = self.heads[..., o:o + head.out_channels].permute(0, 3, 1, 2).contiguous()
            o += head.out_channels
        outs['pyramid'] = 'collab'
        return outs

    def heads_act(self):
        from . import ops
        return ops.Act(self.heads, "f32")

    def _head_conv(self, x, out_act):
        from .engine import conv_bn_act
        fh = self.model._heads
        fh.prepare()
        conv_bn_act(x, fh._conv, None, relu=False, out=out_act, out_fmt="f32")

    def time_exchange(self, iters: int = 20):
        """The pyramid exchange alone (same buffers, outside the graph): CUDA-event ms per exchange on this rank.
        nccl: one all_gather_into_tensor; p2p: the pushes of all levels + the flag barrier (no compute to overlap with)."""
        torch.cuda.synchronize(self.dev)
        if self.world > 1:
            dist.barrier(group=self.group)
        sd = self.sides[0]
        S = self.slots

        def once():
            if self.sym is None:
                self._exchange_pyramid_nccl(sd)
                return
            for li, (h, w, c) in enumerate(self.level_shapes):
                self.sym.push(self.gather_off[0] + self.rank * self.chunk + self.foffs[li], self.planes * S * h * w * c * 2)
            occ_bytes = sum(S * h * w * 4 for (h, w, c) in self.level_shapes)
            self.sym.push(self.gather_off[0] + self.rank * self.chunk + self.ooffs[0], (occ_bytes + 15) // 16 * 16)
            self.sym.signal_wait(2)
        for _ in range(3):
            once()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            once()
        b.record()
        torch.cuda.synchronize(self.dev)
        return {"ms": a.elapsed_time(b) / iters, "bytes_per_rank": int(self.chunk), "comm": self.comm}

    time_allgather = time_exchange
