"""Tensor-level wrappers over the C ABI (include/heal_b200.h).

PyTorch is used here only for device memory, streams and shapes: every wrapper passes raw device
pointers + the current CUDA stream to libheal_b200.so.  There is no eager / CPU fallback: a tensor
that is not on a CUDA device raises.

Activations travel between kernels as `Act` objects: channels-last buffers in one of three storage
formats — 'f32' (N,H,W,C) fp32; 'bf16' (1,N,H,W,C) bf16; 'split' (2,N,H,W,C) bf16 planes (hi, lo) with
x ~= hi + lo (16 mantissa bits), the operand format of the wgmma fp32-equivalent convolution.
At module boundaries feature maps are *logically* (N,C,H,W) fp32 torch tensors that are *physically*
channels-last (`x.permute(0,2,3,1)` contiguous), which keeps the reference's shapes at zero cost.
"""
from __future__ import annotations

import ctypes
import functools
from typing import Optional, Sequence

import numpy as np
import torch

from ._lib import lib, check, HealAct, HealCavHeads

_vp = ctypes.c_void_p
FMT = {"f32": 0, "bf16": 1, "split": 2}


def _p(t: Optional[torch.Tensor]):
    return _vp(t.data_ptr()) if t is not None else _vp(0)


def _stream():
    """Current stream of the CURRENT device.  Every public wrapper that launches is decorated with `_guard`, which makes the
    tensors' device current first, so the launch, the stream and the per-device kernel attributes all agree."""
    return _vp(torch.cuda.current_stream().cuda_stream)


def _call(symbol: str, *args):
    """Launch `symbol` of libheal_b200.so on the current stream (appended as the last argument); raise on an error code.
    Pass `Act.view()` results as they are: ctypes passes a HealAct by reference where the argtype is a pointer to it."""
    check(getattr(lib, symbol)(*args, _stream()), symbol)


# ------------------------------------------------------------------------------------------------
# device guard: the library launches on the CURRENT device and on the stream passed in; every public wrapper that launches
# therefore runs with its tensors' device made current (a model on cuda:1 while cuda:0 is current, or one process driving
# two GPUs).
# ------------------------------------------------------------------------------------------------
def _device_of(x):
    if isinstance(x, torch.Tensor):
        return x.device if x.is_cuda else None
    if isinstance(x, (Act, SparseCanvas)):
        return x.device
    if isinstance(x, SparseTensor):
        return x.coords.device
    return None


def _first_device_arg(*args, **kwargs):
    """The first argument, positional then keyword, that carries a CUDA device."""
    for a in (*args, *kwargs.values()):
        if _device_of(a) is not None:
            return a
    return None


def _guard(fn=None, *, device_arg=_first_device_arg):
    """Decorator: run `fn` with the device of `device_arg(*args, **kwargs)` current (no device context when it already
    is).  The wrapper keeps `device_arg` as an attribute, which marks it as guarded."""
    if fn is None:
        return functools.partial(_guard, device_arg=device_arg)

    @functools.wraps(fn)
    def wrapped(*args, **kwargs):
        dev = _device_of(device_arg(*args, **kwargs))
        if dev is None or dev.index is None or dev.index == torch.cuda.current_device():
            return fn(*args, **kwargs)
        with torch.cuda.device(dev):
            return fn(*args, **kwargs)
    wrapped.device_arg = device_arg
    return wrapped


def _need_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise RuntimeError("heal_b200 ops need CUDA tensors (no CPU fallback in the product path)")


def _host_f32(vals: Sequence[float]):
    return (ctypes.c_float * len(vals))(*[float(np.float32(v)) for v in vals])


def _box_range_f32(gt_range: Sequence[float]):
    """The box range mask's [minx miny minz maxx maxy maxz] as fp32 limits that make the kernel's fp32 test exact.
    mask_boxes_outside_range_numpy compares fp32 corners with a float64 slice of the range (box_utils.py:415-416).  Each lower
    limit becomes the smallest fp32 >= it and each upper limit the largest fp32 <= it, so for any fp32 corner c,
    `c >= lo_f32` is `double(c) >= lo` and `c <= hi_f32` is `double(c) <= hi`.  (Rounding to nearest would keep a corner at
    float32(-25.6), which lies below -25.6.)"""
    out = []
    for k, v in enumerate(gt_range):
        v = float(v)
        f = np.float32(v)
        if k < 3 and float(f) < v:
            f = np.nextafter(f, np.float32(np.inf))
        elif k >= 3 and float(f) > v:
            f = np.nextafter(f, np.float32(-np.inf))
        out.append(float(f))
    assert len(out) == 6
    return (ctypes.c_float * 6)(*out)


def _host_i32(vals: Sequence[int]):
    return (ctypes.c_int * len(vals))(*[int(v) for v in vals])


_WS = {}

# bench.py instrumentation: when PROFILE is a list, every wrapper brackets its C-ABI call with CUDA events
# on the launching stream and appends (kernel family, algorithmic flops, start, end).
PROFILE = None


class _Prof:
    """`work` = algorithmic FLOPs, `nbytes` = algorithmic HBM bytes of the call (SURVEY.md 8d formulas); either may be a
    zero-argument callable that is evaluated after the instrumented pass has synchronised (data-dependent sizes)."""

    def __init__(self, name, work=0.0, nbytes=0.0):
        self.name, self.work, self.nbytes = name, work, nbytes

    def __enter__(self):
        if PROFILE is not None:
            self.a = torch.cuda.Event(enable_timing=True)
            self.b = torch.cuda.Event(enable_timing=True)
            self.l0 = lib.heal_launch_count()
            self.a.record()
        return self

    def __exit__(self, *exc):
        if PROFILE is not None:
            self.b.record()
            PROFILE.append((self.name, self.work, self.a, self.b, self.nbytes, int(lib.heal_launch_count() - self.l0)))
        return False


def _workspace(dev: torch.device, nbytes: int) -> torch.Tensor:
    """Scratch for one C-ABI call.  Eager calls share one growable buffer per (device, stream).  While a CUDA graph is being
    captured the buffer is a fresh allocation from the graph's private pool instead: a captured kernel's scratch pointer is
    baked into the graph, so it must never be the shared buffer that a later, larger eager call replaces and frees."""
    if torch.cuda.is_current_stream_capturing():
        return torch.empty(max(int(nbytes), 256), dtype=torch.uint8, device=dev)
    key = (dev.type, dev.index, torch.cuda.current_stream(dev).cuda_stream)
    ws = _WS.get(key)
    if ws is None or ws.numel() < nbytes:
        ws = torch.empty(max(int(nbytes), 1 << 20), dtype=torch.uint8, device=dev)
        _WS[key] = ws
    return ws


BPE = {"f32": 4, "bf16": 2, "split": 4}     # bytes per activation element by storage format


# ------------------------------------------------------------------------------------------------
# activations
# ------------------------------------------------------------------------------------------------
class Act:
    """Channels-last activation buffer.  fmt 'f32': t is (N,H,W,C) fp32; 'bf16'/'split': t is (P,N,H,W,C) bf16."""

    def __init__(self, t: torch.Tensor, fmt: str):
        _need_cuda(t)
        self.t, self.fmt = t, fmt
        if fmt == "f32":
            assert t.dtype == torch.float32 and t.dim() == 4
            n, h, w, c = t.shape
            sn, sh, sw, sc = t.stride()
            self.plane_stride = 0
        else:
            assert t.dtype == torch.bfloat16 and t.dim() == 5 and t.shape[0] == (2 if fmt == "split" else 1)
            _, n, h, w, c = t.shape
            sp, sn, sh, sw, sc = t.stride()
            self.plane_stride = sp
        assert sc == 1 and sh == w * sw and (n == 1 or sn == h * sh), "Act needs a channels-last dense pixel grid"
        self.N, self.H, self.W, self.C, self.cstride = n, h, w, c, sw

    @property
    def planes(self):
        return {"f32": 0, "bf16": 1, "split": 2}[self.fmt]

    @property
    def device(self):
        return self.t.device

    def view(self, coffset: int = 0) -> HealAct:
        return HealAct(self.t.data_ptr(), FMT[self.fmt], self.cstride, coffset, self.plane_stride)

    def images(self, a: int, b: int) -> "Act":
        return Act(self.t[a:b] if self.fmt == "f32" else self.t[:, a:b], self.fmt)

    def image(self, b: int) -> "Act":
        return self.images(b, b + 1)

    def rows(self, a: int, b: int) -> "Act":
        """Rows [a, b) of a single-image map as a zero-copy view (rows of a channels-last image are contiguous)."""
        assert self.N == 1 and 0 <= a < b <= self.H
        return Act(self.t[:, a:b] if self.fmt == "f32" else self.t[:, :, a:b], self.fmt)


def _act_new(new, N, H, W, C, fmt: str, device) -> Act:
    if fmt == "f32":
        return Act(new((N, H, W, C), dtype=torch.float32, device=device), fmt)
    return Act(new((2 if fmt == "split" else 1, N, H, W, C), dtype=torch.bfloat16, device=device), fmt)


def act_empty(N, H, W, C, fmt: str, device) -> Act:
    return _act_new(torch.empty, N, H, W, C, fmt, device)


def act_zeros(N, H, W, C, fmt: str, device) -> Act:
    """Zero-filled Act (all-zero bits are 0.0 in every storage format): a canvas the kernel writes at hit cells only."""
    return _act_new(torch.zeros, N, H, W, C, fmt, device)


def _out_act(out: Optional[Act], N, H, W, C, fmt: str, device) -> Act:
    """A wrapper's whole-tensor output: `out` when given (it must be (N,H,W,C)), else a new Act in `fmt`."""
    if out is None:
        return act_empty(N, H, W, C, fmt, device)
    assert (out.N, out.H, out.W, out.C) == (N, H, W, C)
    return out


def _theta64(theta: torch.Tensor, n: int) -> torch.Tensor:
    """(n,2,3) affine poses as the contiguous fp64 array the fusion kernels read."""
    th = theta.to(torch.float64).contiguous()
    assert th.shape == (n, 2, 3)
    return th


@_guard
def convert(a: Act, fmt: str, out: Optional[Act] = None) -> Act:
    """`a` in storage format `fmt`: `a` itself when it already is, unless `out` (a (N,H,W,C) Act in `fmt`, a channel view of a
    wider map is fine) is given to receive the copy."""
    if out is None and a.fmt == fmt:
        return a
    out = _out_act(out, a.N, a.H, a.W, a.C, fmt, a.device)
    assert out.fmt == fmt
    with _Prof("act_convert", 0, a.N * a.H * a.W * float(a.C) * (BPE[a.fmt] + BPE[fmt])):
        _call("heal_act_convert", a.view(), out.view(), a.N * a.H * a.W, a.C)
    return out


def _first_map(feats, *args, **kwargs):
    return next(iter(feats.values()), None)


@_guard(device_arg=_first_map)
def agent_stack(feats: dict, agent_modality_list: Sequence[str], crops: Optional[dict] = None, fmt: str = "f32",
                out: Optional[Act] = None) -> Act:
    """The (n_agents, H, W, C) map of a heterogeneous scene in scene order, one heal_agent_stack launch: agent i is the next
    image of `feats[agent_modality_list[i]]` (an Act per modality, any format).  `crops[m] = (th, tw)` center-crops or zero-pads
    modality m's maps as torchvision CenterCrop does (the camera modalities); every other modality's maps must already have
    the scene's size.  The result is in `fmt`: 'f32' is the hand-off the heterogeneous models' forwards use."""
    crops = crops or {}
    mods = list(dict.fromkeys(agent_modality_list))
    sizes = {m: tuple(crops[m]) if m in crops else (feats[m].H, feats[m].W) for m in mods}
    H, W = next((sizes[m] for m in mods if m not in crops), sizes[mods[0]])
    C = feats[mods[0]].C
    for m in mods:
        f = feats[m]
        if sizes[m] != (H, W) or f.C != C:
            raise ValueError(f"agent_stack: {m} gives {f.C}-channel {sizes[m][0]}x{sizes[m][1]} maps, the scene is "
                             f"{C}-channel {H}x{W}")
        if agent_modality_list.count(m) > f.N:
            raise ValueError(f"agent_stack: {agent_modality_list.count(m)} {m} agents, {f.N} {m} maps")
    from ._lib import HealStackSource
    srcs = (HealStackSource * len(mods))(*[HealStackSource(feats[m].view(), feats[m].N, feats[m].H, feats[m].W, int(m in crops))
                                           for m in mods])
    seen = {m: 0 for m in mods}
    src_of, img_of = [], []
    for m in agent_modality_list:
        src_of.append(mods.index(m))
        img_of.append(seen[m])
        seen[m] += 1
    n = len(agent_modality_list)
    out = _out_act(out, n, H, W, C, fmt, feats[mods[0]].device)
    assert out.fmt == fmt
    nbytes = sum(H * W * float(C) * (BPE[feats[m].fmt] + BPE[fmt]) for m in agent_modality_list)
    with _Prof("agent_stack", 0, nbytes):
        _call("heal_agent_stack", srcs, len(mods), _host_i32(src_of), _host_i32(img_of), n, C, out.view(), H, W)
    return out


def to_nhwc(x: torch.Tensor) -> torch.Tensor:
    """(N,C,H,W) logical tensor -> contiguous (N,H,W,C) buffer (view if already channels-last)."""
    assert x.dim() == 4
    xp = x.permute(0, 2, 3, 1)
    return xp if xp.is_contiguous() else xp.contiguous()


def from_nhwc(buf: torch.Tensor) -> torch.Tensor:
    """contiguous (N,H,W,C) buffer -> logical (N,C,H,W) view (channels-last strides)."""
    return buf.permute(0, 3, 1, 2)


def to_act(x: torch.Tensor) -> Act:
    """logical (N,C,H,W) fp32 tensor -> Act('f32')."""
    _need_cuda(x)
    return Act(to_nhwc(x.float()), "f32")


def act_to_nchw(a: Act) -> torch.Tensor:
    """Act -> logical (N,C,H,W) fp32 tensor (channels-last strides)."""
    return from_nhwc(convert(a, "f32").t)


def split_bf16(x: torch.Tensor, planes: int = 2) -> torch.Tensor:
    """fp32 (...) -> bf16 (planes, ...) with hi = bf16(x), lo = bf16(x - hi)  (host-side packing / test helper)."""
    hi = x.to(torch.bfloat16)
    if planes == 1:
        return hi.unsqueeze(0).contiguous()
    lo = (x - hi.float()).to(torch.bfloat16)
    return torch.stack([hi, lo]).contiguous()


def merge_bf16(s: torch.Tensor) -> torch.Tensor:
    return s.float().sum(0)


# ------------------------------------------------------------------------------------------------
# voxelization
# ------------------------------------------------------------------------------------------------
def grid_size_of(lidar_range, voxel_size):
    """round((max-min)/vs) as sp_voxel_preprocessor.py:41-43 does (fp64 numpy)."""
    g = (np.array(lidar_range[3:6]) - np.array(lidar_range[0:3])) / np.array(voxel_size)
    return np.round(g).astype(np.int64)


@_guard
def voxelize(points: torch.Tensor, agent_offsets: torch.Tensor, lidar_range, voxel_size,
             max_points_per_voxel: int, max_voxels: int, capacity: Optional[int] = None):
    """GPU SpVoxelPreprocessor.preprocess + collate for all agents of a scene.

    points (P,4) f32 cuda; agent_offsets (A+1) i32 cuda.  Returns (voxels (cap,T,4), coords (cap,4) i32
    [b,z,y,x], num_points (cap) i32, num_voxels (1+A) i32 device tensor).  Rows >= num_voxels[0] are
    undefined; use `trim_voxels` for the exact-size reference-shaped dict (one host sync)."""
    _need_cuda(points, agent_offsets)
    assert points.dtype == torch.float32 and points.dim() == 2 and points.shape[1] == 4 and points.is_contiguous()
    assert agent_offsets.dtype == torch.int32
    A = agent_offsets.numel() - 1
    P = points.shape[0]
    grid = grid_size_of(lidar_range, voxel_size)
    cap = int(capacity) if capacity is not None else max(1, min(P, A * max_voxels))
    dev = points.device
    T = int(max_points_per_voxel)
    voxels = torch.empty((cap, T, 4), dtype=torch.float32, device=dev)
    coords = torch.empty((cap, 4), dtype=torch.int32, device=dev)
    npts = torch.empty((cap,), dtype=torch.int32, device=dev)
    nvox = torch.zeros((1 + A,), dtype=torch.int32, device=dev)
    ws_bytes = lib.heal_voxelize_workspace(P, cap, A)
    ws = _workspace(dev, ws_bytes)
    with _Prof("voxelize", 0, lambda: 16.0 * P + float(nvox[0].item()) * (16 * T + 20)):
        _call("heal_voxelize", _p(points), _p(agent_offsets), A, P,
              _host_f32(lidar_range[0:3]), _host_f32(voxel_size), _host_i32(grid),
              T, int(max_voxels), cap, _p(voxels), _p(coords), _p(npts), _p(nvox), _p(ws), ws.numel())
    return voxels, coords, npts, nvox


@_guard
def mask_points(points: torch.Tensor, agent_offsets: torch.Tensor, lidar_range, remove_ego: bool = True,
                perm: Optional[torch.Tensor] = None):
    """shuffle_points (host-drawn `perm`, optional) -> mask_ego_points -> mask_points_by_range on the GPU (pcd_utils.py:41-95), a
    stable compaction per agent.  Returns (points_out (P,4) f32 [rows >= offsets_out[-1] undefined], offsets_out (A+1) i32 device)."""
    _need_cuda(points, agent_offsets)
    assert points.dtype == torch.float32 and points.dim() == 2 and points.shape[1] == 4 and points.is_contiguous()
    assert agent_offsets.dtype == torch.int32
    P, A = points.shape[0], agent_offsets.numel() - 1
    out = torch.empty_like(points)
    offs_out = torch.empty_like(agent_offsets)
    ws = _workspace(points.device, lib.heal_mask_points_workspace(P))
    pm = perm.to(torch.int32).contiguous() if perm is not None else None
    with _Prof("mask_points", 0, 32.0 * P):
        _call("heal_mask_points", _p(points), _p(pm), _p(agent_offsets), A, P, _host_f32(lidar_range), 1 if remove_ego else 0,
              _p(out), _p(offs_out), _p(ws), ws.numel())
    return out, offs_out


def raw_points_of(inp: dict, lidar_range):
    """(points, agent_offsets) of a raw-points `inputs_<m>` dict.  With `filter_points` set (GpuVoxelPreprocessor, `filter_on_gpu`),
    the clouds are still unfiltered and the reference's host filters run here first (mask_points); otherwise as given."""
    pts, offs = inp['points'], inp['agent_offsets']
    if inp.get('filter_points'):
        pts, offs = mask_points(pts, offs, lidar_range, bool(inp.get('remove_ego', True)), inp.get('shuffle_perm'))
    return pts, offs


def trim_voxels(voxels, coords, npts, nvox):
    m = int(nvox[0].item())
    return {"voxel_features": voxels[:m], "voxel_coords": coords[:m], "voxel_num_points": npts[:m]}


@_guard
def mean_vfe(voxels: torch.Tensor, num_points: torch.Tensor) -> torch.Tensor:
    _need_cuda(voxels, num_points)
    M, T, C = voxels.shape
    assert C == 4 and voxels.dtype == torch.float32 and voxels.is_contiguous()
    npts = num_points.to(torch.int32).contiguous()
    out = torch.empty((M, 4), dtype=torch.float32, device=voxels.device)
    with _Prof("mean_vfe", 0, M * (T * 16.0 + 4 + 16)):
        _call("heal_mean_vfe", _p(voxels), _p(npts), M, T, _p(out))
    return out


# ------------------------------------------------------------------------------------------------
# PillarVFE + scatter
# ------------------------------------------------------------------------------------------------
def fold_linear_bn(weight: torch.Tensor, bn_w, bn_b, bn_mean, bn_var, eps: float):
    """Linear(no bias) followed by eval BatchNorm1d -> (W' (Cin,Cout) fp32, b' (Cout) fp32), folded in fp64."""
    w = weight.detach().double().cpu()                      # (Cout, Cin)
    scale = bn_w.detach().double().cpu() / torch.sqrt(bn_var.detach().double().cpu() + eps)
    shift = bn_b.detach().double().cpu() - bn_mean.detach().double().cpu() * scale
    wf = (w * scale[:, None]).t().contiguous()              # (Cin, Cout)
    return wf.float(), shift.float()


@_guard
def pillar_vfe_scatter(voxel_features, voxel_num_points, voxel_coords, w_folded, b_folded,
                       voxel_size, lidar_range, nx: int, ny: int, batch_size: int,
                       want_pillar_features: bool = False, want_canvas: bool = True,
                       num_voxels_dev: Optional[torch.Tensor] = None, canvas_fmt: str = "f32", split_rows_out: Optional[torch.Tensor] = None):
    """Returns (pillar_features (M,64) | None, canvas Act (B,ny,nx,64) in `canvas_fmt` | None).  `split_rows_out`: optional
    (M,128) bf16 buffer that receives the pillar features as split rows [hi | lo] (tensor-core sparse stem input)."""
    _need_cuda(voxel_features, voxel_num_points, voxel_coords, w_folded, b_folded)
    M, T, C = voxel_features.shape
    assert C == 4
    dev = voxel_features.device
    vf = voxel_features.contiguous().float()
    npts = voxel_num_points.to(torch.int32).contiguous()
    coords = voxel_coords.to(torch.int32).contiguous()
    cout = w_folded.shape[1]
    pf = torch.empty((M, cout), dtype=torch.float32, device=dev) if want_pillar_features else None
    vs = [float(v) for v in voxel_size]
    off = [vs[i] / 2 + float(lidar_range[i]) for i in range(3)]
    def _bytes():
        m = float(num_voxels_dev[0].item()) if num_voxels_dev is not None else float(M)
        b = m * (T * 16 + 20)                                   # voxel slots + count + coords (SURVEY 8d)
        if want_pillar_features:
            b += m * cout * 4
        if want_canvas:
            b += float(batch_size) * ny * nx * cout * BPE[canvas_fmt]
        return b
    with _Prof("pillar_vfe_scatter" + ("(+canvas memset)" if want_canvas else ""), lambda: 2.0 * T * w_folded.shape[0] * cout *
               (float(num_voxels_dev[0].item()) if num_voxels_dev is not None else float(M)), _bytes):
        canvas = act_zeros(batch_size, ny, nx, cout, canvas_fmt, dev) if want_canvas else None
        _call("heal_pillar_vfe_scatter", _p(vf), _p(npts), _p(coords), _p(num_voxels_dev), M, T,
              _p(w_folded), _p(b_folded), w_folded.shape[0], cout, _host_f32(vs), _host_f32(off), int(nx), int(ny),
              _p(pf), _p(split_rows_out), canvas.view() if canvas is not None else None)
    return pf, canvas


@_guard
def pillar_scatter(pillar_features: torch.Tensor, voxel_coords: torch.Tensor, nx: int, ny: int, batch_size: int,
                   fmt: str = "f32", num_voxels_dev: Optional[torch.Tensor] = None) -> Act:
    """Stand-alone PointPillarScatter: (M,C) f32 rows -> Act (B,ny,nx,C) (zero elsewhere)."""
    _need_cuda(pillar_features, voxel_coords)
    M, C = pillar_features.shape
    coords = voxel_coords.to(torch.int32).contiguous()
    with _Prof("pillar_scatter(+canvas memset)", 0, M * (C * 4.0 + 16) + batch_size * float(ny) * nx * C * BPE[fmt]):
        canvas = act_zeros(batch_size, ny, nx, C, fmt, coords.device)
        _call("heal_pillar_scatter", _p(pillar_features), _p(coords), _p(num_voxels_dev), M, C, int(nx), int(ny), canvas.view())
    return canvas


# ------------------------------------------------------------------------------------------------
# conv2d: parameter folding / packing
# ------------------------------------------------------------------------------------------------
def _bn_scale_shift(bn, cout):
    if bn is None:
        return torch.ones(cout, dtype=torch.float64), torch.zeros(cout, dtype=torch.float64)
    scale = bn.weight.detach().double().cpu() / torch.sqrt(bn.running_var.detach().double().cpu() + bn.eps)
    shift = bn.bias.detach().double().cpu() - bn.running_mean.detach().double().cpu() * scale
    return scale, shift


class PackedConv:
    """Folded + packed parameters of one Conv2d(+BN)(+ReLU) for heal_conv2d_simt (fp32 CUDA-core path)."""

    def __init__(self, weight, bias, kh, kw, stride, pad, groups, cin, cout, relu, w_cstride, deconv_up=1):
        self.weight, self.bias = weight, bias
        self.kh, self.kw, self.stride, self.pad, self.groups = kh, kw, stride, pad, groups
        self.cin, self.cout, self.relu, self.w_cstride, self.deconv_up = cin, cout, relu, w_cstride, deconv_up

    def to(self, device):
        self.weight = self.weight.to(device)
        self.bias = self.bias.to(device) if self.bias is not None else None
        return self


def pack_conv(conv: torch.nn.Conv2d, bn: Optional[torch.nn.Module], relu: bool, extra_pad: int = 0,
              cin_to: Optional[int] = None) -> PackedConv:
    """Fold eval-mode BN into the conv (fp64 on the host) and pack for heal_conv2d_simt.  `cin_to` (groups 1): zero weights for
    input channels [Cin, cin_to), for an input whose channel count is padded to the multiple of 4 the kernel reads."""
    w = conv.weight.detach().double().cpu()            # (Cout, Cin/g, kh, kw)
    cout, cing, kh, kw = w.shape
    g = conv.groups
    if cin_to is not None and cin_to > cing:
        assert g == 1
        w = torch.cat([w, w.new_zeros((cout, cin_to - cing, kh, kw))], 1)
        cing = cin_to
    scale, shift = _bn_scale_shift(bn, cout)
    b = shift.clone()
    if conv.bias is not None:
        b = b + conv.bias.detach().double().cpu() * scale
    w = w * scale[:, None, None, None]
    assert conv.stride[0] == conv.stride[1] and conv.padding[0] == conv.padding[1] and conv.dilation == (1, 1)
    pad = conv.padding[0] + extra_pad
    if g == 1:
        cpad = (cout + 3) // 4 * 4
        wp = torch.zeros((kh, kw, cing, cpad), dtype=torch.float64)
        wp[..., :cout] = w.permute(2, 3, 1, 0)
        return PackedConv(wp.float().contiguous(), b.float().contiguous(), kh, kw, conv.stride[0], pad, 1,
                          cing, cout, relu, cpad)
    cg = cout // g
    assert cing == cg and kh == 3 and kw == 3
    wg = w.view(g, cg, cg, kh * kw)                     # (G, co, ci, tap)
    wp = wg.permute(3, 2, 1, 0).contiguous()            # (tap, ci, co, G)
    return PackedConv(wp.float(), b.float().contiguous(), kh, kw, conv.stride[0], pad, g, cing * g, cout, relu, 0)


def pack_deconv(deconv: torch.nn.ConvTranspose2d, bn, relu: bool) -> PackedConv:
    """ConvTranspose2d with kernel == stride (no overlap) -> up*up 1x1 weight planes [i][j][Cin][Cout]."""
    w = deconv.weight.detach().double().cpu()          # (Cin, Cout, k, k)
    cin, cout, k, k2 = w.shape
    assert k == k2 == deconv.stride[0] == deconv.stride[1] and deconv.padding == (0, 0) and deconv.groups == 1
    scale, shift = _bn_scale_shift(bn, cout)
    b = shift.clone()
    if deconv.bias is not None:
        b = b + deconv.bias.detach().double().cpu() * scale
    w = w * scale[None, :, None, None]
    cpad = (cout + 3) // 4 * 4
    wp = torch.zeros((k, k, cin, cpad), dtype=torch.float64)
    wp[..., :cout] = w.permute(2, 3, 0, 1)
    return PackedConv(wp.float().contiguous(), b.float().contiguous(), 1, 1, 1, 0, 1, cin, cout, relu, cpad, deconv_up=k)


def _coutp(cout: int) -> int:
    for c in (16, 32, 64):
        if cout <= c:
            return c
    return (cout + 127) // 128 * 128


class PackedConvTC:
    """Folded + packed split-bf16 parameters for heal_conv2d_tc (wgmma path)."""

    def __init__(self, w, bias, kh, kw, pad, cin, cout, coutp, relu, up, planes, stride=1, blockdiag=False, groups=1):
        self.w, self.bias = w, bias
        self.kh, self.kw, self.pad, self.cin, self.cout, self.coutp = kh, kw, pad, cin, cout, coutp
        self.relu, self.up, self.planes = relu, up, planes
        self.stride, self.groups, self.blockdiag = stride, groups, blockdiag
        self.w_diag = None       # grouped convs: [plane][tap][co][16] diagonal sub-blocks (what the kernel streams)

    def to(self, device):
        self.w = self.w.to(device)
        self.bias = self.bias.to(device)
        if self.w_diag is not None:
            self.w_diag = self.w_diag.to(device)
        return self


TC_STRIDED = True      # stride-2 convs through TMA element strides
TC_GROUPED = True      # grouped 3x3 convs as block-diagonal 64-channel blocks on the tensor cores


def tc_eligible(conv) -> bool:
    if isinstance(conv, torch.nn.ConvTranspose2d):
        return conv.in_channels % 64 == 0 and conv.groups == 1
    if conv.in_channels % 64 or conv.dilation != (1, 1) or conv.stride[0] != conv.stride[1]:
        return False
    if conv.stride[0] not in ((1, 2) if TC_STRIDED else (1,)):
        return False
    if conv.groups == 1:
        return True
    cg = conv.in_channels // conv.groups
    return TC_GROUPED and conv.in_channels == conv.out_channels and conv.kernel_size == (3, 3) and 16 % cg == 0


def pack_conv_tc(conv, bn, relu: bool, planes: int = 2, extra_pad: int = 0, cin_to: Optional[int] = None) -> PackedConvTC:
    """Fold BN (fp64), lay weights out as [plane][tap*coutp + co][Cin] (split-)bf16 for heal_conv2d_tc.  `cin_to` (dense convs):
    zero weights for input channels [Cin, cin_to), for an input zero-padded to a multiple of 64 channels."""
    if isinstance(conv, torch.nn.ConvTranspose2d):
        w = conv.weight.detach().double().cpu()            # (Cin, Cout, k, k)
        cin, cout, k, _ = w.shape
        scale, shift = _bn_scale_shift(bn, cout)
        b = shift + (conv.bias.detach().double().cpu() * scale if conv.bias is not None else 0)
        w = w * scale[None, :, None, None]
        coutp = _coutp(cout)
        rows = torch.zeros((k * k, coutp, cin), dtype=torch.float64)
        rows[:, :cout, :] = w.permute(2, 3, 1, 0).reshape(k * k, cout, cin)
        wp = split_bf16(rows.reshape(k * k * coutp, cin).float(), planes)
        return PackedConvTC(wp, b.float().contiguous(), 1, 1, 0, cin, cout, coutp, relu, k, planes)
    w = conv.weight.detach().double().cpu()                # (Cout, Cin/g, kh, kw)
    cout, cin, kh, kw = w.shape
    scale, shift = _bn_scale_shift(bn, cout)
    b = shift + (conv.bias.detach().double().cpu() * scale if conv.bias is not None else 0)
    w = w * scale[:, None, None, None]
    if conv.groups > 1:
        # block-diagonal: row = tap*width + co, column = input channel inside co's 64-channel block
        g, width, cg = conv.groups, cout, cin
        assert width % 64 == 0 and 16 % cg == 0 and conv.in_channels == width
        rows = torch.zeros((kh * kw, width, 64), dtype=torch.float64)
        co = torch.arange(width)
        col0 = (co // cg) * cg - (co // 64) * 64                     # first input channel of co's group, block-local
        wt = w.permute(2, 3, 0, 1).reshape(kh * kw, width, cg)        # (tap, co, ci)
        for ci in range(cg):
            rows[:, co, col0 + ci] = wt[:, :, ci]
        wp = split_bf16(rows.reshape(kh * kw * width, 64).float(), planes)
        pc = PackedConvTC(wp, b.float().contiguous(), kh, kw, conv.padding[0] + extra_pad, width, width, width, relu, 1,
                          planes, stride=conv.stride[0], blockdiag=True, groups=g)
        # diagonal 16x16 sub-blocks only: column = input channel inside co's 16-channel sub-block
        diag = torch.zeros((kh * kw, width, 16), dtype=torch.float64)
        c16 = (co // cg) * cg - (co // 16) * 16
        for ci in range(cg):
            diag[:, co, c16 + ci] = wt[:, :, ci]
        pc.w_diag = split_bf16(diag.reshape(kh * kw * width, 16).float(), planes)
        return pc
    coutp = _coutp(cout)
    cin_w = cin
    if cin_to is not None and cin_to > cin:
        cin = cin_to
    rows = torch.zeros((kh * kw, coutp, cin), dtype=torch.float64)
    rows[:, :cout, :cin_w] = w.permute(2, 3, 0, 1).reshape(kh * kw, cout, cin_w)
    wp = split_bf16(rows.reshape(kh * kw * coutp, cin).float(), planes)
    return PackedConvTC(wp, b.float().contiguous(), kh, kw, conv.padding[0] + extra_pad, cin, cout, coutp, relu, 1, planes,
                        stride=conv.stride[0])


class PackedConvNarrow:
    """Folded + packed parameters of one 3x3 Conv2d(+BN)(+ReLU) with a narrow input for heal_conv3x3_narrow_tc."""

    def __init__(self, w, bias, cin, cout, relu):
        self.w, self.bias, self.cin, self.cout, self.relu = w, bias, cin, cout, relu

    def to(self, device):
        self.w = self.w.to(device)
        self.bias = self.bias.to(device)
        return self


def narrow_eligible(conv) -> bool:
    """A conv heal_conv3x3_narrow_tc takes: 3x3, stride 1, pad 1, groups 1, 1 <= Cin <= 63, Cout a multiple of 16 up to 256."""
    return (isinstance(conv, torch.nn.Conv2d) and conv.kernel_size == (3, 3) and conv.stride == (1, 1)
            and conv.padding == (1, 1) and conv.dilation == (1, 1) and conv.groups == 1 and 1 <= conv.in_channels <= 63
            and conv.out_channels % 16 == 0 and conv.out_channels <= 256)


def pack_conv3x3_narrow(conv, bn, relu: bool) -> PackedConvNarrow:
    """Fold BN (fp64) and lay the weights out as heal_conv3x3_narrow_tc reads them: K = (tap, channel) with the channel count
    rounded up to even, padded to a multiple of 16; per 64-channel output block and 64-wide K block [hi 64 rows | lo 64 rows]."""
    assert narrow_eligible(conv)
    w = conv.weight.detach().double().cpu()                # (Cout, Cin, 3, 3)
    cout, cin = w.shape[:2]
    scale, shift = _bn_scale_shift(bn, cout)
    b = shift + (conv.bias.detach().double().cpu() * scale if conv.bias is not None else 0)
    w = w * scale[:, None, None, None]
    cinp = cin + (cin & 1)
    k = (9 * cinp + 15) // 16 * 16
    kb, nblk = (k + 63) // 64, (cout + 63) // 64
    rows = torch.zeros((nblk * 64, 9, cinp), dtype=torch.float64)
    rows[:cout, :, :cin] = w.permute(0, 2, 3, 1).reshape(cout, 9, cin)
    mat = torch.zeros((nblk * 64, kb * 64), dtype=torch.float32)
    mat[:, :9 * cinp] = rows.reshape(nblk * 64, 9 * cinp).float()
    hi, lo = split_bf16(mat, 2)                            # (nblk*64, kb*64) each
    wp = torch.stack([hi.view(nblk, 64, kb, 64), lo.view(nblk, 64, kb, 64)], 2)   # (nblk, 64 rows, plane, kb, 64)
    wp = wp.permute(0, 3, 2, 1, 4).contiguous()            # (nblk, kb, plane, 64 rows, 64)
    return PackedConvNarrow(wp, b.float().contiguous(), cin, cout, relu)


# ------------------------------------------------------------------------------------------------
# conv2d launchers
# ------------------------------------------------------------------------------------------------
@_guard
def conv2d_simt(x: Act, pc: PackedConv, residual: Optional[Act] = None, out: Optional[Act] = None,
                out_fmt: str = "f32", out_coffset: int = 0, in_coffset: int = 0, cin: Optional[int] = None) -> Act:
    """fp32 CUDA-core conv; any storage format in/out."""
    _need_cuda(pc.weight)
    N, H, W = x.N, x.H, x.W
    cin = pc.cin if cin is None else cin
    assert cin + in_coffset <= x.C
    up = pc.deconv_up
    Ho = (H + 2 * pc.pad - pc.kh) // pc.stride + 1
    Wo = (W + 2 * pc.pad - pc.kw) // pc.stride + 1
    if out is None:
        out = act_empty(N, Ho * up, Wo * up, pc.cout, out_fmt, x.device)
    assert out.N == N and out.H == Ho * up and out.W == Wo * up
    if residual is not None:
        assert (residual.N, residual.H, residual.W) == (out.N, out.H, out.W)
    xv, ov = x.view(in_coffset), out.view(out_coffset)
    rv = residual.view() if residual is not None else None
    fam = ("conv_grouped3x3_simt" if pc.groups > 1 else f"conv_dense{pc.kh}x{pc.kw}_simt")
    flops = 2.0 * N * Ho * Wo * pc.cout * (cin // pc.groups) * pc.kh * pc.kw * up * up
    nbytes = N * H * W * cin * BPE[x.fmt] + N * out.H * out.W * pc.cout * BPE[out.fmt] + pc.weight.numel() * 4.0 \
        + (N * out.H * out.W * pc.cout * BPE[residual.fmt] if residual is not None else 0)
    with _Prof(fam, flops, nbytes):
        for i in range(up):
            for j in range(up):
                wptr = pc.weight if up == 1 else pc.weight[i, j]
                _call("heal_conv2d_simt", xv, N, H, W, cin, _p(wptr), pc.w_cstride, _p(pc.bias), pc.kh, pc.kw, pc.stride,
                      pc.pad, pc.groups, rv, ov, Ho, Wo, pc.cout, up, i, j, int(pc.relu))
    return out


@_guard
def conv2d_tc(x: Act, pc: PackedConvTC, residual: Optional[Act] = None, out: Optional[Act] = None,
              out_coffset: int = 0, in_coffset: int = 0, want_split: bool = True,
              out_f32: Optional[Act] = None, want_f32: bool = False, out32_coffset: int = 0):
    """wgmma conv.  x: Act 'split' (planes 2) or 'bf16' (planes 1).  Returns (Act split/bf16 | None, Act f32 | None)."""
    _need_cuda(pc.w)
    assert x.planes in (1, 2) and pc.planes >= x.planes      # weights may carry a lo plane the activations do not ('bf16' mode)
    N, H, W = x.N, x.H, x.W
    up = pc.up
    Ho, Wo = (H + 2 * pc.pad - pc.kh) // pc.stride + 1, (W + 2 * pc.pad - pc.kw) // pc.stride + 1
    if want_split and out is None:
        out = act_empty(N, Ho * up, Wo * up, pc.cout, x.fmt, x.device)
    if want_f32 and out_f32 is None:
        out_f32 = act_empty(N, Ho * up, Wo * up, pc.cout, "f32", x.device)
    res_split = res_f32 = None
    res_cs = res_plane = 0
    if residual is not None:
        if residual.fmt == "f32":
            res_f32, res_cs = residual.t, residual.cstride
        else:
            assert residual.planes == x.planes
            res_split, res_cs, res_plane = residual.t, residual.cstride, residual.plane_stride
    fam = f"conv_tc{pc.kh}x{pc.kw}" + ("_deconv" if up > 1 else "") + ("_grouped" if pc.blockdiag else "") + (f"_s{pc.stride}" if pc.stride > 1 else "")
    flops = 2.0 * N * Ho * Wo * pc.cout * (pc.cin // pc.groups) * pc.kh * pc.kw * up * up
    epb = 2.0 * x.planes
    nbytes = N * H * W * pc.cin * epb + (pc.w_diag if pc.w_diag is not None else pc.w).numel() * 2.0 \
        + (N * Ho * Wo * up * up * pc.cout * epb if out is not None else 0) \
        + (N * Ho * Wo * up * up * pc.cout * 4.0 if out_f32 is not None else 0) \
        + (N * Ho * Wo * up * up * pc.cout * BPE[residual.fmt] if residual is not None else 0)
    with _Prof(fam, flops, nbytes):
        _call("heal_conv2d_tc", _p(x.t), x.plane_stride, N, H, W, pc.cin, x.cstride, in_coffset,
              _p(pc.w), _p(pc.w_diag), pc.w.shape[1], pc.coutp, _p(pc.bias), pc.kh, pc.kw, pc.stride, pc.pad,
              1 if pc.blockdiag else 0, x.planes, pc.planes,
              _p(res_split), res_plane, _p(res_f32), res_cs, 0,
              _p(out.t) if out is not None else _vp(0), out.plane_stride if out is not None else 0,
              out.cstride if out is not None else 0, out_coffset,
              _p(out_f32.t) if out_f32 is not None else _vp(0),
              out_f32.cstride if out_f32 is not None else 0, out32_coffset,
              Ho, Wo, pc.cout, up, int(pc.relu))
    return out, out_f32


@_guard
def conv3x3_narrow_tc(x: Act, pc: PackedConvNarrow, planes: int, out: Optional[Act] = None, out_fmt: str = "split") -> Act:
    """wgmma 3x3 conv of a narrow input (Cin < 64).  x: any storage format, may be a channel slice of a wider map.  planes 2:
    split-bf16 products ('tc32'), 1: bf16 activations x split weights ('bf16').  `out` (optional): (N,H,W,Cout) Act."""
    _need_cuda(pc.w)
    assert x.C == pc.cin and planes in (1, 2)
    N, H, W = x.N, x.H, x.W
    out = _out_act(out, N, H, W, pc.cout, out_fmt, x.device)
    flops = 2.0 * N * H * W * pc.cout * pc.cin * 9
    nbytes = N * H * W * (pc.cin * BPE[x.fmt] + pc.cout * BPE[out.fmt]) + pc.w.numel() * 2.0
    with _Prof("conv_tc3x3_narrow", flops, nbytes):
        _call("heal_conv3x3_narrow_tc", x.view(), N, H, W, pc.cin, _p(pc.w), _p(pc.bias), pc.cout, planes, int(pc.relu),
              out.view())
    return out


@_guard
def bottleneck_tc(x: Act, pc1: PackedConvTC, pc2: PackedConvTC, pc3: PackedConvTC, out: Optional[Act] = None,
                  out_coffset: int = 0) -> Act:
    """ResNeXt bottleneck ReLU(conv3(conv2(conv1(x))) + x) in one kernel (64 -> 128 -> 64 channels, grouped 3x3, stride 1):
    bit-identical to conv2d_tc(pc1) -> conv2d_tc(pc2) -> conv2d_tc(pc3, residual=x).  x: Act 'split' or 'bf16'; the packed
    weights carry both planes.  `out` (optional, x's format): written at channels [out_coffset, out_coffset + 64)."""
    _need_cuda(pc1.w, pc2.w_diag, pc3.w)
    assert x.planes in (1, 2) and pc1.planes == pc2.planes == pc3.planes == 2
    assert (pc1.kh, pc1.cin, pc1.cout, pc3.kh, pc3.cin, pc3.cout) == (1, x.C, 2 * x.C, 1, 2 * x.C, x.C)
    assert pc2.blockdiag and pc2.kh == 3 and pc2.stride == 1 and pc2.cin == 2 * x.C
    N, H, W, C = x.N, x.H, x.W, x.C
    if out is None:
        out = act_empty(N, H, W, C, x.fmt, x.device)
    assert out.fmt == x.fmt and (out.N, out.H, out.W) == (N, H, W) and out_coffset + C <= out.C
    flops = 2.0 * N * H * W * (C * 2 * C + 2 * C * (2 * C // pc2.groups) * 9 + 2 * C * C)
    epb = 2.0 * x.planes
    nbytes = 2.0 * N * H * W * C * epb + 2.0 * (pc1.w.numel() + pc2.w_diag.numel() + pc3.w.numel())
    with _Prof("conv_tc_bottleneck", flops, nbytes):
        _call("heal_bottleneck_tc", _p(x.t), x.plane_stride, N, H, W, C, x.cstride,
              _p(pc1.w), _p(pc1.bias), _p(pc2.w_diag), _p(pc2.bias), _p(pc3.w), _p(pc3.bias),
              x.planes, pc1.planes, _p(out.t), out.plane_stride, out.cstride, out_coffset)
    return out


@_guard
def gconv_reduce_tc(mid: Act, pc2: PackedConvTC, pc3: PackedConvTC, residual: Act, out: Optional[Act] = None,
                    out_coffset: int = 0) -> Act:
    """ReLU(conv3(conv2(mid)) + residual) of a stride-1 ResNeXt bottleneck (grouped 3x3 width -> width, 1x1 width -> C) in one
    kernel: bit-identical to conv2d_tc(pc2) -> conv2d_tc(pc3, residual=residual).  mid, residual: Acts 'split' or 'bf16' of the
    same format; the packed weights carry both planes.  `out` (optional, that format): written at channels
    [out_coffset, out_coffset + C)."""
    _need_cuda(pc2.w_diag, pc3.w)
    assert mid.planes in (1, 2) and residual.fmt == mid.fmt and pc2.planes == pc3.planes == 2
    assert pc2.blockdiag and pc2.kh == 3 and pc2.stride == 1 and pc2.cin == pc2.cout == mid.C
    assert (pc3.kh, pc3.cin, pc3.cout, pc3.coutp) == (1, mid.C, residual.C, residual.C)
    N, H, W, C, width = mid.N, mid.H, mid.W, residual.C, mid.C
    assert (residual.N, residual.H, residual.W) == (N, H, W)
    if out is None:
        out = act_empty(N, H, W, C, mid.fmt, mid.device)
    assert out.fmt == mid.fmt and (out.N, out.H, out.W) == (N, H, W) and out_coffset + C <= out.C
    flops = 2.0 * N * H * W * (width * (width // pc2.groups) * 9 + width * C)
    epb = 2.0 * mid.planes
    nbytes = N * H * W * (width + 2.0 * C) * epb + 2.0 * (pc2.w_diag.numel() + pc3.w.numel())
    with _Prof("conv_tc_gconv_reduce", flops, nbytes):
        _call("heal_gconv_reduce_tc", _p(mid.t), mid.plane_stride, N, H, W, width, mid.cstride,
              _p(pc2.w_diag), _p(pc2.bias), _p(pc3.w), _p(pc3.bias), C,
              _p(residual.t), residual.plane_stride, residual.cstride, mid.planes, pc3.planes,
              _p(out.t), out.plane_stride, out.cstride, out_coffset)
    return out


# ------------------------------------------------------------------------------------------------
# ConvNeXt aligner front half, ResNet-stem max pooling
# ------------------------------------------------------------------------------------------------
@_guard
def dwconv_layernorm(x: Act, dw_weight: torch.Tensor, dw_bias, ksize: int, ln_weight, ln_bias, eps: float,
                     out_fmt: Optional[str] = None) -> Act:
    """depthwise ksize x ksize conv (+bias) + LayerNorm over channels.  dw_weight (ksize*ksize, C) fp32 tap-major."""
    _need_cuda(dw_weight, ln_weight, ln_bias)
    N, H, W, C = x.N, x.H, x.W, x.C
    assert dw_weight.shape == (ksize * ksize, C) and dw_weight.is_contiguous()
    out = act_empty(N, H, W, C, out_fmt or x.fmt, x.device)
    lw, lb = ln_weight.float().contiguous(), ln_bias.float().contiguous()
    with _Prof("dwconv_layernorm", 2.0 * N * H * W * C * ksize * ksize, N * H * W * float(C) * (BPE[x.fmt] + BPE[out.fmt])):
        _call("heal_dwconv_layernorm", x.view(), N, H, W, C, _p(dw_weight), _p(dw_bias), int(ksize), _p(lw), _p(lb),
              float(eps), out.view())
    return out


@_guard
def maxpool3x3s2(x: Act, out_fmt: Optional[str] = None, depth_to_space_in: bool = False) -> Act:
    """3x3 / stride 2 / pad 1 max pooling (torchvision ResNet stem).  depth_to_space_in: x is (N,H/2,W/2,4C) phase-major
    (channel block (y&1)*2+(x&1)) and stands for the logical (N,H,W,C) map."""
    N, H, W, C = x.N, x.H, x.W, x.C
    if depth_to_space_in:
        H, W, C = 2 * H, 2 * W, C // 4
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    out = act_empty(N, Ho, Wo, C, out_fmt or x.fmt, x.device)
    with _Prof("maxpool3x3s2", 0, N * float(C) * (H * W * BPE[x.fmt] + Ho * Wo * BPE[out.fmt])):
        _call("heal_maxpool3x3s2", x.view(), N, H, W, C, 1 if depth_to_space_in else 0, out.view())
    return out


# ------------------------------------------------------------------------------------------------
# fusion
# ------------------------------------------------------------------------------------------------
@_guard
def pyramid_fuse_level(feat: Act, occ: torch.Tensor, theta: torch.Tensor, align_corners: bool,
                       crop_windows: Optional[torch.Tensor] = None, out: Optional[Act] = None,
                       out_fmt: Optional[str] = None, out_coffset: int = 0,
                       agent_offsets=None, n_agents: Optional[int] = None, rows=None) -> Act:
    """feat: Act (n,H,W,C); occ (n,H,W) f32 logits; theta (n,2,3) f64 -> out Act (1,H,W,C) (one scene).
    agent_offsets = (feat element offsets, occ float offsets) per agent when the maps are NOT a dense stack (they live inside
    an all-gathered buffer: `feat` then describes ONE agent's map geometry at the buffer base and `n_agents` gives n);
    rows = (row0, nrows): produce only that slab of output rows (out is then (1,nrows,W,C))."""
    _need_cuda(occ, theta)
    n, H, W, C = (feat.N if n_agents is None else n_agents), feat.H, feat.W, feat.C
    assert occ.dtype == torch.float32
    if agent_offsets is None:
        assert occ.is_contiguous() and occ.numel() == n * H * W
    th = _theta64(theta, n)
    row0, nrows = rows if rows is not None else (0, H)
    if out is None:
        out = act_empty(1, nrows, W, C, out_fmt or feat.fmt, feat.device)
    assert out.H == nrows and out.W == W
    cw = crop_windows.to(torch.int32).contiguous() if crop_windows is not None else None
    fo = oo = None
    if agent_offsets is not None:
        fo = (ctypes.c_longlong * n)(*[int(v) for v in agent_offsets[0]])
        oo = (ctypes.c_longlong * n)(*[int(v) for v in agent_offsets[1]])
    with _Prof("pyramid_fuse_level", 0, (n * (C * BPE[feat.fmt] + 4.0) + C * BPE[out.fmt]) * float(nrows) * W):
        _call("heal_pyramid_fuse_level", feat.view(), _p(occ), _p(th), _p(cw), n, H, W, C,
              1 if align_corners else 0, fo, oo, int(row0), int(nrows), out.view(out_coffset))
    return out


@_guard
def att_fuse(feat: Act, theta: torch.Tensor, out: Optional[Act] = None, out_fmt: Optional[str] = None) -> Act:
    """feat: Act (n,H,W,C), theta (n,2,3) f64 -> Act (1,H,W,C)."""
    _need_cuda(theta)
    n, H, W, C = feat.N, feat.H, feat.W, feat.C
    th = _theta64(theta, n)
    out = _out_act(out, 1, H, W, C, out_fmt or feat.fmt, feat.device)
    with _Prof("att_fuse", 4.0 * n * C * H * W, (n * BPE[feat.fmt] + BPE[out.fmt]) * float(C) * H * W):
        _call("heal_att_fuse", feat.view(), _p(th), n, H, W, C, out.view())
    return out


@_guard
def max_fuse(feat: Act, theta: torch.Tensor, out: Optional[Act] = None, out_fmt: Optional[str] = None) -> Act:
    """MaxFusion of one scene: feat Act (n,H,W,C), theta (n,2,3) f64 -> Act (1,H,W,C) = max_j warp(feat_j, theta_j)."""
    _need_cuda(theta)
    n, H, W, C = feat.N, feat.H, feat.W, feat.C
    th = _theta64(theta, n)
    out = _out_act(out, 1, H, W, C, out_fmt or feat.fmt, feat.device)
    with _Prof("max_fuse", 4.0 * n * C * H * W, (n * BPE[feat.fmt] + BPE[out.fmt]) * float(C) * H * W):
        _call("heal_max_fuse", feat.view(), _p(th), n, H, W, C, out.view())
    return out


@_guard
def warp_affine(src: Act, src_index: Sequence[int], theta: torch.Tensor, out: Optional[Act] = None,
                out_fmt: Optional[str] = None) -> Act:
    """Batched warp_affine_simple (bilinear, zeros, align_corners=False): out image k = warp(src image src_index[k], theta[k]).
    src Act (n,H,W,C); theta (K,2,3) f64 on the device; `src_index` a host sequence of K image indices -> Act (K,H,W,C)."""
    _need_cuda(theta)
    K, H, W, C = len(src_index), src.H, src.W, src.C
    th = _theta64(theta, K)
    assert all(0 <= int(s) < src.N for s in src_index)
    out = _out_act(out, K, H, W, C, out_fmt or src.fmt, src.device)
    with _Prof("warp_affine", 8.0 * K * C * H * W, K * (BPE[src.fmt] + BPE[out.fmt]) * float(C) * H * W):
        _call("heal_warp_affine", src.view(), _host_i32(src_index), _p(th), K, H, W, C, out.view())
    return out


@_guard
def v2v_aggregate(q: Act, p_node: Act, x: Act, theta: torch.Tensor, nodes: Sequence[Sequence[int]], agg_max: bool,
                  gru: bool, out: Optional[Act] = None, out_fmt: Optional[str] = None) -> Act:
    """V2VNet message aggregation.  nodes[u] = (x image, P image, first pair row r, neighbour count n) of updated node u;
    pair row r + j holds q = W[:, :C] (*) warp(x_j, theta[r + j]).  Returns Act (U,H,W,2C) = [x | agg] when `gru`, else
    Act (U,H,W,C) = x + agg; agg = mean_j (agg_max False) or max_j of mask_j * (q[r + j] + p_node[P image])."""
    _need_cuda(theta)
    H, W, C, U = x.H, x.W, x.C, len(nodes)
    th = _theta64(theta, q.N)
    assert (q.H, q.W, q.C) == (H, W, C) and (p_node.H, p_node.W, p_node.C) == (H, W, C)
    flat = [int(v) for nd in nodes for v in nd]
    assert len(flat) == 4 * U
    cout = 2 * C if gru else C
    out = _out_act(out, U, H, W, cout, out_fmt or x.fmt, x.device)
    pairs = float(sum(nd[3] for nd in nodes))
    with _Prof("v2v_aggregate", 3.0 * pairs * C * H * W,
               (pairs * BPE[q.fmt] + U * (BPE[p_node.fmt] + BPE[x.fmt]) + U * (cout // C) * BPE[out.fmt]) * float(C) * H * W):
        _call("heal_v2v_aggregate", q.view(), p_node.view(), x.view(), _p(th), _host_i32(flat), U, H, W, C,
              1 if agg_max else 0, 1 if gru else 0, out.view())
    return out


@_guard
def gru_gate(zc: Act, out: Optional[Act] = None, out_fmt: Optional[str] = None) -> Act:
    """Zero-hidden ConvGRU cell output: zc Act (N,H,W,2C) = (update-gate | candidate) conv output -> Act (N,H,W,C)
    = sigmoid(zc[..., :C]) * tanh(zc[..., C:])."""
    N, H, W = zc.N, zc.H, zc.W
    assert zc.C % 2 == 0
    C = zc.C // 2
    out = _out_act(out, N, H, W, C, out_fmt or zc.fmt, zc.device)
    npix = N * H * W
    with _Prof("gru_gate", 4.0 * npix * C, npix * float(C) * (2 * BPE[zc.fmt] + BPE[out.fmt])):
        _call("heal_gru_gate", zc.view(), npix, C, out.view())
    return out


@_guard
def ego_mha(q: Act, kv: Act, kv_bias: torch.Tensor, theta: torch.Tensor, n_agents: Sequence[int], heads: int = 8,
            kv_coffset: int = 0, out: Optional[Act] = None, out_fmt: Optional[str] = None) -> Act:
    """Where2comm's per-pixel multi-head attention of each scene's warped ego over its warped agents.  q Act (B,H,W,C) = the
    in-projected warped egos (bias included, unscaled); kv Act (N,H,W,>=kv_coffset+2C) = the bias-free k | v projection of the
    UNWARPED agent maps from channel kv_coffset, N = sum(n_agents), record_len order; kv_bias (2C) fp32 device; theta (N,2,3)
    = affine[b, 0, j] stacked scene by scene -> Act (B,H,W,C), the merged heads before out_proj."""
    _need_cuda(kv_bias, theta)
    B, H, W, C = len(n_agents), q.H, q.W, q.C
    N = sum(int(v) for v in n_agents)
    assert q.N == B and kv.N == N and (kv.H, kv.W) == (H, W) and kv_coffset + 2 * C <= kv.C
    assert kv_bias.dtype == torch.float32 and kv_bias.is_contiguous() and kv_bias.shape == (2 * C,)
    th = _theta64(theta, N)
    out = _out_act(out, B, H, W, C, out_fmt or q.fmt, q.device)
    with _Prof("ego_mha", 4.0 * N * H * W * C + 16.0 * N * H * W * C,
               B * H * W * float(C) * (BPE[q.fmt] + BPE[out.fmt]) + N * H * W * 2.0 * C * BPE[kv.fmt]):
        _call("heal_ego_mha", q.view(), kv.view(kv_coffset), _p(kv_bias), _p(th), _host_i32(n_agents), B, H, W, C, int(heads),
              out.view())
    return out


@_guard
def swap_attention(qkv: Act, n_agents: Sequence[int], L: int, window_size: int, grid: bool, bias: torch.Tensor,
                   out: Optional[Act] = None, out_fmt: Optional[str] = None) -> Act:
    """CoBEVT window (grid False) or grid (grid True) attention core.  qkv Act (B*L,H,W,3C) = to_qkv output with q pre-scaled;
    n_agents: host sequence of the B scenes' real-agent counts; bias (C/32, n, n) fp32 device, key-major (bias[h, j, i]),
    n = L * window_size^2 -> Act (B*L,H,W,C) = softmax over the real agents' keys of (q k^T + bias) v, heads merged."""
    _need_cuda(bias)
    B, H, W, C = len(n_agents), qkv.H, qkv.W, qkv.C // 3
    n = L * window_size * window_size
    assert qkv.N == B * L and qkv.C == 3 * C and bias.dtype == torch.float32 and bias.is_contiguous()
    assert bias.shape == (C // 32, n, n)
    out = _out_act(out, B * L, H, W, C, out_fmt or qkv.fmt, qkv.device)
    keys = float(sum(int(v) for v in n_agents)) * window_size * window_size     # valid keys per query, summed over scenes
    wins = (H // window_size) * (W // window_size)
    with _Prof("swap_attention", 4.0 * keys * C * wins * n,
               B * L * H * W * float(C) * (3 * BPE[qkv.fmt] + BPE[out.fmt])):
        _call("heal_swap_attention", qkv.view(), _host_i32(n_agents), B, L, H, W, C, int(window_size), 1 if grid else 0,
              _p(bias), out.view())
    return out


@_guard
def mean_layernorm(x: Act, n_avg: int, ln_weight: torch.Tensor, ln_bias: torch.Tensor, eps: float,
                   out: Optional[Act] = None, out_fmt: Optional[str] = None) -> Act:
    """x Act (N*n_avg,H,W,C) -> Act (N,H,W,C): LayerNorm over channels of the mean of every n_avg consecutive images
    (n_avg = 1: a plain channels-last LayerNorm)."""
    _need_cuda(ln_weight, ln_bias)
    assert x.N % n_avg == 0
    N, H, W, C = x.N // n_avg, x.H, x.W, x.C
    out = _out_act(out, N, H, W, C, out_fmt or x.fmt, x.device)
    lw, lb = ln_weight.float().contiguous(), ln_bias.float().contiguous()
    with _Prof("mean_layernorm", 0, N * H * W * float(C) * (n_avg * BPE[x.fmt] + BPE[out.fmt])):
        _call("heal_mean_layernorm", x.view(), N, int(n_avg), H, W, C, _p(lw), _p(lb), float(eps), out.view())
    return out


@_guard
def window_attention(qkv: Act, heads: int, dim_head: int, window_size: int, bias: torch.Tensor, qkv_coffset: int = 0,
                     out: Optional[Act] = None, out_coffset: int = 0, out_fmt: Optional[str] = None) -> Act:
    """One V2X-ViT window-attention branch.  qkv Act (N,H,W,>=3*heads*dim_head): q | k | v of the branch from channel
    qkv_coffset (q pre-scaled); bias (w^2, w^2) fp32 device, query-major -> Act (N,H,W,heads*dim_head), or written to
    channels out_coffset .. of `out`: softmax(q k^T + bias) v per window and head, heads merged."""
    _need_cuda(bias)
    N, H, W = qkv.N, qkv.H, qkv.W
    inner, n = heads * dim_head, window_size * window_size
    assert qkv_coffset + 3 * inner <= qkv.C and bias.dtype == torch.float32 and bias.is_contiguous() and bias.shape == (n, n)
    if out is None:
        out = act_empty(N, H, W, inner, out_fmt or qkv.fmt, qkv.device)
    assert (out.N, out.H, out.W) == (N, H, W) and out_coffset + inner <= out.C
    with _Prof("window_attention", 4.0 * N * H * W * n * inner,
               N * H * W * float(inner) * (3 * BPE[qkv.fmt] + BPE[out.fmt])):
        _call("heal_window_attention", qkv.view(qkv_coffset), N, H, W, int(heads), int(dim_head), int(window_size), _p(bias),
              out.view(out_coffset))
    return out


@_guard
def cav_attention(qkv: Act, n_agents: Sequence[int], ego_only: bool, out: Optional[Act] = None,
                  out_fmt: Optional[str] = None) -> Act:
    """V2X-ViT per-pixel agent attention (HGTCavAttention with agent types 0).  qkv Act (N,H,W,3C), N = sum(n_agents), images
    ordered egos first (image b = ego of scene b), then each scene's other agents in scene order -> Act (N,H,W,C), or
    (B,H,W,C) for the egos only: softmax over the scene's agents of q_i . k_j, then sum_j p_j v_j, per head of 32."""
    B, H, W, C = len(n_agents), qkv.H, qkv.W, qkv.C // 3
    total = sum(int(v) for v in n_agents)
    assert qkv.N == total and qkv.C == 3 * C
    nq = B if ego_only else total
    out = _out_act(out, nq, H, W, C, out_fmt or qkv.fmt, qkv.device)
    pairs = float(sum(int(v) for v in n_agents)) if ego_only else float(sum(int(v) ** 2 for v in n_agents))
    with _Prof("cav_attention", 4.0 * pairs * H * W * C, H * W * float(C) * (2 * total + nq) * BPE[qkv.fmt]
               + nq * H * W * float(C) * BPE[out.fmt]):
        _call("heal_cav_attention", qkv.view(), _host_i32(n_agents), B, H, W, C, 1 if ego_only else 0, out.view())
    return out


@_guard
def split_attn(o: Act, x: Act, fc1_t: torch.Tensor, ln_weight: torch.Tensor, ln_bias: torch.Tensor, eps: float,
               fc2_t: torch.Tensor, out: Optional[Act] = None, out_fmt: Optional[str] = None) -> Act:
    """SplitAttn + residual.  o Act (N,H,W,3C) = the three branch outputs side by side, x Act (N,H,W,C) -> Act (N,H,W,C) =
    sum_r o_r * gate_r + x, gate = the per-image softmax gate of split_attn.py (fc1_t (C,C), fc2_t (C,3C): transposed Linear
    weights, fp32 device)."""
    _need_cuda(fc1_t, fc2_t, ln_weight, ln_bias)
    N, H, W, C = x.N, x.H, x.W, x.C
    assert (o.N, o.H, o.W, o.C) == (N, H, W, 3 * C)
    assert fc1_t.shape == (C, C) and fc2_t.shape == (C, 3 * C) and fc1_t.is_contiguous() and fc2_t.is_contiguous()
    out = _out_act(out, N, H, W, C, out_fmt or x.fmt, x.device)
    lw, lb = ln_weight.float().contiguous(), ln_bias.float().contiguous()
    nbytes = int(lib.heal_split_attn_workspace(N, C))
    ws = _workspace(x.device, nbytes)
    with _Prof("split_attn", N * (2.0 * C * C * 4 + 6.0 * H * W * C),
               N * H * W * float(C) * (6 * BPE[o.fmt] + BPE[x.fmt] + BPE[out.fmt])):
        _call("heal_split_attn", o.view(), x.view(), N, H, W, C, _p(fc1_t), _p(lw), _p(lb), float(eps),
              _p(fc2_t), _p(ws), ws.numel(), out.view())
    return out


@_guard
def sttf_resample(src: Act, theta: torch.Tensor, out: Optional[Act] = None, out_fmt: Optional[str] = None) -> Act:
    """V2X-ViT STTF warp: out image k = grid_sample(src image k, affine_grid(theta[k])), bilinear, zeros, align_corners=True.
    theta (N,2,3) fp32 on the device."""
    _need_cuda(theta)
    N, H, W, C = src.N, src.H, src.W, src.C
    assert theta.dtype == torch.float32 and theta.is_contiguous() and theta.shape == (N, 2, 3)
    out = _out_act(out, N, H, W, C, out_fmt or src.fmt, src.device)
    with _Prof("sttf_resample", 8.0 * N * C * H * W, N * (BPE[src.fmt] + BPE[out.fmt]) * float(C) * H * W):
        _call("heal_sttf_resample", src.view(), _p(theta), N, H, W, C, out.view())
    return out


# ------------------------------------------------------------------------------------------------
# Lift-Splat-Shoot
# ------------------------------------------------------------------------------------------------
@_guard
def lss_camera_matrices(rots, intrins, post_rots):
    """(…,3,3) f32 each -> (post_rots^-1, rots @ intrins^-1) as (BN,3,3) f32; one capturable launch (torch.inverse is not)."""
    _need_cuda(rots, intrins, post_rots)
    r = rots.reshape(-1, 3, 3).contiguous().float()
    k = intrins.reshape(-1, 3, 3).contiguous().float()
    pr = post_rots.reshape(-1, 3, 3).contiguous().float()
    post_inv, combine = torch.empty_like(pr), torch.empty_like(r)
    _call("heal_lss_camera_matrices", _p(r), _p(k), _p(pr), r.shape[0], _p(post_inv), _p(combine))
    return post_inv, combine


@_guard
def lss_cell_index(frustum, post_rots_inv, post_trans, combine, trans, lower, dx, nx) -> torch.Tensor:
    """frustum (D,fH,fW,3); per-image 3x3 / 3-vectors (BN,...) -> int32 (BN,D,fH,fW) BEV cell or -1."""
    _need_cuda(frustum, post_rots_inv, post_trans, combine, trans)
    D, fH, fW, _ = frustum.shape
    BN = post_trans.shape[0]
    cell = torch.empty((BN, D, fH, fW), dtype=torch.int32, device=frustum.device)
    with _Prof("lss_cell_index", 0, BN * D * fH * fW * 4.0 + D * fH * fW * 12.0):
        _call("heal_lss_cell_index", _p(frustum.contiguous().float()), D, fH, fW, _p(post_rots_inv.contiguous().float()),
              _p(post_trans.contiguous().float()), _p(combine.contiguous().float()),
              _p(trans.contiguous().float()), BN, _host_f32(lower), _host_f32(dx), _host_i32(nx), _p(cell))
    return cell


@_guard
def lss_pool(depth_logits, feat, cell, cams_per_agent: int, nx, ny) -> Act:
    """depth_logits (BN,D,fH,fW), feat (BN,C,fH,fW) f32 NCHW, cell (BN,D,fH,fW) -> Act f32 (agents, ny, nx, C)."""
    _need_cuda(depth_logits, feat, cell)
    BN, D, fH, fW = depth_logits.shape
    C = feat.shape[1]
    agents = BN // cams_per_agent
    with _Prof("lss_pool(+bev memset)", 2.0 * BN * D * fH * fW * C,
               BN * fH * fW * 4.0 * (2 * D + C) + agents * float(ny) * nx * C * 4):
        out = act_zeros(agents, ny, nx, C, "f32", feat.device)
        _call("heal_lss_pool", _p(depth_logits.contiguous().float()), _p(feat.contiguous().float()), _p(cell.contiguous()),
              BN, cams_per_agent, D, C, fH, fW, nx * ny, _p(out.t))
    return out


@_guard
def lss_pool_sorted(logits: torch.Tensor, l_strides, feat: torch.Tensor, f_strides, cell: torch.Tensor, cams_per_agent: int,
                    D: int, C: int, fH: int, fW: int, nx: int, ny: int, out_fmt: str = "f32") -> Act:
    """Deterministic LSS pooling (heal_lss_pool_sorted).  `logits` / `feat` are fp32 tensors whose data_ptr is the first logit /
    feature element, described by ELEMENT strides (image, depth-bin | channel, pixel); cell (BN,D,fH,fW) i32.
    Returns Act (agents, ny, nx, C) in `out_fmt` (zero where no frustum point lands)."""
    _need_cuda(logits, feat, cell)
    assert logits.dtype == torch.float32 and feat.dtype == torch.float32 and cell.dtype == torch.int32 and cell.is_contiguous()
    BN = cell.shape[0]
    agents = BN // cams_per_agent
    out = act_zeros(agents, ny, nx, C, out_fmt, feat.device)
    wsb = lib.heal_lss_pool_sorted_workspace(BN, D, fH, fW, agents, nx * ny)
    ws = _workspace(feat.device, wsb)
    npts = BN * D * fH * fW
    with _Prof("lss_pool_sorted", 2.0 * npts * C, BN * fH * fW * 4.0 * (2 * D + C) + agents * float(ny) * nx * C * BPE[out_fmt]):
        _call("heal_lss_pool_sorted", _p(logits), int(l_strides[0]), int(l_strides[1]), int(l_strides[2]),
              _p(feat), int(f_strides[0]), int(f_strides[1]), int(f_strides[2]),
              _p(cell), BN, cams_per_agent, D, C, fH, fW, nx * ny, out.view(), _p(ws), ws.numel())
    return out


# ------------------------------------------------------------------------------------------------
# EfficientNet-B0 camera trunk (csrc/mbconv.cu): dense channels-last fp32 tensors, BN folded on the host in fp64
# ------------------------------------------------------------------------------------------------
def _fold_conv_bn(conv, bn):
    """(weight * bn scale (Cout, Cin/g, kh, kw), bias) in fp64 on the host."""
    w = conv.weight.detach().double().cpu()
    scale, shift = _bn_scale_shift(bn, w.shape[0])
    b = shift + (conv.bias.detach().double().cpu() * scale if conv.bias is not None else 0)
    return w * scale[:, None, None, None], b


def pack_stem_conv(conv, bn):
    """Conv2d(3, 32, 3, stride 2) + BN -> (weight (27, 32), row = (ci*3 + ky)*3 + kx; bias (32)) for heal_stem_conv_swish."""
    w, b = _fold_conv_bn(conv, bn)
    assert w.shape == (32, 3, 3, 3) and conv.stride == (2, 2)
    return w.reshape(32, 27).t().contiguous().float(), b.float().contiguous()


def pack_dwconv(conv, bn):
    """depthwise Conv2d(C, C, k, groups=C) + BN -> (weight (k*k, C) tap-major, bias (C)) for heal_dwconv_bn_swish."""
    w, b = _fold_conv_bn(conv, bn)
    C, one, k, k2 = w.shape
    assert one == 1 and k == k2 and conv.groups == C
    return w.reshape(C, k * k).t().contiguous().float(), b.float().contiguous()


def pack_pwconv(conv, bn):
    """Conv2d(Cin, Cout, 1) (+ BN) -> (weight (Cin, Cout), bias (Cout)) for heal_pwconv."""
    w, b = _fold_conv_bn(conv, bn)
    assert w.shape[2:] == (1, 1) and conv.groups == 1
    return w[:, :, 0, 0].t().contiguous().float(), b.float().contiguous()


def pack_se(se_reduce, se_expand):
    """The two biased 1x1 convs of squeeze-and-excitation -> (w_reduce (Csq, C), b_reduce, w_expand_t (Csq, C), b_expand)."""
    wr, we = se_reduce.weight.detach()[:, :, 0, 0], se_expand.weight.detach()[:, :, 0, 0]
    return (wr.float().contiguous().cpu(), se_reduce.bias.detach().float().contiguous().cpu(),
            we.t().float().contiguous().cpu(), se_expand.bias.detach().float().contiguous().cpu())


def _dense_f32(a: Act):
    assert a.fmt == "f32" and a.cstride == a.C and a.t.is_contiguous(), "the MBConv kernels read dense fp32 channels-last maps"


@_guard
def stem_conv_swish(x: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor) -> Act:
    """x (N, 3|4, H, W) fp32 NCHW -> Act f32 (N, (H-2)//2+1, (W-2)//2+1, 32): 3x3/2 conv of the first 3 channels, pad (0, 1), swish."""
    _need_cuda(x, weight, bias)
    assert x.dtype == torch.float32 and x.dim() == 4 and x.is_contiguous() and weight.shape == (27, 32)
    N, Cx, H, W = x.shape
    Ho, Wo = (H - 2) // 2 + 1, (W - 2) // 2 + 1
    out = act_empty(N, Ho, Wo, 32, "f32", x.device)
    with _Prof("stem_conv_swish", 2.0 * N * Ho * Wo * 32 * 27, 4.0 * N * (3 * H * W + Ho * Wo * 32)):
        _call("heal_stem_conv_swish", _p(x), N, Cx, H, W, _p(weight), _p(bias), _p(out.t))
    return out


@_guard
def dwconv_bn_swish(x: Act, weight: torch.Tensor, bias: torch.Tensor, ksize: int, stride: int, pads):
    """Depthwise conv + folded BN + swish.  pads = (top, bottom, left, right).  Returns (Act f32, sums (N, C) fp32): sums is the sum
    of the output over its pixels (the squeeze of squeeze-and-excitation before the division), bit-identical run to run."""
    _need_cuda(weight, bias)
    _dense_f32(x)
    N, H, W, C = x.N, x.H, x.W, x.C
    assert weight.shape == (ksize * ksize, C)
    pt, pb, pl, pr = pads
    Ho, Wo = (H + pt + pb - ksize) // stride + 1, (W + pl + pr - ksize) // stride + 1
    out = act_empty(N, Ho, Wo, C, "f32", x.device)
    sums = torch.empty((N, C), dtype=torch.float32, device=x.device)
    ws = _workspace(x.device, lib.heal_dwconv_bn_swish_workspace(N, C, Ho, Wo))
    with _Prof("dwconv_bn_swish", 2.0 * N * Ho * Wo * C * ksize * ksize, 4.0 * N * C * (H * W + Ho * Wo)):
        _call("heal_dwconv_bn_swish", _p(x.t), N, H, W, C, _p(weight), _p(bias), int(ksize), int(stride), int(pt), int(pl),
              Ho, Wo, _p(out.t), _p(sums), _p(ws), ws.numel())
    return out, sums


@_guard
def se_gate(sums: torch.Tensor, hw: int, w_reduce, b_reduce, w_expand_t, b_expand) -> torch.Tensor:
    """sums (N, C) over hw pixels -> gate (N, C) = sigmoid(expand(swish(reduce(sums / hw))))."""
    _need_cuda(sums, w_reduce, b_reduce, w_expand_t, b_expand)
    N, C = sums.shape
    Csq = w_reduce.shape[0]
    assert sums.is_contiguous() and w_reduce.shape == (Csq, C) and w_expand_t.shape == (Csq, C)
    gate = torch.empty_like(sums)
    with _Prof("se_gate", 4.0 * N * C * Csq, 8.0 * C * Csq + 8.0 * N * C):
        _call("heal_se_gate", _p(sums), N, C, Csq, int(hw), _p(w_reduce), _p(b_reduce), _p(w_expand_t), _p(b_expand), _p(gate))
    return gate


@_guard
def pwconv(x: Act, weight: torch.Tensor, bias: torch.Tensor, gate: Optional[torch.Tensor] = None, swish: bool = False,
           residual: Optional[Act] = None) -> Act:
    """1x1 conv with folded BN: out = act((x * gate[image]) @ weight + bias) + residual.  weight (Cin, Cout)."""
    _need_cuda(weight, bias, gate)
    _dense_f32(x)
    N, H, W, Cin = x.N, x.H, x.W, x.C
    Cout = weight.shape[1]
    assert weight.shape[0] == Cin and weight.is_contiguous()
    if gate is not None:
        assert gate.shape == (N, Cin) and gate.is_contiguous()
    if residual is not None:
        _dense_f32(residual)
        assert (residual.N, residual.H, residual.W, residual.C) == (N, H, W, Cout)
    out = act_empty(N, H, W, Cout, "f32", x.device)
    with _Prof("pwconv", 2.0 * N * H * W * Cin * Cout,
               4.0 * N * H * W * (Cin + Cout * (2 if residual is not None else 1)) + 4.0 * Cin * Cout):
        _call("heal_pwconv", _p(x.t), N, H * W, Cin, Cout, _p(weight), _p(bias), _p(gate), 1 if swish else 0,
              _p(residual.t) if residual is not None else _vp(0), _p(out.t))
    return out


@_guard
def upsample2x_concat(x1: Act, x2: Act, out_fmt: str) -> Act:
    """`Up`'s front half (lss_submodule.py:33-35): Act (N, 2*H1, 2*W1, C) in `out_fmt` holding [x2 | bilinear x2 (align_corners=True) of
    x1 | zeros], C = C2 + C1 rounded up to a multiple of 64 (the tensor-core convolution's input-channel granularity)."""
    N, H1, W1 = x1.N, x1.H, x1.W
    assert (x2.N, x2.H, x2.W) == (N, 2 * H1, 2 * W1)
    C = (x1.C + x2.C + 63) // 64 * 64
    out = act_empty(N, 2 * H1, 2 * W1, C, out_fmt, x1.device)
    with _Prof("upsample2x_concat", 8.0 * N * 4 * H1 * W1 * x1.C,
               N * H1 * W1 * (x1.C * BPE[x1.fmt] + 4.0 * x2.C * BPE[x2.fmt] + 4.0 * C * BPE[out_fmt])):
        _call("heal_upsample2x_concat", x1.view(), x2.view(), N, H1, W1, x1.C, x2.C, out.view(), C)
    return out


# ------------------------------------------------------------------------------------------------
# camera input (csrc/camera_input.cu): raw uint8 frames -> the reference's inference resize, crop and normalisation
# ------------------------------------------------------------------------------------------------
CAMERA_LAYOUTS = {"nchw": 0, "s2d": 1}


@_guard
def camera_input(frames: torch.Tensor, plan, layout: str = "nchw"):
    """frames uint8 (n, H0, W0, 3) CUDA, HWC as decoded; plan = data_utils.camera_input.inference_plan(conf, H0, W0).
    layout 'nchw' -> fp32 (n, 3, fH, fW), what normalize_img returns per frame (CamEncode's input);
    layout 's2d'  -> Act f32 (n, fH/4, fW/4, 64), channel c*16 + dy*4 + dx with c == 3 zero: pixel_unshuffle(image with a zero 4th
                     plane, 4), the ResNet-101 stem's space-to-depth input."""
    if not isinstance(frames, torch.Tensor) or frames.dtype != torch.uint8:
        raise TypeError(f"camera_input: frames must be a uint8 tensor, got {getattr(frames, 'dtype', type(frames))}")
    if frames.dim() != 4 or frames.shape[3] != 3:
        raise ValueError(f"camera_input: frames must be (n, H0, W0, 3) RGB, got {tuple(frames.shape)}")
    if not frames.is_contiguous():
        raise ValueError("camera_input: frames must be contiguous")
    if layout not in CAMERA_LAYOUTS:
        raise ValueError(f"camera_input: layout '{layout}', expected one of {sorted(CAMERA_LAYOUTS)}")
    n, H0, W0, _ = frames.shape
    if (H0, W0) != (plan.H0, plan.W0):
        raise ValueError(f"camera_input: frames are {H0}x{W0}, the plan was made for {plan.H0}x{plan.W0}")
    fH, fW = plan.final_dim
    l, t, r, b = plan.crop
    if (b - t, r - l) != (fH, fW):
        raise ValueError(f"camera_input: crop {plan.crop} is {b - t}x{r - l}, final_dim is {fH}x{fW}")
    if layout == "s2d" and (fH % 8 or fW % 8):
        raise ValueError(f"camera_input: the space-to-depth layout needs sides that are multiples of 8, final_dim is {fH}x{fW}")
    _need_cuda(frames)
    cols, ck, rows, rk, span = plan.tables(frames.device)
    if layout == "nchw":
        out = torch.empty((n, 3, fH, fW), dtype=torch.float32, device=frames.device)
        res = out
    else:
        res = act_empty(n, fH // 4, fW // 4, 64, "f32", frames.device)
        out = res.t
    with _Prof("camera_input", 0, float(n) * H0 * W0 * 3 + 4.0 * out.numel()):
        _call("heal_camera_input", _p(frames), n, H0, W0, _p(cols), ck, _p(rows), rk, fH, fW, span, CAMERA_LAYOUTS[layout],
              _p(out))
    return res


# ------------------------------------------------------------------------------------------------
# sparse 3-D convolution (SECOND)
# ------------------------------------------------------------------------------------------------
class SparseTensor:
    """feats (cap,C) f32 | None, coords (cap,4) i32 [b,z,y,x], rows_dev (1,) i32 device count or None (= cap rows live),
    spatial_shape [Z,Y,X], batch.  `table` (keys, vals) maps a site to its row (built on demand)."""

    def __init__(self, feats, coords, rows_dev, spatial_shape, batch, table=None, table_capacity=None):
        self.feats, self.coords, self.rows_dev = feats, coords, rows_dev
        self.spatial_shape, self.batch, self.table = [int(v) for v in spatial_shape], int(batch), table
        self.capacity = coords.shape[0]
        self.table_capacity = table_capacity if table_capacity is not None else self.capacity

    def with_feats(self, feats):
        return SparseTensor(feats, self.coords, self.rows_dev, self.spatial_shape, self.batch, self.table, self.table_capacity)

    def dense(self):
        """(B, C, D, H, W) like spconv's SparseConvTensor.dense() (test / API helper; one host sync)."""
        m = int(self.rows_dev[0].item()) if self.rows_dev is not None else self.capacity
        m = min(m, self.capacity)
        c = self.coords[:m].long()
        out = torch.zeros((self.batch, self.feats.shape[1], *self.spatial_shape), dtype=torch.float32, device=self.feats.device)
        out[c[:, 0], :, c[:, 1], c[:, 2], c[:, 3]] = self.feats[:m]
        return out


@_guard
def sp_build_table(st: SparseTensor):
    if st.table is None:
        ts = lib.heal_spconv_table_size(st.capacity)
        keys = torch.empty((ts,), dtype=torch.int32, device=st.coords.device)
        vals = torch.empty((ts,), dtype=torch.int32, device=st.coords.device)
        with _Prof("spconv_rulebook"):
            _call("heal_spconv_build_table", _p(st.coords), _p(st.rows_dev), st.capacity, _host_i32(st.spatial_shape), st.batch,
                  _p(keys), _p(vals))
        st.table = (keys, vals)
    return st.table


@_guard
def sp_subm_neighbors(st: SparseTensor, ksize) -> torch.Tensor:
    keys, vals = sp_build_table(st)
    K = int(ksize[0] * ksize[1] * ksize[2])
    nbr = torch.empty((st.capacity, K), dtype=torch.int32, device=st.coords.device)
    with _Prof("spconv_rulebook"):
        _call("heal_spconv_subm_neighbors", _p(st.coords), _p(st.rows_dev), st.capacity, _host_i32(st.spatial_shape),
              _host_i32(ksize), _p(keys), _p(vals), st.table_capacity, _p(nbr))
    return nbr


SP_GROWTH = 2.0     # default output-row capacity of a strided sparse conv relative to its input capacity (see sp_strided)


@_guard
def sp_strided(st: SparseTensor, ksize, stride, pad, out_capacity: Optional[int] = None):
    """SparseConv3d rulebook: returns (output SparseTensor without feats, nbr (out_cap, K)).  No host sync: the live output
    row count stays on the device (`rows_dev`; rows beyond `out_capacity` are dropped by the kernels and show up as
    rows_dev > capacity, which `sp_check_overflow` reports).  Default capacity = SP_GROWTH x the input capacity, bounded by
    the exact worst case (fan-out x inputs, number of cells): a stride-2 3x3x3 conv dilates LiDAR surfaces by ~1.3x at the
    0.1 m level and shrinks them afterwards, and the voxeliser's own capacity already carries ~1.6x headroom."""
    oshape = [(st.spatial_shape[i] + 2 * pad[i] - ksize[i]) // stride[i] + 1 for i in range(3)]
    K = int(ksize[0] * ksize[1] * ksize[2])
    if out_capacity is None:
        fan = 1
        for i in range(3):
            fan *= -(-ksize[i] // stride[i])
        out_capacity = int(min(st.capacity * fan, st.batch * oshape[0] * oshape[1] * oshape[2],
                               max(int(st.capacity * SP_GROWTH), 1024), 1 << 20))        # 2^20 rows: the rulebook scan's limit
    dev = st.coords.device
    ts = lib.heal_spconv_table_size(out_capacity)
    okeys = torch.empty((ts,), dtype=torch.int32, device=dev)
    ovals = torch.empty((ts,), dtype=torch.int32, device=dev)
    ocoords = torch.empty((out_capacity, 4), dtype=torch.int32, device=dev)
    orows = torch.zeros((1,), dtype=torch.int32, device=dev)
    nbr = torch.empty((out_capacity, K), dtype=torch.int32, device=dev)
    wsb = lib.heal_spconv_strided_workspace(st.capacity, out_capacity, K)
    ws = _workspace(dev, wsb)
    with _Prof("spconv_rulebook"):
        _call("heal_spconv_strided_rulebook", _p(st.coords), _p(st.rows_dev), st.capacity, _host_i32(oshape), st.batch,
              _host_i32(ksize), _host_i32(stride), _host_i32(pad), out_capacity,
              _p(ocoords), _p(orows), _p(okeys), _p(ovals), _p(nbr), _p(ws), ws.numel())
    return SparseTensor(None, ocoords, orows, oshape, st.batch, (okeys, ovals), table_capacity=out_capacity), nbr


def sp_check_overflow(tensors) -> None:
    """ONE host sync for a whole encoder: raises if any strided conv produced more rows than its capacity."""
    live = [t for t in tensors if t.rows_dev is not None]
    if not live:
        return
    counts = torch.cat([t.rows_dev[:1] for t in live]).tolist()
    for t, n in zip(live, counts):
        if n > t.capacity:
            raise RuntimeError(f"sparse conv output rows {n} exceed the capacity {t.capacity} (spatial shape {t.spatial_shape}); "
                               "raise heal_b200.ops.SP_GROWTH or pass out_capacity")


@_guard
def sp_gather_gemm(feats: torch.Tensor, nbr: torch.Tensor, rows_dev, weight: torch.Tensor, bias, relu: bool) -> torch.Tensor:
    """feats (Min,Cin) f32; nbr (cap,K) i32; weight (K,Cin,Cout) f32 (BN folded) -> (cap,Cout) f32."""
    _need_cuda(feats, nbr, weight)
    cap, K = nbr.shape
    Kw, cin, cout = weight.shape
    assert Kw == K and feats.shape[1] == cin and feats.is_contiguous()
    out = torch.empty((cap, cout), dtype=torch.float32, device=feats.device)
    def _pairs():
        m = cap if rows_dev is None else min(cap, int(rows_dev[0].item()))
        return float((nbr[:m] >= 0).sum().item()), float(m)
    with _Prof("spconv_gather_gemm", lambda: 2.0 * _pairs()[0] * cin * cout,
               lambda: _pairs()[0] * (cin * 4.0 + 4.0) + _pairs()[1] * (cout * 4.0 + K * 4.0)):
        _call("heal_spconv_gather_gemm", _p(feats), _p(nbr), _p(rows_dev), cap, K, _p(weight), _p(bias), cin, cout,
              1 if relu else 0, _p(out))
    return out


def pack_spconv_tc(wp: torch.Tensor) -> torch.Tensor:
    """Folded sparse-conv weights (K, Cin, Cout) fp32 -> [2 planes][KB*Cout rows][64] bf16 for heal_spconv_gather_gemm_tc:
    K-block kb holds the 64/Cin kernel offsets kb*TPK .. kb*TPK+TPK-1 side by side along K (zero columns for padding offsets)."""
    K, cin, cout = wp.shape
    assert cin in (16, 32, 64)
    tpk = 64 // cin
    kb = -(-K // tpk)
    rows = torch.zeros((kb, cout, 64), dtype=torch.float32)
    w = wp.detach().float().cpu()
    for k in range(K):
        b, tl = divmod(k, tpk)
        rows[b, :, tl * cin:(tl + 1) * cin] = w[k].t()
    return split_bf16(rows.reshape(kb * cout, 64), 2).to(wp.device)


@_guard
def rows_to_split(feats: torch.Tensor, rows_dev) -> torch.Tensor:
    """(cap, C) fp32 rows -> (cap, 2C) bf16 split rows [hi | lo]."""
    cap, C = feats.shape
    out = torch.empty((cap, 2 * C), dtype=torch.bfloat16, device=feats.device)
    with _Prof("rows_to_split", 0, cap * C * 8.0):
        _call("heal_rows_to_split", _p(feats), _p(rows_dev), cap, C, _p(out))
    return out


@_guard
def sp_gather_gemm_tc(feats_split: torch.Tensor, nbr: torch.Tensor, rows_dev, w_packed: torch.Tensor, bias, relu: bool,
                      cin: int, cout: int, want_f32: bool = False) -> torch.Tensor:
    """feats_split (Min, 2*Cin) bf16 split rows; nbr (cap,K) i32 -> (cap, 2*Cout) bf16 split rows, or (cap, Cout) fp32."""
    _need_cuda(feats_split, nbr, w_packed)
    cap, K = nbr.shape
    assert feats_split.dtype == torch.bfloat16 and feats_split.shape[1] == 2 * cin and feats_split.is_contiguous()
    dev = feats_split.device
    out = torch.empty((cap, cout), dtype=torch.float32, device=dev) if want_f32 else torch.empty((cap, 2 * cout), dtype=torch.bfloat16, device=dev)

    def _pairs():
        m = cap if rows_dev is None else min(cap, int(rows_dev[0].item()))
        return float((nbr[:m] >= 0).sum().item()), float(m)
    with _Prof("spconv_gather_gemm_tc", lambda: 2.0 * _pairs()[0] * cin * cout,
               lambda: _pairs()[0] * (cin * 4.0 + 4.0) + _pairs()[1] * (cout * 4.0 + K * 4.0)):
        _call("heal_spconv_gather_gemm_tc", _p(feats_split), _p(nbr), _p(rows_dev), cap, K, _p(w_packed), _p(bias), cin, cout,
              1 if relu else 0, _vp(0) if want_f32 else _p(out), _p(out) if want_f32 else _vp(0), 0, 0, 0, 0)
    return out


@_guard
def sparse_to_bev(st: SparseTensor) -> Act:
    """HeightCompression: (B, H, W, C*D) channels-last fp32 with channel = c*D + z."""
    D, H, W = st.spatial_shape
    C = st.feats.shape[1]
    with _Prof("sparse_to_bev(+memset)", 0, st.batch * float(H) * W * C * D * 4 + st.capacity * (C * 4.0 + 16)):
        out = act_zeros(st.batch, H, W, C * D, "f32", st.feats.device)
        _call("heal_sparse_to_bev", _p(st.feats), _p(st.coords), _p(st.rows_dev), st.capacity, C, D, H, W, _p(out.t))
    return out


# ------------------------------------------------------------------------------------------------
# sparse stem (PointPillars canvas never materialised)
# ------------------------------------------------------------------------------------------------
class SparseCanvas:
    """Stands for the (B, ny, nx, 64) scatter canvas: pillar features + a cell -> pillar-row map.  `dense(fmt)` materialises
    the canvas for consumers that need it; the first stride-2 residual block consumes it directly (heal_sparse_stem)."""

    def __init__(self, feats, idmap, B, ny, nx, densify, feats_split=None):
        self.feats, self.idmap, self.feats_split = feats, idmap, feats_split
        self.N, self.H, self.W, self.C = B, ny, nx, feats.shape[1]
        self._densify = densify
        self.fmt = "sparse"

    @property
    def device(self):
        return self.feats.device

    def dense(self, fmt: str = "f32") -> Act:
        return self._densify(fmt)


@_guard
def pillar_vfe_sparse(voxel_features, voxel_num_points, voxel_coords, w_folded, b_folded, voxel_size, lidar_range,
                      nx: int, ny: int, batch_size: int, num_voxels_dev: Optional[torch.Tensor] = None,
                      want_split_rows: bool = False) -> SparseCanvas:
    """PillarVFE -> pillar features (M,64) (+ the same as split rows) + id map; no dense canvas."""
    fsplit = torch.empty((voxel_features.shape[0], 2 * w_folded.shape[1]), dtype=torch.bfloat16, device=voxel_features.device) \
        if want_split_rows else None
    pf, _ = pillar_vfe_scatter(voxel_features, voxel_num_points, voxel_coords, w_folded, b_folded, voxel_size, lidar_range,
                               nx, ny, batch_size, want_pillar_features=True, want_canvas=False, num_voxels_dev=num_voxels_dev,
                               split_rows_out=fsplit)
    coords = voxel_coords.to(torch.int32).contiguous()
    idmap = torch.empty((batch_size, ny, nx), dtype=torch.int32, device=pf.device)
    with _Prof("pillar_idmap", 0, batch_size * float(ny) * nx * 4 + coords.shape[0] * 16.0):
        _call("heal_pillar_idmap", _p(coords), _p(num_voxels_dev), coords.shape[0], batch_size, ny, nx, _p(idmap))

    def densify(fmt):
        _, canvas = pillar_vfe_scatter(voxel_features, voxel_num_points, voxel_coords, w_folded, b_folded, voxel_size,
                                       lidar_range, nx, ny, batch_size, num_voxels_dev=num_voxels_dev, canvas_fmt=fmt)
        return canvas

    return SparseCanvas(pf, idmap, batch_size, ny, nx, densify, feats_split=fsplit)


# The stem as two wgmma gather-GEMMs (heal_stem_rulebook + heal_spconv_gather_gemm_tc with planar I/O) instead of k_sparse_stem.
# Correct and tested, but slower on the C2 frame on the B200 build it was first measured on (2 560 output tiles x up to 9 K-blocks
# of mostly zero-filled rows, weights re-streamed per tile) -> opt-in; the fp32 gather kernel stays the default.
STEM_GATHER_TC = False


def _sparse_stem_gather_tc(sc: SparseCanvas, pc_conv: PackedConv, pc_down: PackedConv, o1: Act, o2: Act):
    """The first stride-2 residual block's 3x3 conv and 1x1 downsample as sparse 2-D convolutions on the tensor cores: a rulebook
    (output pixel x kernel offset -> pillar row, from the cell->row id map) + the SECOND encoder's gather-GEMM kernel, which reads
    the pillar list's split rows and writes straight into the dense BEV maps (planar split Acts).  Only offsets that hit a pillar
    somewhere in a 128-pixel tile cost an MMA; empty tiles cost one."""
    B, Ho, Wo = sc.N, sc.H // 2, sc.W // 2
    rows = B * Ho * Wo
    dev = sc.device
    for pc in (pc_conv, pc_down):
        if getattr(pc, "_sp_packed", None) is None or pc._sp_packed.device != dev:
            K = pc.kh * pc.kw
            pc._sp_packed = pack_spconv_tc(pc.weight.reshape(K, pc.cin, pc.w_cstride)[:, :, :pc.cout].contiguous())
    nbr9 = torch.empty((rows, 9), dtype=torch.int32, device=dev)
    nbr1 = torch.empty((rows, 1), dtype=torch.int32, device=dev)
    with _Prof("sparse_stem_rulebook", 0, rows * 40.0 + B * float(sc.H) * sc.W * 4):
        _call("heal_stem_rulebook", _p(sc.idmap), B, sc.H, sc.W, 3, 1, _p(nbr9))
        _call("heal_stem_rulebook", _p(sc.idmap), B, sc.H, sc.W, 1, 0, _p(nbr1))

    def _hits():
        return float((sc.idmap >= 0).sum().item())
    with _Prof("sparse_stem_tc", lambda: 2.0 * 64 * 64 * (2.25 + 0.25) * _hits(),
               lambda: rows * 40.0 + _hits() * 2.5 * 256.0 + 2.0 * rows * 64 * 4):
        for nbr, pc, o, relu in ((nbr9, pc_conv, o1, 1), (nbr1, pc_down, o2, 0)):
            _call("heal_spconv_gather_gemm_tc", _p(sc.feats_split), _p(nbr), _vp(0), rows, nbr.shape[1], _p(pc._sp_packed),
                  _p(pc.bias), 64, 64, relu, _p(o.t), _vp(0), 0, 0, o.cstride, o.plane_stride)
    return o1, o2


@_guard
def sparse_stem(sc: SparseCanvas, pc_conv: PackedConv, pc_down: PackedConv, out_fmt: str, tensor_cores: bool = False):
    """BasicBlock.conv1(3x3 s2 p1)+bn1+ReLU and downsample(1x1 s2)+bn from the pillar list. Returns (Act conv, Act down).
    tensor_cores: split-bf16 mma.sync variant (fp32-equivalent; the tc32 / bf16 engine modes), else fp32 FMAs."""
    assert pc_conv.kh == 3 and pc_conv.stride == 2 and pc_conv.pad == 1 and pc_conv.cin == 64 and pc_conv.cout == 64 and pc_conv.relu
    assert pc_down.kh == 1 and pc_down.stride == 2 and pc_down.pad == 0 and pc_down.cin == 64 and pc_down.cout == 64 and not pc_down.relu
    o1 = act_empty(sc.N, sc.H // 2, sc.W // 2, 64, out_fmt, sc.device)
    o2 = act_empty(sc.N, sc.H // 2, sc.W // 2, 64, out_fmt, sc.device)
    if STEM_GATHER_TC and out_fmt == "split" and sc.feats_split is not None:
        return _sparse_stem_gather_tc(sc, pc_conv, pc_down, o1, o2)
    symbol = "heal_sparse_stem_tc" if (tensor_cores and sc.W % 32 == 0) else "heal_sparse_stem"
    def _stem():
        hits = float((sc.idmap >= 0).sum().item())
        return hits
    with _Prof("sparse_stem", lambda: 2.0 * 64 * 64 * (2.25 + 0.25) * _stem(),
               lambda: sc.N * float(sc.H) * sc.W * 4 + _stem() * 256.0 + 2.0 * sc.N * (sc.H // 2) * (sc.W // 2) * 64 * BPE[out_fmt]):
        _call(symbol, _p(sc.feats), _p(sc.idmap), sc.N, sc.H, sc.W, _p(pc_conv.weight), _p(pc_conv.bias),
              _p(pc_down.weight), _p(pc_down.bias), 64, o1.view(), o2.view())
    return o1, o2


# ------------------------------------------------------------------------------------------------
# detection post-processing (box decode + score filter + rotated NMS), SURVEY 8f rank 1
# ------------------------------------------------------------------------------------------------
class PostprocessBuffers:
    """Caller-owned outputs + workspace of heal_box_decode_nms for one (H, W, anchors, top) geometry (reusable, graph-safe)."""

    def __init__(self, H: int, W: int, A: int, top: int, device):
        self.H, self.W, self.A, self.top = H, W, A, top
        nbytes = int(lib.heal_postprocess_workspace(H, W, A, top))
        if nbytes == 0:
            raise ValueError("bad post-processing geometry")
        self.workspace = torch.empty((nbytes,), dtype=torch.uint8, device=device)
        self.boxes = torch.zeros((top, 8, 3), dtype=torch.float32, device=device)
        self.scores = torch.zeros((top,), dtype=torch.float32, device=device)
        self.count = torch.zeros((1,), dtype=torch.int32, device=device)
        self.stats = torch.zeros((2,), dtype=torch.int32, device=device)


def _head_act(t) -> Act:
    """Accept an Act (f32) or a logical-NCHW fp32 tensor (any strides; channels-last storage is used as is)."""
    if isinstance(t, Act):
        assert t.fmt == "f32"
        return t
    return to_act(t)


@_guard
def box_decode_nms(cls_preds, reg_preds, dir_preds, anchors: torch.Tensor, transform, score_threshold: float, nms_threshold: float,
                   dir_offset: float = 0.0, num_bins: int = 2, order: str = "hwl", gt_range=None, top: int = 1000,
                   buffers: Optional[PostprocessBuffers] = None) -> PostprocessBuffers:
    """VoxelPostprocessor.post_process for one cav on the GPU (no host sync): heads (1,A,H,W) / (1,7A,H,W) / (1,A*bins,H,W) or None,
    anchors (H,W,A,7) fp32 device, transform 4x4 (host values).  Returns the buffers: boxes[:count], scores[:count] in pick order."""
    c, r = _head_act(cls_preds), _head_act(reg_preds)
    d = _head_act(dir_preds) if dir_preds is not None else None
    assert c.N == 1 and r.N == 1 and r.C == 7 * c.C and (d is None or d.C == c.C * num_bins)
    H, W, A = c.H, c.W, c.C
    _need_cuda(anchors)
    assert anchors.dtype == torch.float32 and anchors.is_contiguous() and anchors.numel() == H * W * A * 7
    if buffers is None:
        buffers = PostprocessBuffers(H, W, A, top, anchors.device)
    assert (buffers.H, buffers.W, buffers.A, buffers.top) == (H, W, A, top)
    T = _host_f32(np.asarray(torch.as_tensor(transform).detach().cpu().numpy(), dtype=np.float64).reshape(16))
    rng = _box_range_f32(gt_range) if gt_range is not None else None
    with _Prof("box_decode_nms", 0):
        _call("heal_box_decode_nms", c.view(), r.view(), d.view() if d is not None else None, _p(anchors),
              H, W, A, float(score_threshold), float(np.float32(dir_offset)), int(num_bins), T,
              1 if order == "hwl" else 0, float(nms_threshold), int(top), rng,
              _p(buffers.boxes), _p(buffers.scores), _p(buffers.count), _p(buffers.stats),
              _p(buffers.workspace), buffers.workspace.numel())
    return buffers


def _first_cav_anchors(cavs, *args, **kwargs):
    """box_decode_nms_multi's device argument: the first cav's anchors (the heads may be Acts or tensors)."""
    return cavs[0]["anchors"] if cavs else None


@_guard(device_arg=_first_cav_anchors)
def box_decode_nms_multi(cavs, score_threshold: float, nms_threshold: float, dir_offset: float = 0.0, num_bins: int = 2,
                         order: str = "hwl", gt_range=None, top: int = 1000, buffers: Optional[PostprocessBuffers] = None) -> PostprocessBuffers:
    """VoxelPostprocessor.post_process for SEVERAL cavs (late fusion) and / or `iou_preds` rescoring on the GPU, no host sync.
    cavs: list of dicts {cls, reg, dir | None, iou | None, anchors (H,W,A,7) fp32 device, transform (4x4 host values)}; all cavs share
    H, W, A.  Candidates are concatenated in list order, then filtered, sorted and NMS-ed together (voxel_postprocessor.py:269-397)."""
    n = len(cavs)
    assert n >= 1
    keep = []           # keep the views / arrays alive until the call returns
    arr = (HealCavHeads * n)()
    H = W = A = None
    for i, c in enumerate(cavs):
        cl, rg = _head_act(c["cls"]), _head_act(c["reg"])
        dr = _head_act(c["dir"]) if c.get("dir") is not None else None
        io = _head_act(c["iou"]) if c.get("iou") is not None else None
        if H is None:
            H, W, A = cl.H, cl.W, cl.C
        assert (cl.H, cl.W, cl.C) == (H, W, A) and cl.N == 1 and rg.C == 7 * A
        an = c["anchors"]
        _need_cuda(an)
        assert an.dtype == torch.float32 and an.is_contiguous() and an.numel() == H * W * A * 7
        views = [cl.view(), rg.view(), dr.view() if dr is not None else None, io.view() if io is not None else None]
        T = _host_f32(np.asarray(torch.as_tensor(c["transform"]).detach().cpu().numpy(), dtype=np.float64).reshape(16))
        keep.append((cl, rg, dr, io, views, T, an))
        arr[i].cls, arr[i].reg = ctypes.pointer(views[0]), ctypes.pointer(views[1])
        arr[i].dir = ctypes.pointer(views[2]) if views[2] is not None else None
        arr[i].iou = ctypes.pointer(views[3]) if views[3] is not None else None
        arr[i].anchors = an.data_ptr()
        arr[i].transform4x4_host = ctypes.cast(T, ctypes.POINTER(ctypes.c_float))
    dev = cavs[0]["anchors"].device
    if buffers is None:
        buffers = PostprocessBuffers(H * n, W, A, top, dev)
    assert (buffers.H, buffers.W, buffers.A, buffers.top) == (H * n, W, A, top)
    rng = _box_range_f32(gt_range) if gt_range is not None else None
    with _Prof("box_decode_nms", 0):
        _call("heal_box_decode_nms_multi", arr, n, H, W, A, float(score_threshold), float(np.float32(dir_offset)), int(num_bins),
              1 if order == "hwl" else 0, float(nms_threshold), int(top), rng,
              _p(buffers.boxes), _p(buffers.scores), _p(buffers.count), _p(buffers.stats),
              _p(buffers.workspace), buffers.workspace.numel())
    return buffers


def _late_heads(t, name: str) -> Act:
    """box_decode_nms_late's head argument: an f32 Act, or a logical (n, C, H, W) fp32 CUDA tensor."""
    if isinstance(t, Act):
        if t.fmt != "f32":
            raise ValueError(f"{name}: the late decode reads fp32 heads, got an Act in '{t.fmt}'")
        return t
    if not isinstance(t, torch.Tensor) or t.dim() != 4 or t.dtype != torch.float32:
        raise ValueError(f"{name}: expected a (n_cav, C, H, W) fp32 tensor or an f32 Act")
    return to_act(t)


@_guard
def box_decode_nms_late(cls_preds, reg_preds, dir_preds, anchors: torch.Tensor, transforms: torch.Tensor, score_threshold: float,
                        nms_threshold: float, dir_offset: float = 0.0, num_bins: int = 2, order: str = "hwl", gt_range=None,
                        top: int = 1000, buffers: Optional[PostprocessBuffers] = None, coffsets=(0, 0, 0)) -> PostprocessBuffers:
    """Late fusion of one scene on the GPU with no host sync and no host-side pose: heads of every cav as one batched map each
    ((n_cav, A, H, W) / (n_cav, 7A, H, W) / (n_cav, A*bins, H, W) or None; or f32 Acts, read from channel `coffsets`), one shared
    anchor grid (H, W, A, 7) and DEVICE transforms (n_cav, 4, 4) fp32.  Same boxes, order and scores as box_decode_nms_multi
    over the same cavs in batch order.  `buffers` may be made for more cavs (H * max_cav rows) than the call has, so that the
    graphs of several cav lists share one set (LateFusionStream)."""
    c, r = _late_heads(cls_preds, "cls_preds"), _late_heads(reg_preds, "reg_preds")
    d = _late_heads(dir_preds, "dir_preds") if dir_preds is not None else None
    oc, orr, od = (int(v) for v in coffsets)
    n, H, W = c.N, c.H, c.W
    if not (1 <= n <= 16):
        raise ValueError(f"box_decode_nms_late: {n} cavs, the call takes 1 to 16")
    _need_cuda(anchors)
    if anchors.dtype != torch.float32 or not anchors.is_contiguous() or anchors.dim() != 4 \
            or tuple(anchors.shape[:2]) != (H, W) or anchors.shape[3] != 7:
        raise ValueError(f"box_decode_nms_late: anchors must be a contiguous fp32 ({H}, {W}, A, 7) grid")
    A = anchors.shape[2]
    for name, a, off, ch in (("cls_preds", c, oc, A), ("reg_preds", r, orr, 7 * A),
                             ("dir_preds", d, od, A * int(num_bins))):
        if a is None:
            continue
        if (a.N, a.H, a.W) != (n, H, W):
            raise ValueError(f"box_decode_nms_late: {name} is {(a.N, a.H, a.W)}, cls_preds is {(n, H, W)}")
        if off < 0 or off + ch > a.C:
            raise ValueError(f"box_decode_nms_late: {name} needs {ch} channels from offset {off}, it has {a.C}")
    if not isinstance(transforms, torch.Tensor) or not transforms.is_cuda or transforms.dtype != torch.float32 \
            or tuple(transforms.shape) != (n, 4, 4) or not transforms.is_contiguous():
        raise ValueError(f"box_decode_nms_late: transforms must be a contiguous ({n}, 4, 4) fp32 CUDA tensor")
    if buffers is None:
        buffers = PostprocessBuffers(H * n, W, A, top, anchors.device)
    if (buffers.W, buffers.A, buffers.top) != (W, A, top) or buffers.H < H * n:     # the C ABI checks the workspace bytes too
        raise ValueError(f"box_decode_nms_late: buffers were made for another geometry: H {buffers.H}, W {buffers.W}, A "
                         f"{buffers.A}, top {buffers.top}; {n} cavs need H >= {H * n}, W {W}, A {A}, top {top}")
    rng = _box_range_f32(gt_range) if gt_range is not None else None
    with _Prof("box_decode_nms", 0):
        _call("heal_box_decode_nms_late", c.view(oc), r.view(orr), d.view(od) if d is not None else None, _p(anchors),
              _p(transforms), n, H, W, A, float(score_threshold), float(np.float32(dir_offset)), int(num_bins),
              1 if order == "hwl" else 0, float(nms_threshold), int(top), rng,
              _p(buffers.boxes), _p(buffers.scores), _p(buffers.count), _p(buffers.stats),
              _p(buffers.workspace), buffers.workspace.numel())
    return buffers


# ------------------------------------------------------------------------------------------------
# detection evaluation (csrc/eval.cu): the TP / FP matching of eval_utils.caluclate_tp_fp for one frame
# ------------------------------------------------------------------------------------------------
class EvalBuffers:
    """Caller-owned outputs + workspace of heal_eval_tp_fp and heal_eval_tp_fp_counted, reusable for every frame of at most K
    detections and G GT boxes (the capacities of eval_tp_fp_counted).  The outputs of a call share one byte buffer, `packed` =
    [status int32 | K sorted scores fp32 | (n_thr, K) TP flags uint8] (K: the frame's count for eval_tp_fp, the detection
    capacity for eval_tp_fp_counted), so one device-to-host copy brings all three back (`unpack`)."""

    def __init__(self, K: int, G: int, device):
        self.K, self.G = int(K), int(G)
        nbytes = int(lib.heal_eval_workspace(self.K, self.G))
        if nbytes == 0:
            raise ValueError(f"bad evaluation sizes K={K}, G={G}")
        self.workspace = torch.empty((nbytes,), dtype=torch.uint8, device=device)
        self.out = torch.empty((4 + 4 * self.K + 8 * self.K,), dtype=torch.uint8, device=device)
        self._bind(0, 1)

    def _bind(self, K: int, n_thr: int):
        n = 4 + 4 * K + n_thr * K
        self.packed = self.out[:n]
        self.status = self.out[:4].view(torch.int32)
        self.scores = self.out[4:4 + 4 * K].view(torch.float32)
        self.tp = self.out[4 + 4 * K:n].view(n_thr, K)

    @staticmethod
    def unpack(packed: torch.Tensor, K: int, n_thr: int):
        """`packed` (a copy of .packed, on any device) -> (status int, scores (K,) fp32, tp (n_thr, K) uint8)."""
        return (int(packed[:4].view(torch.int32)[0]), packed[4:4 + 4 * K].view(torch.float32),
                packed[4 + 4 * K:4 + 4 * K + n_thr * K].view(n_thr, K))


def _eval_boxes(t, name: str) -> torch.Tensor:
    if not isinstance(t, torch.Tensor) or t.dtype != torch.float32 or t.dim() != 3 or tuple(t.shape[1:]) != (8, 3):
        raise ValueError(f"eval_tp_fp: {name} must be a (N, 8, 3) fp32 tensor")
    _need_cuda(t)
    if not t.is_contiguous():
        raise ValueError(f"eval_tp_fp: {name} must be contiguous")
    return t


@_guard
def eval_tp_fp(det: torch.Tensor, scores: torch.Tensor, gt: torch.Tensor, thresholds: Sequence[float],
               buffers: Optional[EvalBuffers] = None) -> EvalBuffers:
    """eval_utils.caluclate_tp_fp for one frame at up to 8 IoU thresholds, on the GPU with no host sync: det (K, 8, 3), scores (K,)
    and gt (G, 8, 3) fp32 CUDA tensors.  Returns the buffers with .scores (K,) fp32 in descending order (ties by ascending index),
    .tp (n_thr, K) uint8 flags in that order (FP = 1 - TP) and .status (1,) int32 (bit HEAL_EVAL_ZERO_UNION = 1: a union of area
    0, where the reference raises ZeroDivisionError).  The rules are those of include/heal_b200.h.  Buffers too small for K or G
    are replaced by larger ones: keep the returned object for the next frame."""
    _eval_boxes(det, "det")
    _eval_boxes(gt, "gt")
    K, G = det.shape[0], gt.shape[0]
    if not isinstance(scores, torch.Tensor) or scores.dtype != torch.float32 or tuple(scores.shape) != (K,) \
            or not scores.is_contiguous():
        raise ValueError(f"eval_tp_fp: scores must be a contiguous ({K},) fp32 tensor")
    _need_cuda(scores)
    if scores.device != det.device or gt.device != det.device:
        raise ValueError("eval_tp_fp: det, scores and gt must be on one device")
    thr = [float(v) for v in thresholds]
    if buffers is None or buffers.K < K or buffers.G < G:
        buffers = EvalBuffers(max(K, buffers.K if buffers else 0), max(G, buffers.G if buffers else 0), det.device)
    with _Prof("eval_tp_fp", 0, 24.0 * 4 * (K + G) + 4.0 * K * G * (1 + len(thr)) + (4.0 + len(thr)) * K):
        _call("heal_eval_tp_fp", _p(det), _p(scores), K, _p(gt), G, _host_f32(thr), len(thr), _p(buffers.out[4:]),
              _p(buffers.out[4 + 4 * K:]), _p(buffers.out), _p(buffers.workspace), buffers.workspace.numel())
    buffers._bind(K, len(thr))
    return buffers


def _eval_count(t, name: str) -> torch.Tensor:
    if not isinstance(t, torch.Tensor) or t.dtype != torch.int32 or tuple(t.shape) != (1,):
        raise ValueError(f"eval_tp_fp_counted: {name} must be a (1,) int32 tensor")
    _need_cuda(t)
    return t


@_guard
def eval_tp_fp_counted(det: torch.Tensor, scores: torch.Tensor, count: torch.Tensor, gt: torch.Tensor, gt_count: torch.Tensor,
                       thresholds: Sequence[float], buffers: Optional[EvalBuffers] = None) -> EvalBuffers:
    """eval_tp_fp with the live sizes on the device, capture-safe (no host read): det (K_cap, 8, 3) and scores (K_cap,) of which
    the first `count[0]` rows are live (e.g. PostprocessBuffers.boxes / .scores / .count), gt (G_cap, 8, 3) of which the first
    `gt_count[0]` rows are live; count and gt_count (1,) int32 CUDA tensors.  Returns the buffers, bound at capacity: .packed =
    [status | K_cap sorted scores | (n_thr, K_cap) flags], of which the first K scores and flags of each threshold are the frame's
    (EvalBuffers.unpack(packed, K_cap, n_thr)).  A count above its capacity sets status bit HEAL_EVAL_OVER_CAPACITY = 2 and
    writes no score or flag.  `buffers` (EvalBuffers(K, G) with K >= K_cap and G >= G_cap) are made when None; a captured graph
    passes its own."""
    _eval_boxes(det, "det")
    _eval_boxes(gt, "gt")
    K, G = det.shape[0], gt.shape[0]
    if not isinstance(scores, torch.Tensor) or scores.dtype != torch.float32 or tuple(scores.shape) != (K,) \
            or not scores.is_contiguous():
        raise ValueError(f"eval_tp_fp_counted: scores must be a contiguous ({K},) fp32 tensor")
    _need_cuda(scores)
    _eval_count(count, "count")
    _eval_count(gt_count, "gt_count")
    if any(t.device != det.device for t in (scores, count, gt, gt_count)):
        raise ValueError("eval_tp_fp_counted: det, scores, count, gt and gt_count must be on one device")
    thr = [float(v) for v in thresholds]
    if buffers is None:
        buffers = EvalBuffers(K, G, det.device)
    if buffers.K < K or buffers.G < G:
        raise ValueError(f"eval_tp_fp_counted: buffers for K={buffers.K}, G={buffers.G}, the capacities are K={K}, G={G}")
    with _Prof("eval_tp_fp", 0, 24.0 * 4 * (K + G) + 4.0 * K * G * (1 + len(thr)) + (4.0 + len(thr)) * K):
        _call("heal_eval_tp_fp_counted", _p(det), _p(scores), _p(count), K, _p(gt), _p(gt_count), G, _host_f32(thr), len(thr),
              _p(buffers.out[4:]), _p(buffers.out[4 + 4 * K:]), _p(buffers.out), _p(buffers.workspace),
              buffers.workspace.numel())
    buffers._bind(K, len(thr))
    return buffers
