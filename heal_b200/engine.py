"""Execution helpers shared by the mirror modules: precision mode, parameter folding/packing cache and
the conv dispatcher (wgmma implicit GEMM where eligible, fp32 CUDA-core kernel otherwise).

Parameters stay ordinary nn.Parameters with the reference's state-dict key names
(SURVEY.md 8b "Parameters / ownership"); what the kernels consume is a *derived* cache (BN folded in
fp64, weights re-laid out for the kernels) that is rebuilt whenever a source tensor's version counter
changes (load_state_dict / optimizer step) or the module moves device.

Precision modes (set_precision):
  'tc32'  (default) dense stride-1 convs on wgmma with split-bf16 operands (3 MMAs / K-step, fp32
          accumulate: fp32-equivalent, meets the 1e-3 parity bar); activations stored as split-bf16.
  'bf16'  same kernels, activations stored as ONE bf16 plane, weights keep both planes (a_hi x [b_hi | b_lo]: the weights are
          not rounded to 8 mantissa bits, only the activations are; 1e-2 parity bar, BASELINE config 4).  HEAL_BF16_WEIGHTS=1
          rounds the weights too (plain bf16 x bf16, for A/B measurements).
  'fp32'  everything on the fp32 CUDA-core kernels with fp32 storage (exact-fp32 cross-check path).
"""
from __future__ import annotations

import weakref
from typing import Optional

import torch
import torch.nn as nn

from . import ops
from .ops import Act

PRECISION = "tc32"
SPARSE_STEM = True     # PointPillars: feed the first stride-2 residual block from the pillar list (no dense canvas)
# mma.sync variant of the sparse stem (heal_sparse_stem_tc): correct and tested, but not faster than the fp32 gather kernel on LiDAR
# occupancy (0.22 vs 0.20 ms: a 16-pixel row block has 1-2 hit rows per tap, so ~90 % of each MMA multiplies zeros) -> opt-in.
import os as _os
STEM_TC = _os.environ.get("HEAL_STEM_TC", "0") == "1"
BF16_WEIGHTS = _os.environ.get("HEAL_BF16_WEIGHTS", "0") == "1"


def set_precision(mode: str):
    global PRECISION
    assert mode in ("tc32", "bf16", "fp32")
    PRECISION = mode


def act_fmt() -> str:
    return {"tc32": "split", "bf16": "bf16", "fp32": "f32"}[PRECISION]


_CACHE = weakref.WeakKeyDictionary()


def _sig(*mods):
    sig = []
    for m in mods:
        if m is None:
            sig.append(None)
            continue
        for t in list(m.parameters(recurse=False)) + list(m.buffers(recurse=False)):
            sig.append((t.data_ptr(), t._version, str(t.device)))
    return tuple(sig)


def packed(conv: nn.Module, bn: Optional[nn.Module], relu: bool, extra_pad: int = 0, kind: str = "simt"):
    """Folded + packed weights for `conv` (+ eval `bn`) on conv.weight's device, cached per (module, kind)."""
    sig = (_sig(conv, bn), relu, extra_pad)
    slot = _CACHE.setdefault(conv, {})
    hit = slot.get(kind)
    if hit is not None and hit[0] == sig:
        return hit[1]
    if kind == "simt":
        pc = ops.pack_deconv(conv, bn, relu) if isinstance(conv, nn.ConvTranspose2d) else ops.pack_conv(conv, bn, relu, extra_pad)
    elif kind == "simt_cin4":
        pc = ops.pack_conv(conv, bn, relu, extra_pad, cin_to=(conv.in_channels + 3) // 4 * 4)
    elif kind == "narrow":
        pc = ops.pack_conv3x3_narrow(conv, bn, relu)
    elif kind == "tc2_cin64":
        pc = ops.pack_conv_tc(conv, bn, relu, planes=2, extra_pad=extra_pad, cin_to=(conv.in_channels + 63) // 64 * 64)
    else:
        pc = ops.pack_conv_tc(conv, bn, relu, planes=2 if kind == "tc2" else 1, extra_pad=extra_pad)
    pc.to(conv.weight.device)
    slot[kind] = (sig, pc)
    return pc


def require_eval(module: nn.Module):
    if module.training:
        raise NotImplementedError(
            f"{type(module).__name__}: the heal_b200 kernels implement the inference path "
            "(model.eval(), torch.no_grad()); autograd through them is a 'next' row (SURVEY.md 8f-4).")


def conv_bn_act(x: Act, conv, bn=None, relu=False, residual: Optional[Act] = None, out: Optional[Act] = None,
                out_coffset: int = 0, extra_pad: int = 0, out_fmt: Optional[str] = None) -> Act:
    """conv(+bn)(+residual)(+relu) as ONE kernel.  `out_fmt` defaults to the mode's activation format;
    pass 'f32' for tensors that leave the conv engine (occupancy logits, prediction heads)."""
    fmt = act_fmt()
    if isinstance(x, ops.SparseCanvas):
        x = x.dense(fmt)
    if out is not None:
        out_fmt = out.fmt
    elif out_fmt is None:
        out_fmt = fmt
    if PRECISION != "fp32" and ops.tc_eligible(conv):
        if x.fmt != fmt:
            x = ops.convert(x, fmt)
        if residual is not None and residual.fmt not in ("f32", fmt):
            residual = ops.convert(residual, fmt)
        pc = packed(conv, bn, relu, extra_pad, kind="tc1" if (PRECISION == "bf16" and BF16_WEIGHTS) else "tc2")
        if out_fmt == "f32":
            _, o32 = ops.conv2d_tc(x, pc, residual=residual, want_split=False, out_f32=out, want_f32=True,
                                   out32_coffset=out_coffset)
            return o32
        o, _ = ops.conv2d_tc(x, pc, residual=residual, out=out, out_coffset=out_coffset)
        return o
    pc = packed(conv, bn, relu, extra_pad, kind="simt")
    return ops.conv2d_simt(x, pc, residual=residual, out=out, out_fmt=out_fmt, out_coffset=out_coffset)
