"""Fusion operator mirrors of opencood/models/fuse_modules/fusion_in_one.py: AttFusion (:126-151), MaxFusion (:87-124) and
V2VNetFusion (:203-318), with the reference's `forward(x, record_len, affine_matrix)` signature (NCHW) and `forward_nhwc`
(conv-engine activations).  DiscoFusion cannot be constructed in the reference (it imports a `disco_fuse` module the reference
does not ship); V2X-ViT, CoBEVT, Where2comm and Who2com are out of scope (SURVEY.md 2.1 row 14)."""
import numpy as np
import torch
import torch.nn as nn

from ... import engine, ops
from ...engine import conv_bn_act


def regroup(x, record_len):
    cum = torch.cumsum(record_len, dim=0)
    return torch.tensor_split(x, cum[:-1].cpu())


def _rl(record_len):
    return [int(v) for v in (record_len.tolist() if torch.is_tensor(record_len) else record_len)]


class ScaledDotProductAttention(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.sqrt_dim = np.sqrt(dim)

    def forward(self, query, key, value):
        raise NotImplementedError("executed fused inside AttFusion (heal_att_fuse)")


class AttFusion(nn.Module):
    def __init__(self, feature_dims):
        super().__init__()
        self.att = ScaledDotProductAttention(feature_dims)
        self.feature_dims = feature_dims

    def forward_nhwc(self, x, record_len, affine_matrix):
        """x: Act (sumN,H,W,C) -> Act (B,H,W,C)"""
        rl = _rl(record_len)
        out = ops.act_empty(len(rl), x.H, x.W, x.C, x.fmt, x.device)
        aff = affine_matrix.to(device=x.device, dtype=torch.float64)
        start = 0
        for b, n in enumerate(rl):
            ops.att_fuse(x.images(start, start + n), aff[b, 0, :n].contiguous(), out=out.image(b))
            start += n
        return out

    def forward(self, xx, record_len, affine_matrix):
        return ops.act_to_nchw(self.forward_nhwc(ops.to_act(xx), record_len, affine_matrix))


class MaxFusion(nn.Module):
    """F-Cooper (fusion_in_one.py:87-124): per scene, max over agents of every agent's map warped to the ego (heal_max_fuse)."""

    def forward_nhwc(self, x, record_len, affine_matrix):
        """x: Act (sumN,H,W,C) -> Act (B,H,W,C)"""
        rl = _rl(record_len)
        out = ops.act_empty(len(rl), x.H, x.W, x.C, x.fmt, x.device)
        aff = affine_matrix.to(device=x.device, dtype=torch.float64)
        start = 0
        for b, n in enumerate(rl):
            ops.max_fuse(x.images(start, start + n), aff[b, 0, :n].contiguous(), out=out.image(b))
            start += n
        return out

    def forward(self, x, record_len, affine_matrix):
        return ops.act_to_nchw(self.forward_nhwc(ops.to_act(x), record_len, affine_matrix))


class ConvGRUCell(nn.Module):
    """Parameter container of sub_modules/convgru.py:7-68 (keys conv_gates.*, conv_can.*).  V2VNetFusion runs it with a zero
    hidden state, through its own stacked conv + heal_gru_gate."""

    def __init__(self, input_size, input_dim, hidden_dim, kernel_size, bias):
        super().__init__()
        self.height, self.width = input_size
        self.padding = kernel_size[0] // 2, kernel_size[1] // 2
        self.hidden_dim = hidden_dim
        self.bias = bias
        self.conv_gates = nn.Conv2d(input_dim + hidden_dim, 2 * hidden_dim, kernel_size=kernel_size, padding=self.padding, bias=bias)
        self.conv_can = nn.Conv2d(input_dim + hidden_dim, hidden_dim, kernel_size=kernel_size, padding=self.padding, bias=bias)


class ConvGRU(nn.Module):
    """Parameter container of sub_modules/convgru.py:71-198: `cell_list.<i>.*` keys."""

    def __init__(self, input_size, input_dim, hidden_dim, kernel_size, num_layers, batch_first=False, bias=True,
                 return_all_layers=False):
        super().__init__()
        kernel_size = kernel_size if isinstance(kernel_size, list) else [kernel_size] * num_layers
        hidden_dim = hidden_dim if isinstance(hidden_dim, list) else [hidden_dim] * num_layers
        if not len(kernel_size) == len(hidden_dim) == num_layers:
            raise ValueError('Inconsistent list length.')
        self.height, self.width = input_size
        self.input_dim, self.hidden_dim, self.kernel_size, self.num_layers = input_dim, hidden_dim, kernel_size, num_layers
        self.batch_first, self.bias, self.return_all_layers = batch_first, bias, return_all_layers
        self.cell_list = nn.ModuleList([
            ConvGRUCell((self.height, self.width), input_dim if i == 0 else hidden_dim[i - 1], hidden_dim[i], kernel_size[i], bias)
            for i in range(num_layers)])


def _conv_from(weight, bias, padding):
    """A stand-alone Conv2d holding derived weights (not a registered submodule; the conv engine packs it like any other)."""
    cout, cin, kh, kw = weight.shape
    c = nn.Conv2d(cin, cout, (kh, kw), padding=padding, bias=bias is not None, device=weight.device)
    with torch.no_grad():
        c.weight.copy_(weight)
        if bias is not None:
            c.bias.copy_(bias)
    return c.eval()


class V2VNetFusion(nn.Module):
    """V2VNet (fusion_in_one.py:203-318) with the reference's ctor, submodule names and state-dict keys.

    The forward computes what the reference computes, up to fp32 reassociation, with three exact shortcuts:
      1. ConvGRU is called on a length-1 sequence with hidden_state=None, so h = 0 on every call and the cell reduces to
         h' = sigmoid(z) * tanh(c) with z = conv_gates(cat[in, 0])[C:2C] (update gate) and c = conv_can(cat[in, 0]).  Only
         the input columns [:, :2C] of both convs and the update-gate rows of conv_gates are live: they are stacked into ONE
         3x3 conv 2C -> 2C, followed by heal_gru_gate.
      2. msg_cnn(cat[warp(x_j), x_i]) = W[:, :C] (*) warp(x_j) + (W[:, C:] (*) x_i + b): the second term depends on i only
         and is computed once per node (P), the first once per pair (Q), as one multi-image conv over all pairs.
      3. Only node 0 of every scene is read after the last iteration, so the last iteration updates node 0 alone.
    One iteration: warp stack (heal_warp_affine) -> Q conv -> P conv -> heal_v2v_aggregate -> GRU conv -> heal_gru_gate.
    The packed weights are a derived cache, rebuilt when a source parameter changes."""

    def __init__(self, args):
        super().__init__()
        in_channels = args['in_channels']
        H, W = args['conv_gru']['H'], args['conv_gru']['W']
        kernel_size = args['conv_gru']['kernel_size']
        num_gru_layers = args['conv_gru']['num_layers']
        self.num_iteration = args['num_iteration']
        self.gru_flag = args['gru_flag']
        self.agg_operator = args['agg_operator']
        if self.agg_operator not in ("avg", "max"):
            raise ValueError("agg_operator has wrong value")
        self.H, self.W, self.in_channels = H, W, in_channels
        self.msg_cnn = nn.Conv2d(in_channels * 2, in_channels, kernel_size=3, stride=1, padding=1)
        self.conv_gru = ConvGRU(input_size=(H, W), input_dim=in_channels * 2, hidden_dim=[in_channels] * num_gru_layers,
                                kernel_size=kernel_size, num_layers=num_gru_layers, batch_first=True, bias=True,
                                return_all_layers=False)
        self.mlp = nn.Linear(in_channels, in_channels)
        self._derived = None

    def _check(self, C, H, W):
        if (H, W) != (self.H, self.W):
            raise ValueError(f"V2VNetFusion: conv_gru H/W is {(self.H, self.W)} but the fused feature map is {(H, W)}; "
                             "the reference fails in torch.cat for this config")
        if C != self.in_channels:
            raise ValueError(f"V2VNetFusion: in_channels is {self.in_channels} but the feature map has {C} channels")
        if self.gru_flag and self.conv_gru.num_layers != 1:
            raise NotImplementedError("V2VNetFusion: only conv_gru.num_layers == 1 is implemented (every shipped config)")

    def _packed(self):
        cell = self.conv_gru.cell_list[0]
        sig = engine._sig(self.msg_cnn, cell.conv_gates, cell.conv_can, self.mlp)
        if self._derived is None or self._derived[0] != sig:
            C = self.in_channels
            w, b = self.msg_cnn.weight.detach(), self.msg_cnn.bias.detach()
            nbr = _conv_from(w[:, :C], None, 1)                     # Q: applied to the warped neighbour
            node = _conv_from(w[:, C:], b, 1)                       # P: applied to x_i, carries the bias
            g, cc = cell.conv_gates, cell.conv_can
            gw = torch.cat([g.weight.detach()[C:2 * C, :2 * C], cc.weight.detach()[:, :2 * C]], 0)
            gb = torch.cat([g.bias.detach()[C:2 * C], cc.bias.detach()], 0) if cell.bias else None
            gru = _conv_from(gw, gb, cell.padding)
            mlp = _conv_from(self.mlp.weight.detach()[:, :, None, None], self.mlp.bias.detach(), 0)
            self._derived = (sig, nbr, node, gru, mlp)
        return self._derived[1:]

    def forward_nhwc(self, x, record_len, affine_matrix):
        """x: Act (sumN,H,W,C) -> Act (B,H,W,C).  Reads record_len on the host (as AttFusion does); no other sync."""
        self._check(x.C, x.H, x.W)
        nbr, node, gru, mlp = self._packed()
        rl = _rl(record_len)
        B, C, H, W = len(rl), x.C, x.H, x.W
        starts = [sum(rl[:b]) for b in range(B)]
        aff = affine_matrix.to(device=x.device, dtype=torch.float64)
        agg_max = self.agg_operator == "max"
        for it in range(self.num_iteration):
            last = it == self.num_iteration - 1
            # pair rows: scene b, updated node i, neighbour j (all nodes; node 0 alone in the last iteration)
            src, nodes, th = [], [], []
            for b, n in enumerate(rl):
                s0 = starts[b]
                upd = 1 if last else n
                for i in range(upd):
                    nodes.append((s0 + i, b if last else s0 + i, len(src), n))
                    src.extend(s0 + j for j in range(n))
                th.append(aff[b, :upd, :n].reshape(upd * n, 2, 3))
            th = torch.cat(th, 0)
            warped = ops.warp_affine(x, src, th, out_fmt=engine.act_fmt())
            q = conv_bn_act(warped, nbr)
            del warped
            if last:
                p = ops.act_empty(B, H, W, C, engine.act_fmt(), x.device)
                for b in range(B):
                    conv_bn_act(x.image(starts[b]), node, out=p.image(b))
            else:
                p = conv_bn_act(x, node)
            if self.gru_flag:
                cat = ops.v2v_aggregate(q, p, x, th, nodes, agg_max, gru=True, out_fmt=engine.act_fmt())
                del q, p
                x = ops.gru_gate(conv_bn_act(cat, gru))
            else:
                x = ops.v2v_aggregate(q, p, x, th, nodes, agg_max, gru=False, out_fmt=engine.act_fmt())
        if self.num_iteration == 0:
            ego = ops.act_empty(B, H, W, C, x.fmt, x.device)
            for b in range(B):
                ego.image(b).t.copy_(x.image(starts[b]).t)
            x = ego
        return conv_bn_act(x, mlp)

    def forward(self, x, record_len, affine_matrix):
        self._check(*x.shape[1:])
        return ops.act_to_nchw(self.forward_nhwc(ops.to_act(x), record_len, affine_matrix))
