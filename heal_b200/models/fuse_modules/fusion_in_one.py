"""Fusion operator mirrors of opencood/models/fuse_modules/fusion_in_one.py: AttFusion (:126-151), MaxFusion (:87-124),
V2VNetFusion (:203-318), V2XViTFusion (:320-372), CoBEVT (:374-429), Where2commFusion (:431-484) and Who2comFusion (:486-539),
with the reference's `forward(x, record_len, affine_matrix)` signature (NCHW) and `forward_nhwc` (conv-engine activations).
DiscoFusion cannot be constructed in the reference (it imports a `disco_fuse` module the reference does not ship)."""
import numpy as np
import torch
import torch.nn as nn

from ... import engine, ops
from ...engine import conv_bn_act, require_eval
from .swap_fusion_modules import SwapFusionBlockMask


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


class CoBEVT(nn.Module):
    """CoBEVT (fusion_in_one.py:374-429) with the reference's ctor and state-dict keys (`layers.{i}.{window,grid}_{attention,ffd}`,
    `mlp_head.2` LayerNorm, `mlp_head.3` Linear; the einops layers of mlp_head are nn.Identity so the indices match).

    Per scene the n_b agents are warped to the ego into slots b*L .. b*L+n_b-1 of a zeroed (B*L, H, W, C) map (heal_warp_affine;
    the padded slots stay zero).  Every pre-norm residual sub-layer is then
        attention: LayerNorm (heal_mean_layernorm) -> to_qkv 1x1 conv (q rows pre-scaled by dim_head^-0.5 in fp64)
                   -> heal_swap_attention (window, then grid) -> to_out 1x1 conv + residual
        FFN:       LayerNorm -> 1x1 conv + bias + GELU -> 1x1 conv + bias + residual
    and mlp_head is heal_mean_layernorm over all L slots (padded ones included, as the reference's Reduce-mean) -> 1x1 conv.
    Padded slots are queries (they become non-zero after the first block); only their keys are masked.  The packed weights and
    the dense relative-position bias are a derived cache, rebuilt when a parameter or the index buffer changes."""

    def __init__(self, args):
        super().__init__()
        self.layers = nn.ModuleList([])
        self.depth = args['depth']
        input_dim = args['input_dim']
        mlp_dim = args['mlp_dim']
        agent_size = args['agent_size']
        window_size = args['window_size']
        drop_out = args['drop_out']
        dim_head = args['dim_head']
        for _ in range(self.depth):
            self.layers.append(SwapFusionBlockMask(input_dim, mlp_dim, dim_head, window_size, agent_size, drop_out))
        self.mlp_head = nn.Sequential(nn.Identity(), nn.Identity(), nn.LayerNorm(input_dim), nn.Linear(input_dim, input_dim),
                                      nn.Identity())
        self.input_dim, self.agent_size, self.window_size, self.dim_head = input_dim, agent_size, window_size, dim_head
        self._derived = None

    def _check(self, C, H, W, L):
        if L != self.agent_size:
            raise ValueError(f"CoBEVT: the affine matrix has L = {L} agent slots but agent_size is {self.agent_size}; the "
                             "reference's relative position bias is sized by agent_size and fails for any other L")
        if H % self.window_size or W % self.window_size:
            raise ValueError(f"CoBEVT: the feature map {(H, W)} is not divisible by window_size {self.window_size}; the "
                             "reference's window rearrange fails for this shape")
        if C != self.input_dim:
            raise ValueError(f"CoBEVT: input_dim is {self.input_dim} but the feature map has {C} channels")
        if self.dim_head != 32:
            raise NotImplementedError(f"CoBEVT: heal_swap_attention implements dim_head 32 (every shipped config), not {self.dim_head}")
        if L * self.window_size ** 2 > 128:
            raise NotImplementedError(f"CoBEVT: heal_swap_attention implements windows of at most 128 tokens, not "
                                      f"agent_size * window_size^2 = {L * self.window_size ** 2}")

    def _packed(self):
        sig = engine._sig(*self.modules())
        if self._derived is None or self._derived[0] != sig:
            blocks = []
            for blk in self.layers:
                parts = []
                for att, ffd in ((blk.window_attention, blk.window_ffd), (blk.grid_attention, blk.grid_ffd)):
                    a = att.fn
                    C = a.to_qkv.in_features
                    wq = a.to_qkv.weight.detach().double()
                    wq = torch.cat([wq[:C] * a.scale, wq[C:]]).float()
                    qkv = _conv_from(wq[:, :, None, None], None, 0)
                    out = _conv_from(a.to_out[0].weight.detach()[:, :, None, None], None, 0)
                    # key-major dense bias: bias[h, j, i] = table[index[i, j], h]
                    bias = a.relative_position_bias_table.weight.detach()[a.relative_position_index]
                    bias = bias.permute(2, 1, 0).float().contiguous()
                    l1, l2 = ffd.fn.net[0], ffd.fn.net[3]
                    f1 = _conv_from(l1.weight.detach()[:, :, None, None], l1.bias.detach(), 0)
                    f2 = _conv_from(l2.weight.detach()[:, :, None, None], l2.bias.detach(), 0)
                    parts.append((att.norm, qkv, bias, out, ffd.norm, f1, f2))
                blocks.append(parts)
            lin = self.mlp_head[3]
            head = _conv_from(lin.weight.detach()[:, :, None, None], lin.bias.detach(), 0)
            self._derived = (sig, blocks, head)
        return self._derived[1:]

    def forward_nhwc(self, x, record_len, affine_matrix):
        """x: Act (sumN,H,W,C), affine_matrix (B,L,L,2,3) -> Act (B,H,W,C).  Reads record_len on the host; no other sync."""
        require_eval(self)
        rl = _rl(record_len)
        B, L = affine_matrix.shape[:2]
        C, H, W = x.C, x.H, x.W
        self._check(C, H, W, L)
        if len(rl) != B or any(n < 1 or n > L for n in rl):
            raise ValueError(f"CoBEVT: record_len {rl} does not fit {B} scenes of at most {L} agents")
        blocks, head = self._packed()
        fmt = engine.act_fmt()
        aff = affine_matrix.to(device=x.device, dtype=torch.float64)
        X = ops.act_empty(B * L, H, W, C, fmt, x.device)
        start = 0
        for b, n in enumerate(rl):
            ops.warp_affine(x, range(start, start + n), aff[b, 0, :n].contiguous(), out=X.images(b * L, b * L + n))
            if n < L:
                X.images(b * L + n, (b + 1) * L).t.zero_()
            start += n
        w = self.window_size
        for parts in blocks:
            for grid, (norm, qkv, bias, out, fnorm, f1, f2) in enumerate(parts):
                y = ops.mean_layernorm(X, 1, norm.weight, norm.bias, norm.eps, out_fmt=fmt)
                a = ops.swap_attention(conv_bn_act(y, qkv), rl, L, w, bool(grid), bias, out_fmt=fmt)
                X = conv_bn_act(a, out, residual=X)
                y = ops.mean_layernorm(X, 1, fnorm.weight, fnorm.bias, fnorm.eps, out_fmt=fmt)
                X = conv_bn_act(conv_bn_act(y, f1, relu=2), f2, residual=X)
        ln = self.mlp_head[2]
        y = ops.mean_layernorm(X, L, ln.weight, ln.bias, ln.eps, out_fmt=fmt)
        return conv_bn_act(y, head)

    def forward(self, x, record_len, affine_matrix):
        require_eval(self)
        self._check(x.shape[1], x.shape[2], x.shape[3], affine_matrix.shape[1])
        return ops.act_to_nchw(self.forward_nhwc(ops.to_act(x), record_len, affine_matrix))


class EncodeLayer(nn.Module):
    """Parameter container of where2comm_attn.py:64-103 (keys attn.{in_proj_weight, in_proj_bias, out_proj.*}, linear{1,2}.*,
    norm{1,2}.*); Where2commFusion runs it."""

    def __init__(self, channels, n_head=8, dropout=0):
        super().__init__()
        self.attn = nn.MultiheadAttention(channels, n_head, dropout)
        self.linear1 = nn.Linear(channels, channels)
        self.linear2 = nn.Linear(channels, channels)
        self.norm1 = nn.LayerNorm(channels)
        self.norm2 = nn.LayerNorm(channels)


def _linear_conv(lin):
    return _conv_from(lin.weight.detach()[:, :, None, None], None if lin.bias is None else lin.bias.detach(), 0)


class Where2commFusion(nn.Module):
    """Where2comm's fusion (fusion_in_one.py:431-484) with the reference's ctor and state-dict keys (`mha_fusion.*`).

    Per scene, EncodeLayer runs with the warped ego X_0 as the one query over the n_b warped agents X_j, per pixel:
    y1 = LN1(X_0 + out_proj(MHA)), out = LN2(y1 + linear2(ReLU(linear1(y1)))).  The k | v in-projection commutes with the
    warp, so it runs as one bias-free 1x1 conv on the UNWARPED maps and heal_ego_mha samples it (adding the bias afterwards):
        warp the egos (heal_warp_affine) -> q 1x1 conv (+ b_q) -> k|v 1x1 conv on x -> heal_ego_mha
        -> out_proj 1x1 conv + X_0 -> heal_mean_layernorm -> linear1 + ReLU -> linear2 + y1 -> heal_mean_layernorm.
    The packed convs and the k|v bias are a derived cache, rebuilt when a parameter changes."""

    def __init__(self, feature_dims):
        super().__init__()
        self.mha_fusion = EncodeLayer(feature_dims)
        self.feature_dims = feature_dims
        self._derived = None

    def _check(self, C):
        if C != self.feature_dims:
            raise ValueError(f"Where2commFusion: feature_dims is {self.feature_dims} but the feature map has {C} channels")
        if C != 256 or self.mha_fusion.attn.num_heads != 8:
            raise NotImplementedError(f"Where2commFusion: heal_ego_mha implements 256 channels in 8 heads (every shipped "
                                      f"config), not {C}")

    def _packed(self):
        enc = self.mha_fusion
        sig = engine._sig(*enc.modules())
        if self._derived is None or self._derived[0] != sig:
            C = self.feature_dims
            w, b = enc.attn.in_proj_weight.detach(), enc.attn.in_proj_bias.detach()
            q = _conv_from(w[:C, :, None, None], b[:C], 0)
            kv = _conv_from(w[C:, :, None, None], None, 0)
            kv_bias = b[C:].float().contiguous()
            self._derived = (sig, q, kv, kv_bias, _linear_conv(enc.attn.out_proj), _linear_conv(enc.linear1),
                             _linear_conv(enc.linear2))
        return self._derived[1:]

    def forward_nhwc(self, x, record_len, affine_matrix):
        """x: Act (sumN,H,W,C) -> Act (B,H,W,C).  Reads record_len on the host; no other sync."""
        require_eval(self)
        self._check(x.C)
        rl = _rl(record_len)
        if sum(rl) != x.N:
            raise ValueError(f"Where2commFusion: record_len {rl} does not sum to the {x.N} feature maps")
        q_conv, kv_conv, kv_bias, out_proj, l1, l2 = self._packed()
        enc = self.mha_fusion
        fmt = engine.act_fmt()
        aff = affine_matrix.to(device=x.device, dtype=torch.float64)
        starts = [sum(rl[:b]) for b in range(len(rl))]
        ego = ops.warp_affine(x, starts, aff[:, 0, 0].contiguous(), out_fmt=fmt)
        theta = torch.cat([aff[b, 0, :n] for b, n in enumerate(rl)])
        a = ops.ego_mha(conv_bn_act(ego, q_conv), conv_bn_act(x, kv_conv), kv_bias, theta, rl, out_fmt=fmt)
        y = conv_bn_act(a, out_proj, residual=ego)
        y1 = ops.mean_layernorm(y, 1, enc.norm1.weight, enc.norm1.bias, enc.norm1.eps, out_fmt=fmt)
        y = conv_bn_act(conv_bn_act(y1, l1, relu=True), l2, residual=y1)
        return ops.mean_layernorm(y, 1, enc.norm2.weight, enc.norm2.bias, enc.norm2.eps, out_fmt=fmt)

    def forward(self, x, record_len, affine_matrix):
        require_eval(self)
        self._check(x.shape[1])
        return ops.act_to_nchw(self.forward_nhwc(ops.to_act(x), record_len, affine_matrix))


class Who2comFusion(nn.Module):
    """Who2com's fusion (fusion_in_one.py:486-539) with the reference's ctor and state-dict keys (`decode_layer.*`).

    Per scene, a = the ego row of the parameter-free ScaledDotProductAttention(C) over the agents warped to the ego (exactly
    AttFusion, heal_att_fuse), then decode_layer(cat[x_0, a]) with x_0 the UNWARPED ego map: heal_att_fuse writes channels
    [C, 2C) of a (B,H,W,2C) map, the ego is converted into [0, C), and the 3x3 conv runs on the conv engine."""

    def __init__(self, feature_dims):
        super().__init__()
        self.att = ScaledDotProductAttention(feature_dims)
        self.decode_layer = nn.Conv2d(feature_dims * 2, feature_dims, kernel_size=3, stride=1, padding=1)
        self.feature_dims = feature_dims

    def forward_nhwc(self, x, record_len, affine_matrix):
        """x: Act (sumN,H,W,C) -> Act (B,H,W,C).  Reads record_len on the host; no other sync."""
        require_eval(self)
        C = x.C
        if C != self.feature_dims:
            raise ValueError(f"Who2comFusion: feature_dims is {self.feature_dims} but the feature map has {C} channels")
        rl = _rl(record_len)
        if sum(rl) != x.N:
            raise ValueError(f"Who2comFusion: record_len {rl} does not sum to the {x.N} feature maps")
        fmt = engine.act_fmt()
        aff = affine_matrix.to(device=x.device, dtype=torch.float64)
        cat = ops.act_empty(len(rl), x.H, x.W, 2 * C, fmt, x.device)
        ego, att = ops.Act(cat.t[..., :C], fmt), ops.Act(cat.t[..., C:], fmt)
        start = 0
        for b, n in enumerate(rl):
            ops.att_fuse(x.images(start, start + n), aff[b, 0, :n].contiguous(), out=att.image(b))
            ops.convert(x.image(start), fmt, out=ego.image(b))
            start += n
        return conv_bn_act(cat, self.decode_layer)

    def forward(self, x, record_len, affine_matrix):
        return ops.act_to_nchw(self.forward_nhwc(ops.to_act(x), record_len, affine_matrix))


_V2XVIT_SCOPE = "outside the heal_b200 hot-path scope"


class V2XViTFusion(nn.Module):
    """V2X-ViT (fusion_in_one.py:320-372) with the reference's ctor and state-dict keys (`fusion_net.encoder.layers.{i}.0.layers.0.
    {0,1}` the HGT and pyramid-window PreNorms, `.{i}.1` the FFN PreNorm, `fusion_net.encoder.prior_feed`).

    The GPU path keeps only what reaches the ego output of the reference:
      - the n_b real agents of each scene, not L padded slots: padded agents are masked as keys of the agent attention and every
        other step is per agent, so they never reach a real one.  Images are ordered egos first, then each scene's others;
      - agent types are always 0 (V2XViTFusion feeds a zero prior encoding), so HGTCavAttention is multi-head attention with
        relation_att[0] and dim_head^-0.5 folded into the q rows and relation_msg[0] into the v rows of one to_qkv 1x1 conv
        (fp64 folding); the ROI mask is all ones for the identity correction, so the key mask is the agent mask;
      - only slot 0 is read after the last agent attention, so the last layer's agent attention has ego queries only and its
        window attention, SplitAttn and FFN run on the egos.
    Per scene the agents are warped to the ego (heal_warp_affine), the others resampled by the STTF matrix (heal_sttf_resample).
    Each layer: LayerNorm -> to_qkv conv -> heal_cav_attention -> a_linears[0] conv + residual; LayerNorm -> the three branch
    to_qkv as one conv -> heal_window_attention per branch -> the three to_out convs -> heal_split_attn (+ residual);
    LayerNorm -> conv + GELU -> conv + residual.  The folded weights, dense biases and STTF matrices are a derived cache."""

    def __init__(self, args):
        super().__init__()
        from ..sub_modules.v2xvit_basic import V2XTransformer
        enc = args['transformer']['encoder']
        cav, pw = enc['cav_att_config'], enc['pwindow_att_config']
        if enc.get('use_RTE') or cav.get('use_RTE'):
            raise NotImplementedError(f"V2XViTFusion: use_RTE is {_V2XVIT_SCOPE} (no shipped config enables it)")
        if not cav['use_hetero']:
            raise NotImplementedError(f"V2XViTFusion: use_hetero false (CavAttention) is {_V2XVIT_SCOPE}")
        if pw['fusion_method'] != 'split_attn':
            raise NotImplementedError(f"V2XViTFusion: window fusion '{pw['fusion_method']}' is {_V2XVIT_SCOPE} (built: split_attn)")
        if pw['dim'] != 256 or cav['dim'] != 256:
            raise ValueError(f"V2XViTFusion: split_attn is SplitAttn(256) in the reference and needs dim 256, not "
                             f"{cav['dim']} / {pw['dim']}")
        if len(pw['window_size']) != 3:
            raise ValueError("V2XViTFusion: split_attn fuses exactly 3 window branches (the reference asserts it)")
        if cav['dim_head'] != 32:
            raise NotImplementedError(f"V2XViTFusion: heal_cav_attention implements dim_head 32, not {cav['dim_head']}")
        for ws, dh in zip(pw['window_size'], pw['dim_head']):
            if ws not in (4, 8, 16) or dh not in (16, 32, 64):
                raise NotImplementedError(f"V2XViTFusion: heal_window_attention implements windows 4/8/16 and dim_head "
                                          f"16/32/64, not window {ws} with dim_head {dh}")
        self.fusion_net = V2XTransformer(args['transformer'])
        self.dim = cav['dim']
        self.window_sizes = list(pw['window_size'])
        self._derived = None

    def _check(self, C, H, W, L):
        if C != self.dim:
            raise ValueError(f"V2XViTFusion: dim is {self.dim} but the feature map has {C} channels")
        for ws in self.window_sizes:
            if H % ws or W % ws:
                raise ValueError(f"V2XViTFusion: the feature map {(H, W)} is not divisible by window size {ws}; the "
                                 "reference's window rearrange fails for this shape")
        if L > 8:
            raise NotImplementedError(f"V2XViTFusion: heal_cav_attention implements at most 8 agents, not L = {L}")

    def _packed(self, H, W, device):
        sig = engine._sig(*self.modules())
        if self._derived is None or self._derived[0] != sig:
            layers = []
            for blk, ffn in self.fusion_net.encoder.layers:
                cav_pre, win_pre = blk.layers[0]
                a = cav_pre.fn
                dh, hd = a.dim_head, a.heads
                q, k, v = a.q_linears[0], a.k_linears[0], a.v_linears[0]
                ra = a.relation_att.detach()[0].double()                        # (heads, p, q)
                rm = a.relation_msg.detach()[0].double()
                wq = q.weight.detach().double().reshape(hd, dh, -1)
                bq = q.bias.detach().double().reshape(hd, dh)
                wv = v.weight.detach().double().reshape(hd, dh, -1)
                bv = v.bias.detach().double().reshape(hd, dh)
                # q'_m = scale * R_att[m]^T q_m, v'_m = R_msg[m]^T v_m
                wq2 = torch.einsum("mpq,mpc->mqc", ra, wq).reshape(hd * dh, -1) * a.scale
                bq2 = torch.einsum("mpq,mp->mq", ra, bq).reshape(-1) * a.scale
                wv2 = torch.einsum("mpc,mpk->mck", rm, wv).reshape(hd * dh, -1)
                bv2 = torch.einsum("mpc,mp->mc", rm, bv).reshape(-1)
                w = torch.cat([wq2, k.weight.detach().double(), wv2]).float()
                b = torch.cat([bq2, k.bias.detach().double(), bv2]).float()
                hgt_qkv = _conv_from(w[:, :, None, None], b, 0)
                al = a.a_linears[0]
                hgt_out = _conv_from(al.weight.detach()[:, :, None, None], al.bias.detach(), 0)
                pwa = win_pre.fn
                wq3, branches, outs = [], [], []
                for br in pwa.pwmsa:
                    inner = br.heads * br.dim_head
                    wt = br.to_qkv.weight.detach().double()
                    wq3.append(torch.cat([wt[:inner] * br.scale, wt[inner:]]))
                    branches.append((br.heads, br.dim_head, br.window_size, br.dense_bias().float().contiguous()))
                    lo = br.to_out[0]
                    outs.append(_conv_from(lo.weight.detach()[:, :, None, None], lo.bias.detach(), 0))
                win_qkv = _conv_from(torch.cat(wq3).float()[:, :, None, None], None, 0)
                sa = pwa.split_attn
                gate = (sa.fc1.weight.detach().float().t().contiguous(), sa.bn1, sa.fc2.weight.detach().float().t().contiguous())
                l1, l2 = ffn.fn.net[0], ffn.fn.net[3]
                f1 = _conv_from(l1.weight.detach()[:, :, None, None], l1.bias.detach(), 0)
                f2 = _conv_from(l2.weight.detach()[:, :, None, None], l2.bias.detach(), 0)
                layers.append((cav_pre.norm, hgt_qkv, hgt_out, win_pre.norm, win_qkv, branches, outs, gate, ffn.norm, f1, f2))
            self._derived = (sig, layers, {})
        thetas = self._derived[2]
        key = (H, W, str(device))
        if key not in thetas:
            thetas[key] = self.fusion_net.encoder.sttf.theta(H, W).to(device)
        return self._derived[1], thetas[key]

    def forward_nhwc(self, x, record_len, affine_matrix):
        """x: Act (sumN,H,W,C), affine_matrix (B,L,L,2,3) -> Act (B,H,W,C), the ego slot.  Reads record_len on the host; no
        other sync."""
        require_eval(self)
        rl = _rl(record_len)
        B, L = affine_matrix.shape[:2]
        C, H, W = x.C, x.H, x.W
        self._check(C, H, W, L)
        if len(rl) != B or any(n < 1 or n > L for n in rl) or sum(rl) != x.N:
            raise ValueError(f"V2XViTFusion: record_len {rl} does not fit {B} scenes of at most {L} agents and {x.N} maps")
        layers, theta = self._packed(H, W, x.device)
        fmt = engine.act_fmt()
        aff = affine_matrix.to(device=x.device, dtype=torch.float64)
        N = sum(rl)
        starts = [sum(rl[:b]) for b in range(B)]
        X = ops.act_empty(N, H, W, C, fmt, x.device)
        ops.warp_affine(x, starts, aff[:, 0, 0].contiguous(), out=X.images(0, B))
        if N > B:
            src = [starts[b] + j for b in range(B) for j in range(1, rl[b])]
            th = torch.cat([aff[b, 0, 1:rl[b]] for b in range(B) if rl[b] > 1])
            warped = ops.warp_affine(x, src, th, out_fmt=fmt)
            ops.sttf_resample(warped, theta.expand(N - B, 2, 3).contiguous(), out=X.images(B, N))
        for i, (n1, hgt_qkv, hgt_out, n2, win_qkv, branches, outs, gate, n3, f1, f2) in enumerate(layers):
            last = i == len(layers) - 1
            y = ops.mean_layernorm(X, 1, n1.weight, n1.bias, n1.eps, out_fmt=fmt)
            a = ops.cav_attention(conv_bn_act(y, hgt_qkv), rl, ego_only=last, out_fmt=fmt)
            X = conv_bn_act(a, hgt_out, residual=X.images(0, B) if last else X)
            y = ops.mean_layernorm(X, 1, n2.weight, n2.bias, n2.eps, out_fmt=fmt)
            qkv = conv_bn_act(y, win_qkv)
            o = ops.act_empty(X.N, H, W, 3 * C, fmt, x.device)
            off = 0
            for k, ((heads, dh, ws, bias), out_conv) in enumerate(zip(branches, outs)):
                att = ops.window_attention(qkv, heads, dh, ws, bias, qkv_coffset=off, out_fmt=fmt)
                conv_bn_act(att, out_conv, out=o, out_coffset=k * C)
                off += 3 * heads * dh
            fc1_t, ln, fc2_t = gate
            X = ops.split_attn(o, X, fc1_t, ln.weight, ln.bias, ln.eps, fc2_t, out_fmt=fmt)
            y = ops.mean_layernorm(X, 1, n3.weight, n3.bias, n3.eps, out_fmt=fmt)
            X = conv_bn_act(conv_bn_act(y, f1, relu=2), f2, residual=X)
        return X

    def forward(self, x, record_len, affine_matrix):
        require_eval(self)
        self._check(x.shape[1], x.shape[2], x.shape[3], affine_matrix.shape[1])
        return ops.act_to_nchw(self.forward_nhwc(ops.to_act(x), record_len, affine_matrix))
