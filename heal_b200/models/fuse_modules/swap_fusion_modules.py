"""Parameter containers of opencood/models/fuse_modules/swap_fusion_modules.py:13-192 (Attention, SwapFusionBlockMask) with
the reference's submodule names, Sequential indices and the int64 `relative_position_index` buffer, built exactly as the
reference builds it.  CoBEVT (fusion_in_one.py) runs them: heal_swap_attention between the to_qkv / to_out 1x1 convs."""
import torch
import torch.nn as nn

from ..sub_modules.base_transformer import FeedForward, PreNormResidual


def relative_position_index(agent_size, window_size):
    """(n, n) int64, n = agent_size * window_size^2: the index of token pair (i, j) into the (Δagent, Δw1, Δw2) bias table,
    tokens ordered (agent, w1, w2) (swap_fusion_modules.py:61-83)."""
    ws = [agent_size, window_size, window_size]
    coords = torch.stack(torch.meshgrid(torch.arange(ws[0]), torch.arange(ws[1]), torch.arange(ws[2]), indexing="ij"))
    flat = torch.flatten(coords, 1)
    rel = (flat[:, :, None] - flat[:, None, :]).permute(1, 2, 0).contiguous()
    rel[:, :, 0] += ws[0] - 1
    rel[:, :, 1] += ws[1] - 1
    rel[:, :, 2] += ws[2] - 1
    rel[:, :, 0] *= (2 * ws[1] - 1) * (2 * ws[2] - 1)
    rel[:, :, 1] *= 2 * ws[2] - 1
    return rel.sum(-1)


class Attention(nn.Module):
    def __init__(self, dim, dim_head=32, dropout=0., agent_size=6, window_size=7):
        super().__init__()
        assert (dim % dim_head) == 0, 'dimension should be divisible by dimension per head'
        self.heads = dim // dim_head
        self.dim_head = dim_head
        self.scale = dim_head ** -0.5
        self.window_size = [agent_size, window_size, window_size]
        self.to_qkv = nn.Linear(dim, dim * 3, bias=False)
        self.attend = nn.Sequential(nn.Softmax(dim=-1))
        self.to_out = nn.Sequential(nn.Linear(dim, dim, bias=False), nn.Dropout(dropout))
        self.relative_position_bias_table = nn.Embedding(
            (2 * agent_size - 1) * (2 * window_size - 1) * (2 * window_size - 1), self.heads)
        self.register_buffer("relative_position_index", relative_position_index(agent_size, window_size))

    def forward(self, x, mask=None):
        raise NotImplementedError("executed by CoBEVT.forward_nhwc (heal_swap_attention between two 1x1 convs)")


class SwapFusionBlockMask(nn.Module):
    def __init__(self, input_dim, mlp_dim, dim_head, window_size, agent_size, drop_out):
        super().__init__()
        self.window_size = window_size
        self.window_attention = PreNormResidual(input_dim, Attention(input_dim, dim_head, drop_out, agent_size, window_size))
        self.window_ffd = PreNormResidual(input_dim, FeedForward(input_dim, mlp_dim, drop_out))
        self.grid_attention = PreNormResidual(input_dim, Attention(input_dim, dim_head, drop_out, agent_size, window_size))
        self.grid_ffd = PreNormResidual(input_dim, FeedForward(input_dim, mlp_dim, drop_out))

    def forward(self, x, mask):
        raise NotImplementedError("executed by CoBEVT.forward_nhwc")
