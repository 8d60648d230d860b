"""Parameter containers of opencood/models/sub_modules/mswin.py (BaseWindowAttention, PyramidWindowAttention) with the
reference's submodule names.  `relative_indices` is a plain attribute in the reference (not a buffer), so it is rebuilt here
the same way.  V2XViTFusion runs the branches as one to_qkv 1x1 conv, heal_window_attention per branch and the to_out convs."""
import torch
import torch.nn as nn

from .split_attn import SplitAttn


def get_relative_distances(window_size):
    """(w^2, w^2, 2) int64: entry [i][j] = (row, col) of token j minus (row, col) of token i, tokens t = row * w + col in
    row-major order (the offsets the reference's mswin.py:13-17 indexes pos_embedding with, before its + w - 1)."""
    rows, cols = torch.meshgrid(torch.arange(window_size), torch.arange(window_size), indexing="ij")
    coords = torch.stack([rows.reshape(-1), cols.reshape(-1)], dim=-1)
    return coords.unsqueeze(0) - coords.unsqueeze(1)


class BaseWindowAttention(nn.Module):
    def __init__(self, dim, heads, dim_head, drop_out, window_size, relative_pos_embedding):
        super().__init__()
        inner_dim = dim_head * heads
        self.heads = heads
        self.dim_head = dim_head
        self.scale = dim_head ** -0.5
        self.window_size = window_size
        self.relative_pos_embedding = relative_pos_embedding
        self.to_qkv = nn.Linear(dim, inner_dim * 3, bias=False)
        if self.relative_pos_embedding:
            self.relative_indices = get_relative_distances(window_size) + window_size - 1
            self.pos_embedding = nn.Parameter(torch.randn(2 * window_size - 1, 2 * window_size - 1))
        else:
            self.pos_embedding = nn.Parameter(torch.randn(window_size ** 2, window_size ** 2))
        self.to_out = nn.Sequential(nn.Linear(inner_dim, dim), nn.Dropout(drop_out))

    def dense_bias(self):
        """The (w^2, w^2) bias added to q k^T, query-major: pos_embedding[relative_indices] (or pos_embedding itself)."""
        pe = self.pos_embedding.detach()
        if self.relative_pos_embedding:
            ri = self.relative_indices.to(pe.device)
            return pe[ri[:, :, 0], ri[:, :, 1]]
        return pe

    def forward(self, x):
        raise NotImplementedError("executed by V2XViTFusion.forward_nhwc (heal_window_attention between 1x1 convs)")


class PyramidWindowAttention(nn.Module):
    def __init__(self, dim, heads, dim_heads, drop_out, window_size, relative_pos_embedding, fuse_method='naive'):
        super().__init__()
        assert isinstance(window_size, list)
        assert isinstance(heads, list)
        assert isinstance(dim_heads, list)
        assert len(dim_heads) == len(heads)
        self.pwmsa = nn.ModuleList([])
        for (head, dim_head, ws) in zip(heads, dim_heads, window_size):
            self.pwmsa.append(BaseWindowAttention(dim, head, dim_head, drop_out, ws, relative_pos_embedding))
        self.fuse_mehod = fuse_method
        if fuse_method == 'split_attn':
            self.split_attn = SplitAttn(256)
        elif fuse_method == 'split_attn128':
            self.split_attn = SplitAttn(128)
        elif fuse_method == 'split_attn64':
            self.split_attn = SplitAttn(64)

    def forward(self, x):
        raise NotImplementedError("executed by V2XViTFusion.forward_nhwc")
