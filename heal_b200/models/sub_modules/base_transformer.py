"""Parameter containers of opencood/models/sub_modules/base_transformer.py:7-39 (PreNorm, PreNormResidual, FeedForward), with
the reference's submodule names and Sequential indices.  Their forward runs inside the fusion module that owns them (CoBEVT,
V2XViTFusion: heal_mean_layernorm for the norm, the conv engine for the Linear layers with GELU / residual in the epilogue)."""
import torch.nn as nn


class PreNormResidual(nn.Module):
    def __init__(self, dim, fn):
        super().__init__()
        self.norm = nn.LayerNorm(dim)
        self.fn = fn

    def forward(self, x, **kwargs):
        raise NotImplementedError("executed by the owning fusion module's forward_nhwc")


class FeedForward(nn.Module):
    def __init__(self, dim, hidden_dim, dropout=0.):
        super().__init__()
        self.net = nn.Sequential(
            nn.Linear(dim, hidden_dim),
            nn.GELU(),
            nn.Dropout(dropout),
            nn.Linear(hidden_dim, dim),
            nn.Dropout(dropout)
        )

    def forward(self, x):
        raise NotImplementedError("executed by the owning fusion module's forward_nhwc")


class PreNorm(nn.Module):
    def __init__(self, dim, fn):
        super().__init__()
        self.norm = nn.LayerNorm(dim)
        self.fn = fn

    def forward(self, x, **kwargs):
        raise NotImplementedError("executed by the owning fusion module's forward_nhwc")
