"""Parameter container of opencood/models/sub_modules/split_attn.py (SplitAttn) with the reference's submodule names.
V2XViTFusion runs it as heal_split_attn (pool, gate MLP and weighted combine with the residual)."""
import torch.nn as nn


class SplitAttn(nn.Module):
    def __init__(self, input_dim):
        super().__init__()
        self.input_dim = input_dim
        self.fc1 = nn.Linear(input_dim, input_dim, bias=False)
        self.bn1 = nn.LayerNorm(input_dim)
        self.act1 = nn.ReLU()
        self.fc2 = nn.Linear(input_dim, input_dim * 3, bias=False)

    def forward(self, window_list):
        raise NotImplementedError("executed by V2XViTFusion.forward_nhwc (heal_split_attn)")
