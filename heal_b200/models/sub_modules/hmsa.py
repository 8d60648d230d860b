"""Parameter container of opencood/models/sub_modules/hmsa.py (HGTCavAttention) with the reference's submodule names.
V2XViTFusion runs it: with every agent of type 0 only q/k/v/a_linears[0], relation_att[0] and relation_msg[0] are live, folded
into one to_qkv 1x1 conv ahead of heal_cav_attention and the a_linears[0] conv after it."""
import torch
from torch import nn


class HGTCavAttention(nn.Module):
    def __init__(self, dim, heads, num_types=2, num_relations=4, dim_head=64, dropout=0.1):
        super().__init__()
        inner_dim = heads * dim_head
        self.heads = heads
        self.dim_head = dim_head
        self.scale = dim_head ** -0.5
        self.num_types = num_types
        self.attend = nn.Softmax(dim=-1)
        self.drop_out = nn.Dropout(dropout)
        self.k_linears = nn.ModuleList()
        self.q_linears = nn.ModuleList()
        self.v_linears = nn.ModuleList()
        self.a_linears = nn.ModuleList()
        self.norms = nn.ModuleList()
        for _ in range(num_types):
            self.k_linears.append(nn.Linear(dim, inner_dim))
            self.q_linears.append(nn.Linear(dim, inner_dim))
            self.v_linears.append(nn.Linear(dim, inner_dim))
            self.a_linears.append(nn.Linear(inner_dim, dim))
        self.relation_att = nn.Parameter(torch.empty(num_relations, heads, dim_head, dim_head))
        self.relation_msg = nn.Parameter(torch.empty(num_relations, heads, dim_head, dim_head))
        nn.init.xavier_uniform_(self.relation_att)
        nn.init.xavier_uniform_(self.relation_msg)

    def forward(self, x, mask, prior_encoding):
        raise NotImplementedError("executed by V2XViTFusion.forward_nhwc (heal_cav_attention between two 1x1 convs)")
