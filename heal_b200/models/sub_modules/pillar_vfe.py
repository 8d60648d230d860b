"""PillarVFE on the fused sm_90a kernel (heal_pillar_vfe_scatter).

Mirror of opencood/models/sub_modules/pillar_vfe.py: same class names, ctor arguments, state-dict keys
(`pfn_layers.0.linear.weight`, `pfn_layers.0.norm.*`) and `forward(batch_dict)` contract
(:105-155): reads voxel_features / voxel_num_points / voxel_coords, writes `pillar_features`.
Supported configuration = the one every HEAL yaml uses: use_norm, use_absolute_xyz, !with_distance,
one PFN layer of 64 filters; anything else raises instead of silently falling back.
"""
import torch
import torch.nn as nn

from ... import ops
from ...engine import require_eval, _sig


class PFNLayer(nn.Module):
    def __init__(self, in_channels, out_channels, use_norm=True, last_layer=False):
        super().__init__()
        self.last_vfe = last_layer
        self.use_norm = use_norm
        if not self.last_vfe:
            out_channels = out_channels // 2
        if self.use_norm:
            self.linear = nn.Linear(in_channels, out_channels, bias=False)
            self.norm = nn.BatchNorm1d(out_channels, eps=1e-3, momentum=0.01)
        else:
            self.linear = nn.Linear(in_channels, out_channels, bias=True)

    def forward(self, inputs):
        raise NotImplementedError("PFNLayer is executed fused inside PillarVFE (heal_pillar_vfe_scatter)")


class PillarVFE(nn.Module):
    def __init__(self, model_cfg, num_point_features, voxel_size, point_cloud_range):
        super().__init__()
        self.model_cfg = model_cfg
        self.use_norm = model_cfg['use_norm']
        self.with_distance = model_cfg['with_distance']
        self.use_absolute_xyz = model_cfg['use_absolute_xyz']
        num_point_features += 6 if self.use_absolute_xyz else 3
        if self.with_distance:
            num_point_features += 1
        self.num_filters = list(model_cfg['num_filters'])
        assert len(self.num_filters) > 0
        dims = [num_point_features] + self.num_filters
        self.pfn_layers = nn.ModuleList(
            [PFNLayer(dims[i], dims[i + 1], self.use_norm, last_layer=(i >= len(dims) - 2))
             for i in range(len(dims) - 1)])
        if not (self.use_norm and self.use_absolute_xyz and not self.with_distance and len(self.num_filters) == 1
                and self.num_filters[0] == 64 and num_point_features == 10):
            raise NotImplementedError("heal_b200 PillarVFE kernel: use_norm, use_absolute_xyz, !with_distance, num_filters=[64]")
        self.voxel_size = [float(v) for v in voxel_size]
        self.point_cloud_range = [float(v) for v in point_cloud_range]
        self._fold = None

    def get_output_feature_dim(self):
        return self.num_filters[-1]

    def folded(self):
        pfn = self.pfn_layers[0]
        sig = _sig(pfn.linear, pfn.norm)
        if self._fold is None or self._fold[0] != sig:
            w, b = ops.fold_linear_bn(pfn.linear.weight, pfn.norm.weight, pfn.norm.bias,
                                      pfn.norm.running_mean, pfn.norm.running_var, pfn.norm.eps)
            dev = pfn.linear.weight.device
            self._fold = (sig, w.to(dev).contiguous(), b.to(dev).contiguous())
        return self._fold[1], self._fold[2]

    def forward(self, batch_dict):
        require_eval(self)
        w, b = self.folded()
        pf, _ = ops.pillar_vfe_scatter(batch_dict['voxel_features'], batch_dict['voxel_num_points'],
                                       batch_dict['voxel_coords'], w, b, self.voxel_size, self.point_cloud_range,
                                       nx=1, ny=1, batch_size=1, want_pillar_features=True, want_canvas=False)
        batch_dict['pillar_features'] = pf.squeeze()   # reference squeezes (pillar_vfe.py:152)
        return batch_dict
