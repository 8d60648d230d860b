"""Single-agent PointPillar mirror (opencood/models/point_pillar.py:17-80; BASELINE config 1):
processed_lidar -> PillarVFE -> PointPillarScatter -> BaseBEVBackbone -> shrink -> cls / reg (/ dir) heads."""
import numpy as np
import torch
import torch.nn as nn

from .. import ops
from ..engine import require_eval, act_fmt
from .sub_modules.pillar_vfe import PillarVFE
from .sub_modules.point_pillar_scatter import PointPillarScatter
from .sub_modules.base_bev_backbone import BaseBEVBackbone
from .sub_modules.base_bev_backbone_resnet import ResNetBEVBackbone
from .sub_modules.downsample_conv import DownsampleConv
from .heter_common import add_heads


class PointPillar(nn.Module):
    def __init__(self, args):
        super().__init__()
        self.pillar_vfe = PillarVFE(args['pillar_vfe'], num_point_features=4, voxel_size=args['voxel_size'],
                                    point_cloud_range=args['lidar_range'])
        if 'grid_size' not in args['point_pillar_scatter']:
            g = (np.array(args['lidar_range'][3:6]) - np.array(args['lidar_range'][0:3])) / np.array(args['voxel_size'])
            args['point_pillar_scatter']['grid_size'] = np.round(g).astype(np.int64)
        self.scatter = PointPillarScatter(args['point_pillar_scatter'])
        is_resnet = args['base_bev_backbone'].get("resnet", False)
        self.backbone = ResNetBEVBackbone(args['base_bev_backbone'], 64) if is_resnet else BaseBEVBackbone(args['base_bev_backbone'], 64)
        self.voxel_size, self.lidar_range = [float(v) for v in args['voxel_size']], [float(v) for v in args['lidar_range']]
        self.voxelize_args = args.get('voxelize', {'max_points_per_voxel': 32, 'max_voxels': 70000})
        self.shrink_flag = 'shrink_header' in args
        if self.shrink_flag:
            self.shrink_conv = DownsampleConv(args['shrink_header'])
            self.out_channel = args['shrink_header']['dim'][-1]
        else:
            self.out_channel = sum(args['base_bev_backbone']['num_upsample_filter'])
        self.use_dir = 'dir_args' in args
        self._heads = add_heads(self, self.out_channel, args, use_dir=self.use_dir)

    def forward(self, data_dict):
        require_eval(self)
        inp = data_dict['processed_lidar']
        nvox_dev = None
        if 'voxel_features' in inp:
            vf, vc, vn = inp['voxel_features'], inp['voxel_coords'], inp['voxel_num_points']
            batch_size = inp.get('batch_size')
            if batch_size is None:
                batch_size = int(vc[:, 0].max().item()) + 1     # host sync, as the reference (point_pillar_scatter.py:45)
        else:
            # raw points (`points`, `agent_offsets`): GPU voxelisation, no host sync (graph-capturable frame)
            va = self.voxelize_args
            pts, offs = ops.raw_points_of(inp, self.lidar_range)
            vf, vc, vn, nvox_dev = ops.voxelize(pts, offs, self.lidar_range, self.voxel_size,
                                                int(inp.get('max_points_per_voxel', va['max_points_per_voxel'])),
                                                int(inp.get('max_voxels', va['max_voxels'])))
            batch_size = inp['agent_offsets'].numel() - 1
        w, b = self.pillar_vfe.folded()
        _, canvas = ops.pillar_vfe_scatter(vf, vn, vc, w, b, self.voxel_size,
                                           self.lidar_range, nx=self.scatter.nx, ny=self.scatter.ny, batch_size=batch_size,
                                           num_voxels_dev=nvox_dev, canvas_fmt=act_fmt())
        x = self.backbone.decode_nhwc(self.backbone.multiscale_nhwc(canvas))
        if self.shrink_flag:
            x = self.shrink_conv.forward_nhwc(x)
        outs = self._heads(x)
        output_dict = {'cls_preds': outs[0], 'reg_preds': outs[1]}
        if self.use_dir:
            output_dict['dir_preds'] = outs[2]
        return output_dict
