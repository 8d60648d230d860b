"""HeterModelBaselineMs mirror (opencood/models/heter_model_baseline_ms.py:26-220), the multi-scale model of every
`*_coalign.yaml`: per-modality encoder -> ResNetBEVBackbone -> AlignNet -> camera CenterCrop -> fusion-backbone levels 1.. on
every agent -> per-level fusion -> decode -> (shrink) -> heads.  Same ctor argument, state-dict keys (the fusion backbone's
layer0 included, which the reference builds but never runs) and forward(data_dict) -> output_dict contract.
`fusion_method`: att (AttFusion per level) and max (MaxFusion per level), the two the reference builds."""
from collections import OrderedDict

import torch.nn as nn

from ..engine import require_eval
from ..utils.transformation_utils import normalize_pairwise_tfm
from .sub_modules.base_bev_backbone_resnet import ResNetBEVBackbone
from .sub_modules.feature_alignnet import AlignNet
from .sub_modules.downsample_conv import DownsampleConv
from .fuse_modules.fusion_in_one import AttFusion, MaxFusion
from .heter_common import HeterFront, add_heads, modality_names


class HeterModelBaselineMs(HeterFront, nn.Module):
    adapter_name = "aligner"

    def __init__(self, args):
        super().__init__()
        self.args = args
        self.modality_name_list = modality_names(args)
        self.ego_modality = args.get('ego_modality')
        self.stage2_added_modality = args.get('stage2_added_modality', None)
        self.cav_range = args['lidar_range']
        self.sensor_type_dict = OrderedDict()
        for m in self.modality_name_list:
            setting = args[m]
            self._add_modality(m, setting, ResNetBEVBackbone(setting['backbone_args']), AlignNet(setting['aligner_args']))
            if setting['sensor_type'] == "camera":
                g = setting['camera_mask_args']['grid_conf']
                setattr(self, f"xdist_{m}", g['xbound'][1] - g['xbound'][0])
                setattr(self, f"ydist_{m}", g['ybound'][1] - g['ybound'][0])
        self.H = self.cav_range[4] - self.cav_range[1]
        self.W = self.cav_range[3] - self.cav_range[0]
        self.fake_voxel_size = 1
        self.supervise_single = bool(args.get("supervise_single", False))
        if self.supervise_single:
            self._heads_single = add_heads(self, args['in_head_single'], args, "_single")

        # fusion: one module per fusion-backbone level; level i has num_filters[i] channels
        self.backbone = ResNetBEVBackbone(args['fusion_backbone'])
        fm = args['fusion_method']
        if fm not in ("att", "max"):
            raise NotImplementedError(f"HeterModelBaselineMs fusion_method '{fm}' is not built (built: att, max)")
        channels = list(args['fusion_backbone']['num_filters'])
        if fm == "att":
            feat_dim = args['att']['feat_dim']
            # heal_att_fuse scales the scores by 1/sqrt(C), the reference by 1/sqrt(feat_dim[i]): they must agree
            if not isinstance(feat_dim, (list, tuple)):
                raise ValueError(f"att.feat_dim {feat_dim!r} must list one entry per fusion level ({len(channels)} entries)")
            feat_dim = list(feat_dim)
            if len(feat_dim) != len(channels):
                raise ValueError(f"att.feat_dim {feat_dim} has {len(feat_dim)} entries for {len(channels)} fusion levels")
            if feat_dim != channels:
                raise ValueError(f"att.feat_dim {feat_dim} differs from the fusion levels' channel counts {channels} "
                                 "(fusion_backbone.num_filters)")
        self.level_channels = channels
        self.fusion_net = nn.ModuleList()
        for i in range(len(channels)):
            self.fusion_net.append(AttFusion(feat_dim[i]) if fm == "att" else MaxFusion())

        self.shrink_flag = 'shrink_header' in args
        if self.shrink_flag:
            self.shrink_conv = DownsampleConv(args['shrink_header'])
        self._heads = add_heads(self, args['in_head'], args)

    def forward(self, data_dict):
        require_eval(self)
        output_dict = {}
        affine = normalize_pairwise_tfm(data_dict['pairwise_t_matrix'], self.H, self.W, self.fake_voxel_size)
        record_len = data_dict['record_len']
        x = self._assemble(data_dict, output_dict)
        if x.C != self.level_channels[0]:
            raise ValueError(f"the per-agent maps have {x.C} channels, the first fusion level {self.level_channels[0]}")
        if self.supervise_single:
            c, r, d = self._heads_single(x)
            output_dict.update({'cls_preds_single': c, 'reg_preds_single': r, 'dir_preds_single': d})
        # the fusion backbone's layer0 is never run: level 0 is the assembled map itself
        levels = [x]
        resnet = self.backbone.resnet
        for i in range(1, len(self.fusion_net)):
            levels.append(resnet._run_level(getattr(resnet, f"layer{i}"), levels[-1]))
        fused = [fuse.forward_nhwc(f, record_len, affine) for fuse, f in zip(self.fusion_net, levels)]
        fused = self.backbone.decode_nhwc(fused)
        if self.shrink_flag:
            fused = self.shrink_conv.forward_nhwc(fused)
        cls, reg, dirp = self._heads(fused)
        output_dict.update({'cls_preds': cls, 'reg_preds': reg, 'dir_preds': dirp})
        return output_dict
