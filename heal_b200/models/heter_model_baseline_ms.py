"""HeterModelBaselineMs mirror (opencood/models/heter_model_baseline_ms.py:26-220), the multi-scale model of every
`*_coalign.yaml`: per-modality encoder -> ResNetBEVBackbone -> AlignNet -> camera CenterCrop -> fusion-backbone levels 1.. on
every agent -> per-level fusion -> decode -> (shrink) -> heads.  Same ctor argument, state-dict keys (the fusion backbone's
layer0 included, which the reference builds but never runs) and forward(data_dict) -> output_dict contract.
`fusion_method`: att (AttFusion per level) and max (MaxFusion per level), the two the reference builds."""
import importlib
from collections import OrderedDict, Counter

import torch.nn as nn

from .. import ops
from ..engine import require_eval
from ..utils.transformation_utils import normalize_pairwise_tfm
from .sub_modules.base_bev_backbone_resnet import ResNetBEVBackbone
from .sub_modules.feature_alignnet import AlignNet
from .sub_modules.downsample_conv import DownsampleConv
from .fuse_modules.fusion_in_one import AttFusion, MaxFusion
from .heter_pyramid_collab import FusedHeads


class HeterModelBaselineMs(nn.Module):
    def __init__(self, args):
        super().__init__()
        self.args = args
        self.modality_name_list = [x for x in args.keys() if x.startswith("m") and x[1:].isdigit()]
        self.ego_modality = args.get('ego_modality')
        self.stage2_added_modality = args.get('stage2_added_modality', None)
        self.cav_range = args['lidar_range']
        self.sensor_type_dict = OrderedDict()
        encoder_lib = importlib.import_module("heal_b200.models.heter_encoders")
        for m in self.modality_name_list:
            setting = args[m]
            self.sensor_type_dict[m] = setting['sensor_type']
            target = setting['core_method'].replace('_', '').lower()
            enc_cls = next((c for n, c in encoder_lib.__dict__.items() if n.lower() == target), None)
            if enc_cls is None:
                raise NotImplementedError(f"encoder '{setting['core_method']}' not available in heal_b200.models.heter_encoders")
            setattr(self, f"encoder_{m}", enc_cls(setting['encoder_args']))
            setattr(self, f"depth_supervision_{m}", bool(setting['encoder_args'].get("depth_supervision", False)))
            setattr(self, f"backbone_{m}", ResNetBEVBackbone(setting['backbone_args']))
            setattr(self, f"aligner_{m}", AlignNet(setting['aligner_args']))
            if setting['sensor_type'] == "camera":
                g = setting['camera_mask_args']['grid_conf']
                setattr(self, f"crop_ratio_W_{m}", self.cav_range[3] / g['xbound'][1])
                setattr(self, f"crop_ratio_H_{m}", self.cav_range[4] / g['ybound'][1])
                setattr(self, f"xdist_{m}", g['xbound'][1] - g['xbound'][0])
                setattr(self, f"ydist_{m}", g['ybound'][1] - g['ybound'][0])
        self.H = self.cav_range[4] - self.cav_range[1]
        self.W = self.cav_range[3] - self.cav_range[0]
        self.fake_voxel_size = 1
        self.supervise_single = bool(args.get("supervise_single", False))
        if self.supervise_single:
            c = args['in_head_single']
            self.cls_head_single = nn.Conv2d(c, args['anchor_number'], kernel_size=1)
            self.reg_head_single = nn.Conv2d(c, args['anchor_number'] * 7, kernel_size=1)
            self.dir_head_single = nn.Conv2d(c, args['anchor_number'] * args['dir_args']['num_bins'], kernel_size=1)
            self._heads_single = FusedHeads([self.cls_head_single, self.reg_head_single, self.dir_head_single])

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
        self.cls_head = nn.Conv2d(args['in_head'], args['anchor_number'], kernel_size=1)
        self.reg_head = nn.Conv2d(args['in_head'], 7 * args['anchor_number'], kernel_size=1)
        self.dir_head = nn.Conv2d(args['in_head'], args['dir_args']['num_bins'] * args['anchor_number'], kernel_size=1)
        self._heads = FusedHeads([self.cls_head, self.reg_head, self.dir_head])

    def model_train_init(self):
        pass

    def forward(self, data_dict):
        require_eval(self)
        output_dict = {}
        aml = data_dict['agent_modality_list']
        affine = normalize_pairwise_tfm(data_dict['pairwise_t_matrix'], self.H, self.W, self.fake_voxel_size)
        record_len = data_dict['record_len']
        count = Counter(aml)
        feats, crops = {}, {}
        for m in self.modality_name_list:
            if m not in count:
                continue
            enc = getattr(self, f"encoder_{m}")
            f = enc.forward_act(data_dict, m) if hasattr(enc, "forward_act") else ops.to_act(enc(data_dict, m))
            bb = getattr(self, f"backbone_{m}")
            f = bb.decode_nhwc(bb.multiscale_nhwc(f))
            f = getattr(self, f"aligner_{m}").forward_nhwc(f)
            if self.sensor_type_dict[m] == "camera":
                crops[m] = (int(f.H * getattr(self, f"crop_ratio_H_{m}")), int(f.W * getattr(self, f"crop_ratio_W_{m}")))
                if getattr(self, f"depth_supervision_{m}"):
                    output_dict[f"depth_items_{m}"] = enc.depth_items
            feats[m] = f
        if len(feats) == 1 and all(a == aml[0] for a in aml) and not crops:
            x = feats[aml[0]]
        else:                                   # fp32 (n_agents, H, W, C) in scene order, camera maps cropped / padded
            x = ops.agent_stack(feats, aml, crops)
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
