"""HeterModelBaseline mirror (opencood/models/heter_model_baseline.py:26-236): per-modality encoder ->
BaseBEVBackbone -> per-agent shrinker -> single-scale fusion -> heads.  Same ctor argument, state-dict keys and forward(data_dict) -> output_dict contract.
`fusion_method`: att (AttFusion), max (F-Cooper MaxFusion), v2vnet (V2VNetFusion), v2xvit (V2XViTFusion), cobevt (CoBEVT),
where2comm (Where2commFusion) and who2com (Who2comFusion).  disconet cannot be constructed in the reference itself."""
import importlib
from collections import OrderedDict, Counter

import torch.nn as nn

from .. import ops
from ..engine import require_eval
from ..utils.transformation_utils import normalize_pairwise_tfm
from .sub_modules.base_bev_backbone import BaseBEVBackbone
from .sub_modules.downsample_conv import DownsampleConv
from .sub_modules.naive_compress import NaiveCompressor
from .fuse_modules.fusion_in_one import (AttFusion, CoBEVT, MaxFusion, V2VNetFusion, V2XViTFusion, Where2commFusion,
                                         Who2comFusion)
from .heter_pyramid_collab import FusedHeads, HeterPyramidCollab

_BUILT = "att, max, v2vnet, v2xvit, cobevt, where2comm, who2com"


class HeterModelBaseline(nn.Module):
    def __init__(self, args):
        super().__init__()
        self.args = args
        self.modality_name_list = [x for x in args.keys() if x.startswith("m") and x[1:].isdigit()]
        self.ego_modality = args.get('ego_modality')
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
            setattr(self, f"backbone_{m}", BaseBEVBackbone(setting['backbone_args'], setting['backbone_args'].get('inplanes', 64)))
            setattr(self, f"shrinker_{m}", DownsampleConv(setting['shrink_header']))
            if setting['sensor_type'] == "camera":
                g = setting['camera_mask_args']['grid_conf']
                setattr(self, f"crop_ratio_W_{m}", self.cav_range[3] / g['xbound'][1])
                setattr(self, f"crop_ratio_H_{m}", self.cav_range[4] / g['ybound'][1])
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
        fm = args['fusion_method']
        if fm == "att":
            self.fusion_net = AttFusion(args['att']['feat_dim'])
        elif fm == "max":
            self.fusion_net = MaxFusion()
        elif fm == "v2vnet":
            self.fusion_net = V2VNetFusion(args['v2vnet'])
        elif fm == "cobevt":
            self.fusion_net = CoBEVT(args['cobevt'])
        elif fm == "v2xvit":
            if 'v2xvit' not in args:
                raise NotImplementedError("fusion_method 'v2xvit' without a `v2xvit:` block is outside the heal_b200 hot-path "
                                          "scope (no shipped config omits it)")
            self.fusion_net = V2XViTFusion(args['v2xvit'])
        elif fm in ("where2comm", "who2com"):
            if fm not in args:
                raise NotImplementedError(f"fusion_method '{fm}' without a `{fm}:` block is outside the heal_b200 hot-path "
                                          f"scope (built: {_BUILT})")
            dims = args[fm]
            if not isinstance(dims, int) or isinstance(dims, bool) or dims != 256:
                raise NotImplementedError(f"fusion_method '{fm}' with `{fm}: {dims!r}` is outside the heal_b200 hot-path "
                                          "scope (built: the int 256, every baseline yaml's in_head)")
            self.fusion_net = Where2commFusion(dims) if fm == "where2comm" else Who2comFusion(dims)
        elif fm == "disconet":
            raise NotImplementedError("fusion_method 'disconet': DiscoFusion cannot be constructed in the reference either "
                                      "(it imports opencood.models.fuse_modules.disco_fuse, which the reference does not ship)")
        else:
            raise NotImplementedError(f"fusion_method '{fm}' is outside the heal_b200 hot-path scope (built: {_BUILT})")
        self.shrink_flag = 'shrink_header' in args
        if self.shrink_flag:
            self.shrink_conv = DownsampleConv(args['shrink_header'])
        self.cls_head = nn.Conv2d(args['in_head'], args['anchor_number'], kernel_size=1)
        self.reg_head = nn.Conv2d(args['in_head'], 7 * args['anchor_number'], kernel_size=1)
        self.dir_head = nn.Conv2d(args['in_head'], args['dir_args']['num_bins'] * args['anchor_number'], kernel_size=1)
        self.compress = 'compressor' in args
        if self.compress:
            self.compressor = NaiveCompressor(args['compressor']['input_dim'], args['compressor']['compress_ratio'])
        self._heads = FusedHeads([self.cls_head, self.reg_head, self.dir_head])
        self.model_train_init()

    model_train_init = HeterPyramidCollab.model_train_init

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
            f = getattr(self, f"shrinker_{m}").forward_nhwc(f)
            if self.sensor_type_dict[m] == "camera":
                crops[m] = (int(f.H * getattr(self, f"crop_ratio_H_{m}")), int(f.W * getattr(self, f"crop_ratio_W_{m}")))
                if getattr(self, f"depth_supervision_{m}"):
                    output_dict[f"depth_items_{m}"] = enc.depth_items
            feats[m] = f
        if len(feats) == 1 and all(a == aml[0] for a in aml) and not crops:
            x = feats[aml[0]]
        else:                                   # fp32 (n_agents, H, W, C) in scene order, camera maps cropped / padded
            x = ops.agent_stack(feats, aml, crops)
        if self.compress:
            x = self.compressor.forward_nhwc(x)
        if self.supervise_single:
            c, r, d = self._heads_single(x)
            output_dict.update({'cls_preds_single': c, 'reg_preds_single': r, 'dir_preds_single': d})
        fused = self.fusion_net.forward_nhwc(x, record_len, affine)
        if self.shrink_flag:
            fused = self.shrink_conv.forward_nhwc(fused)
        cls, reg, dirp = self._heads(fused)
        output_dict.update({'cls_preds': cls, 'reg_preds': reg, 'dir_preds': dirp})
        return output_dict
