"""HeterModelBaseline mirror (opencood/models/heter_model_baseline.py:26-236): per-modality encoder ->
BaseBEVBackbone -> per-agent shrinker -> single-scale fusion -> heads.  Same ctor argument, state-dict keys and forward(data_dict) -> output_dict contract.
`fusion_method`: att (AttFusion), max (F-Cooper MaxFusion), v2vnet (V2VNetFusion), v2xvit (V2XViTFusion), cobevt (CoBEVT),
where2comm (Where2commFusion) and who2com (Who2comFusion).  disconet cannot be constructed in the reference itself."""
from collections import OrderedDict

import torch.nn as nn

from ..engine import require_eval
from ..utils.transformation_utils import normalize_pairwise_tfm
from .sub_modules.base_bev_backbone import BaseBEVBackbone
from .sub_modules.downsample_conv import DownsampleConv
from .sub_modules.naive_compress import NaiveCompressor
from .fuse_modules.fusion_in_one import (AttFusion, CoBEVT, MaxFusion, V2VNetFusion, V2XViTFusion, Where2commFusion,
                                         Who2comFusion)
from .heter_common import HeterFront, add_heads, modality_names

_BUILT = "att, max, v2vnet, v2xvit, cobevt, where2comm, who2com"


class HeterModelBaseline(HeterFront, nn.Module):
    adapter_name = "shrinker"

    def __init__(self, args):
        super().__init__()
        self.args = args
        self.modality_name_list = modality_names(args)
        self.ego_modality = args.get('ego_modality')
        self.cav_range = args['lidar_range']
        self.sensor_type_dict = OrderedDict()
        for m in self.modality_name_list:
            setting = args[m]
            self._add_modality(m, setting, BaseBEVBackbone(setting['backbone_args'], setting['backbone_args'].get('inplanes', 64)),
                               DownsampleConv(setting['shrink_header']))
        self.H = self.cav_range[4] - self.cav_range[1]
        self.W = self.cav_range[3] - self.cav_range[0]
        self.fake_voxel_size = 1
        self.supervise_single = bool(args.get("supervise_single", False))
        if self.supervise_single:
            self._heads_single = add_heads(self, args['in_head_single'], args, "_single")
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
        self._heads = add_heads(self, args['in_head'], args)
        self.compress = 'compressor' in args
        if self.compress:
            self.compressor = NaiveCompressor(args['compressor']['input_dim'], args['compressor']['compress_ratio'])
        self.model_train_init()

    def forward(self, data_dict):
        require_eval(self)
        output_dict = {}
        affine = normalize_pairwise_tfm(data_dict['pairwise_t_matrix'], self.H, self.W, self.fake_voxel_size)
        record_len = data_dict['record_len']
        x = self._assemble(data_dict, output_dict)
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
