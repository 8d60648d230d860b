"""HeterPyramidCollab mirror (opencood/models/heter_pyramid_collab.py:21-209): same ctor argument
(`hypes['model']['args']`), same state-dict keys, same forward(data_dict) -> output_dict contract."""
from collections import OrderedDict

import torch.nn as nn

from .. import ops
from ..engine import require_eval
from ..utils.transformation_utils import normalize_pairwise_tfm
from .sub_modules.base_bev_backbone_resnet import ResNetBEVBackbone
from .sub_modules.feature_alignnet import AlignNet
from .sub_modules.downsample_conv import DownsampleConv
from .sub_modules.naive_compress import NaiveCompressor
from .fuse_modules.pyramid_fuse import PyramidFusion
from .heter_common import HeterFront, add_heads, crop_tensor, modality_names


class HeterPyramidCollab(HeterFront, nn.Module):
    adapter_name = "aligner"     # identity, or the ConvNeXt aligner (HEAL stage 2)
    # the CenterCrop the collab forward applied before heal_agent_stack; tests restate that sequence through the class
    _crop_tensor = staticmethod(crop_tensor)

    def __init__(self, args):
        super().__init__()
        self.args = args
        self.modality_name_list = modality_names(args)
        self.cav_range = args['lidar_range']
        self.sensor_type_dict = OrderedDict()
        self.cam_crop_info = {}
        for m in self.modality_name_list:
            setting = args[m]
            self._add_modality(m, setting, ResNetBEVBackbone(setting['backbone_args']), AlignNet(setting['aligner_args']))
            if setting['sensor_type'] == "camera":
                self.cam_crop_info[m] = {f"crop_ratio_W_{m}": getattr(self, f"crop_ratio_W_{m}"),
                                         f"crop_ratio_H_{m}": getattr(self, f"crop_ratio_H_{m}")}
        self.H = self.cav_range[4] - self.cav_range[1]
        self.W = self.cav_range[3] - self.cav_range[0]
        self.fake_voxel_size = 1
        self.pyramid_backbone = PyramidFusion(args['fusion_backbone'])
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
        output_dict = {'pyramid': 'collab'}
        aml = data_dict['agent_modality_list']
        affine = normalize_pairwise_tfm(data_dict['pairwise_t_matrix'], self.H, self.W, self.fake_voxel_size)
        record_len = data_dict['record_len']
        x = self._assemble(data_dict, output_dict)
        if self.compress:
            x = self.compressor.forward_nhwc(x)
        fused, occs = self.pyramid_backbone.forward_collab_nhwc(x, record_len, affine, aml, self.cam_crop_info)
        if self.shrink_flag:
            fused = self.shrink_conv.forward_nhwc(fused)
        cls, reg, dirp = self._heads(fused)
        output_dict.update({'cls_preds': cls, 'reg_preds': reg, 'dir_preds': dirp})
        output_dict['occ_single_list'] = [ops.act_to_nchw(o) for o in occs]
        return output_dict
