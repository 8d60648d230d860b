"""HeterPyramidSingle mirror (opencood/models/heter_pyramid_single.py:19-136): HEAL's stage-2 model (`*_single_pyramid.yaml`), a
new agent type trained against the frozen Pyramid Fusion and validated on its own: encoder -> ResNetBEVBackbone -> aligner
(identity or ConvNeXt) -> camera CenterCrop -> PyramidFusion.forward_single -> shrink -> shared heads.  Same ctor argument,
state-dict keys and forward(data_dict) -> output_dict contract; `forward_late` as in heter_model_late.py."""
from collections import OrderedDict

import torch.nn as nn

from .. import ops
from .sub_modules.base_bev_backbone_resnet import ResNetBEVBackbone
from .sub_modules.feature_alignnet import AlignNet
from .sub_modules.downsample_conv import DownsampleConv
from .fuse_modules.pyramid_fuse import PyramidFusion
from .heter_common import HeterFront, add_heads, center_crop_nhwc, modality_names
from .heter_model_late import LateForward


class HeterPyramidSingle(LateForward, HeterFront, nn.Module):
    adapter_name = "aligner"

    def __init__(self, args):
        super().__init__()
        self.modality_name_list = modality_names(args)
        self.cav_range = args['lidar_range']
        self.sensor_type_dict = OrderedDict()
        for m in self.modality_name_list:
            setting = args[m]
            self._add_modality(m, setting, ResNetBEVBackbone(setting['backbone_args']), AlignNet(setting['aligner_args']))
        self.pyramid_backbone = PyramidFusion(args['fusion_backbone'])
        self.shrink_flag = 'shrink_header' in args
        if self.shrink_flag:
            self.shrink_conv = DownsampleConv(args['shrink_header'])
        self._heads = add_heads(self, args['in_head'], args)

    def _any_heads(self):
        return self._heads

    def _base_output(self):
        return {'pyramid': 'single'}

    def _heads_act(self, data_dict, m, extras, out=None):
        f, crop = self._agent_feature(data_dict, m, extras)       # the aligner runs before the crop here
        if crop is not None:
            f = center_crop_nhwc(f, *crop)
        pb = self.pyramid_backbone
        feats = pb.multiscale_nhwc(f)
        extras['occ_single_list'] = [ops.act_to_nchw(pb._occ_nhwc(x, i)) for i, x in enumerate(feats)]
        f = pb.decode_nhwc(feats)
        if self.shrink_flag:
            f = self.shrink_conv.forward_nhwc(f)
        return self._heads.act(f, out=out)
