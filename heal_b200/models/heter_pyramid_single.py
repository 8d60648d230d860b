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
from .heter_pyramid_collab import FusedHeads
from .heter_model_late import LateForward, build_encoder, crop_camera, encode


class HeterPyramidSingle(LateForward, nn.Module):
    def __init__(self, args):
        super().__init__()
        self.modality_name_list = [x for x in args.keys() if x.startswith("m") and x[1:].isdigit()]
        self.cav_range = args['lidar_range']
        self.sensor_type_dict = OrderedDict()
        for m in self.modality_name_list:
            setting = args[m]
            self.sensor_type_dict[m] = setting['sensor_type']
            setattr(self, f"encoder_{m}", build_encoder(setting))
            setattr(self, f"depth_supervision_{m}", bool(setting['encoder_args'].get("depth_supervision", False)))
            setattr(self, f"backbone_{m}", ResNetBEVBackbone(setting['backbone_args']))
            if setting['sensor_type'] == "camera":
                g = setting['camera_mask_args']['grid_conf']
                setattr(self, f"crop_ratio_W_{m}", self.cav_range[3] / g['xbound'][1])
                setattr(self, f"crop_ratio_H_{m}", self.cav_range[4] / g['ybound'][1])
            setattr(self, f"aligner_{m}", AlignNet(setting['aligner_args']))
        self.pyramid_backbone = PyramidFusion(args['fusion_backbone'])
        self.shrink_flag = 'shrink_header' in args
        if self.shrink_flag:
            self.shrink_conv = DownsampleConv(args['shrink_header'])
        self.cls_head = nn.Conv2d(args['in_head'], args['anchor_number'], kernel_size=1)
        self.reg_head = nn.Conv2d(args['in_head'], 7 * args['anchor_number'], kernel_size=1)
        self.dir_head = nn.Conv2d(args['in_head'], args['dir_args']['num_bins'] * args['anchor_number'], kernel_size=1)
        self._heads = FusedHeads([self.cls_head, self.reg_head, self.dir_head])

    def model_train_init(self):
        pass

    def _any_heads(self):
        return self._heads

    def _base_output(self):
        return {'pyramid': 'single'}

    def _heads_act(self, data_dict, m, extras, out=None):
        f = getattr(self, f"aligner_{m}").forward_nhwc(encode(self, data_dict, m))   # the aligner runs before the crop here
        f = crop_camera(self, f, m, extras)
        pb = self.pyramid_backbone
        feats = pb.multiscale_nhwc(f)
        extras['occ_single_list'] = [ops.act_to_nchw(pb._occ_nhwc(x, i)) for i, x in enumerate(feats)]
        f = pb.decode_nhwc(feats)
        if self.shrink_flag:
            f = self.shrink_conv.forward_nhwc(f)
        return self._heads.act(f, out=out)
