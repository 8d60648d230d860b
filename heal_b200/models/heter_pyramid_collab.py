"""HeterPyramidCollab mirror (opencood/models/heter_pyramid_collab.py:21-209): same ctor argument
(`hypes['model']['args']`), same state-dict keys, same forward(data_dict) -> output_dict contract."""
import importlib
from collections import OrderedDict, Counter

import torch
import torch.nn as nn

from .. import ops
from ..engine import conv_bn_act, require_eval
from ..utils.transformation_utils import normalize_pairwise_tfm
from .sub_modules.base_bev_backbone_resnet import ResNetBEVBackbone
from .sub_modules.feature_alignnet import AlignNet
from .sub_modules.downsample_conv import DownsampleConv
from .sub_modules.naive_compress import NaiveCompressor
from .fuse_modules.pyramid_fuse import PyramidFusion


class FusedHeads:
    """cls/reg/dir 1x1 heads evaluated as one conv with concatenated output channels."""

    def __init__(self, heads):
        self.heads = heads
        self._conv = None
        self._sig = None

    def prepare(self):
        """(Re)build the concatenated 1x1 conv when a head's parameters changed."""
        from ..engine import _sig
        sig = _sig(*self.heads)
        if self._conv is None or self._sig != sig:
            cin = self.heads[0].in_channels
            cout = sum(h.out_channels for h in self.heads)
            conv = nn.Conv2d(cin, cout, 1).to(self.heads[0].weight.device)
            with torch.no_grad():
                conv.weight.copy_(torch.cat([h.weight for h in self.heads], 0))
                conv.bias.copy_(torch.cat([h.bias for h in self.heads], 0))
            self._conv, self._sig = conv, sig

    def act(self, x_nhwc, out=None):
        """The fused (B,H,W,sum) fp32 output as an Act; `out` may be an f32 Act of that shape (e.g. images of a larger buffer)."""
        self.prepare()
        return conv_bn_act(x_nhwc, self._conv, None, relu=False, out=out, out_fmt="f32")

    def split(self, y):
        """(B,H,W,sum) fp32 -> one logical-NCHW tensor per head."""
        outs, o = [], 0
        for h in self.heads:
            outs.append(y[..., o:o + h.out_channels].permute(0, 3, 1, 2).contiguous())
            o += h.out_channels
        return outs

    def __call__(self, x_nhwc):
        return self.split(self.act(x_nhwc).t)


class HeterPyramidCollab(nn.Module):
    def __init__(self, args):
        super().__init__()
        self.args = args
        self.modality_name_list = [x for x in args.keys() if x.startswith("m") and x[1:].isdigit()]
        self.cav_range = args['lidar_range']
        self.sensor_type_dict = OrderedDict()
        self.cam_crop_info = {}
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
                self.cam_crop_info[m] = {f"crop_ratio_W_{m}": getattr(self, f"crop_ratio_W_{m}"),
                                         f"crop_ratio_H_{m}": getattr(self, f"crop_ratio_H_{m}")}
        self.H = self.cav_range[4] - self.cav_range[1]
        self.W = self.cav_range[3] - self.cav_range[0]
        self.fake_voxel_size = 1
        self.pyramid_backbone = PyramidFusion(args['fusion_backbone'])
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

    def model_train_init(self):
        """The reference's: with a compressor, freeze everything and leave only the compressor in train mode (the forward then
        refuses to run until `.eval()`: training is not implemented)."""
        if self.compress:
            self.eval()
            for p in self.parameters():
                p.requires_grad_(False)
            self.compressor.train()
            for p in self.compressor.parameters():
                p.requires_grad_(True)

    @staticmethod
    def _center_crop_nhwc(act, th, tw):
        """torchvision CenterCrop semantics on a channels-last map: crops, or zero-pads when the target is larger
        (heter_pyramid_collab.py:153-163).  Layout plumbing on the fp32 view."""
        f = ops.convert(act, "f32").t
        f = HeterPyramidCollab._crop_tensor(f, th, tw)
        return ops.Act(f, "f32")

    @staticmethod
    def _crop_tensor(f, th, tw):
        n, h, w, c = f.shape
        if th > h or tw > w:
            pl, pt = (tw - w) // 2 if tw > w else 0, (th - h) // 2 if th > h else 0
            pr, pb = (tw - w + 1) // 2 if tw > w else 0, (th - h + 1) // 2 if th > h else 0
            f = torch.nn.functional.pad(f, (0, 0, pl, pr, pt, pb))
            n, h, w, c = f.shape
            if th == h and tw == w:
                return f.contiguous()
        top, left = int(round((h - th) / 2.0)), int(round((w - tw) / 2.0))
        return f[:, top:top + th, left:left + tw, :].contiguous()

    def forward(self, data_dict):
        require_eval(self)
        output_dict = {'pyramid': 'collab'}
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
            f = bb.decode_nhwc(bb.multiscale_nhwc(f))                             # Act
            f = getattr(self, f"aligner_{m}").forward_nhwc(f)                     # identity, or the ConvNeXt aligner (HEAL stage 2)
            if self.sensor_type_dict[m] == "camera":
                crops[m] = (int(f.H * getattr(self, f"crop_ratio_H_{m}")), int(f.W * getattr(self, f"crop_ratio_W_{m}")))
                if getattr(self, f"depth_supervision_{m}"):
                    output_dict[f"depth_items_{m}"] = getattr(self, f"encoder_{m}").depth_items
            feats[m] = f
        if len(feats) == 1 and all(a == aml[0] for a in aml) and not crops:
            x = feats[aml[0]]
        else:                                   # fp32 (n_agents, H, W, C) in scene order, camera maps cropped / padded
            x = ops.agent_stack(feats, aml, crops)
        if self.compress:
            x = self.compressor.forward_nhwc(x)
        fused, occs = self.pyramid_backbone.forward_collab_nhwc(x, record_len, affine, aml, self.cam_crop_info)
        if self.shrink_flag:
            fused = self.shrink_conv.forward_nhwc(fused)
        cls, reg, dirp = self._heads(fused)
        output_dict.update({'cls_preds': cls, 'reg_preds': reg, 'dir_preds': dirp})
        output_dict['occ_single_list'] = [ops.act_to_nchw(o) for o in occs]
        return output_dict
