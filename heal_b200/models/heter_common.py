"""What the HEAL mirrors (HeterPyramidCollab, HeterModelBaseline, HeterModelBaselineMs, HeterModelLate, HeterPyramidSingle) have
in common: the encoder lookup, the cls/reg/dir heads run as one fused 1x1 conv, the camera CenterCrop, and `HeterFront`, the
per-modality front (encoder -> backbone -> aligner or shrinker) and the agent assembly of an intermediate-fusion scene."""
import importlib

import torch
import torch.nn as nn

from .. import ops
from ..engine import conv_bn_act


def modality_names(args):
    """The modality keys of a model's args (`m1`, `m2`, ...), in args order."""
    return [x for x in args.keys() if x.startswith("m") and x[1:].isdigit()]


def build_encoder(setting):
    encoder_lib = importlib.import_module("heal_b200.models.heter_encoders")
    target = setting['core_method'].replace('_', '').lower()
    enc_cls = next((c for n, c in encoder_lib.__dict__.items() if n.lower() == target), None)
    if enc_cls is None:
        raise NotImplementedError(f"encoder '{setting['core_method']}' not available in heal_b200.models.heter_encoders")
    return enc_cls(setting['encoder_args'])


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


def add_heads(module, in_ch, args, suffix="", use_dir=True):
    """Set `cls_head{suffix}`, `reg_head{suffix}` and (with use_dir) `dir_head{suffix}` on module, in that order (the reference's
    state-dict order), and return them as one FusedHeads."""
    a = args['anchor_number']
    heads = [nn.Conv2d(in_ch, a, kernel_size=1), nn.Conv2d(in_ch, 7 * a, kernel_size=1)]
    if use_dir:
        heads.append(nn.Conv2d(in_ch, args['dir_args']['num_bins'] * a, kernel_size=1))
    for name, h in zip(("cls", "reg", "dir"), heads):
        setattr(module, f"{name}_head{suffix}", h)
    return FusedHeads(heads)


def crop_tensor(f, th, tw):
    """torchvision CenterCrop semantics on a (N,H,W,C) tensor: crops, or zero-pads when the target is larger
    (heter_pyramid_collab.py:153-163)."""
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


def center_crop_nhwc(act, th, tw):
    """CenterCrop of an Act, as an fp32 Act (layout plumbing on the fp32 view)."""
    return ops.Act(crop_tensor(ops.convert(act, "f32").t, th, tw), "f32")


class HeterFront:
    """The per-modality front of a HEAL mirror (an nn.Module that sets `cav_range` and an empty `sensor_type_dict` before
    adding modalities).  `adapter_name` names the per-modality module run after the backbone: "aligner", "shrinker" or None."""
    adapter_name = None

    def _add_modality(self, m, setting, backbone, adapter=None):
        """Register modality m: `encoder_{m}`, `depth_supervision_{m}`, `backbone_{m}`, the adapter `{adapter_name}_{m}` when
        given, and for a camera the CenterCrop ratios of its map to the lidar range."""
        self.sensor_type_dict[m] = setting['sensor_type']
        setattr(self, f"encoder_{m}", build_encoder(setting))
        setattr(self, f"depth_supervision_{m}", bool(setting['encoder_args'].get("depth_supervision", False)))
        setattr(self, f"backbone_{m}", backbone)
        if adapter is not None:
            setattr(self, f"{self.adapter_name}_{m}", adapter)
        if setting['sensor_type'] == "camera":
            g = setting['camera_mask_args']['grid_conf']
            setattr(self, f"crop_ratio_W_{m}", self.cav_range[3] / g['xbound'][1])
            setattr(self, f"crop_ratio_H_{m}", self.cav_range[4] / g['ybound'][1])

    def _encode(self, data_dict, m):
        """encoder -> backbone (resnet + deblocks) of modality m, as an Act."""
        enc = getattr(self, f"encoder_{m}")
        f = enc.forward_act(data_dict, m) if hasattr(enc, "forward_act") else ops.to_act(enc(data_dict, m))
        bb = getattr(self, f"backbone_{m}")
        return bb.decode_nhwc(bb.multiscale_nhwc(f))

    def _agent_feature(self, data_dict, m, out):
        """-> (modality m's map after the adapter, its camera CenterCrop size (H, W) or None); adds `depth_items_{m}` to out
        when the camera's depth is supervised."""
        f = self._encode(data_dict, m)
        if self.adapter_name is not None:
            f = getattr(self, f"{self.adapter_name}_{m}").forward_nhwc(f)
        if self.sensor_type_dict[m] != "camera":
            return f, None
        if getattr(self, f"depth_supervision_{m}"):
            out[f"depth_items_{m}"] = getattr(self, f"encoder_{m}").depth_items
        return f, (int(f.H * getattr(self, f"crop_ratio_H_{m}")), int(f.W * getattr(self, f"crop_ratio_W_{m}")))

    def _assemble(self, data_dict, out):
        """The scene's per-agent maps as one Act in scene order.  A single-modality scene without a crop keeps its map in the
        engine format; otherwise heal_agent_stack gathers fp32 (n_agents, H, W, C), camera maps cropped / padded."""
        aml = data_dict['agent_modality_list']
        feats, crops = {}, {}
        for m in self.modality_name_list:
            if m not in aml:
                continue
            feats[m], crop = self._agent_feature(data_dict, m, out)
            if crop is not None:
                crops[m] = crop
        if len(feats) == 1 and all(a == aml[0] for a in aml) and not crops:
            return feats[aml[0]]
        return ops.agent_stack(feats, aml, crops)

    def model_train_init(self):
        """The reference's: with a compressor, freeze everything and leave only the compressor in train mode (the forward then
        refuses to run until `.eval()`: training is not implemented)."""
        if getattr(self, "compress", False):
            self.eval()
            for p in self.parameters():
                p.requires_grad_(False)
            self.compressor.train()
            for p in self.compressor.parameters():
                p.requires_grad_(True)
