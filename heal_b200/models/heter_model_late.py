"""HeterModelLate mirror (opencood/models/heter_model_late.py:16-112): the single-agent models of HEAL's `Single/*` configs, one
complete detector per modality (encoder -> ResNetBEVBackbone -> camera CenterCrop -> ResNetBEVBackbone levels 1.. ->
deblocks -> shrink -> own heads).  Same ctor argument (`hypes['model']['args']`), state-dict keys and
forward(data_dict) -> output_dict contract.

`forward_late(batch_data)` runs a late-fusion batch (`{cav_id: cav_content}`, what the late datasets collate and
`inference_late_fusion` loops over) as ONE batched forward per modality present; `LateForward` holds that part, which
HeterPyramidSingle shares."""
from collections import OrderedDict

import torch
import torch.nn as nn

from .. import ops
from ..engine import require_eval
from .sub_modules.base_bev_backbone_resnet import ResNetBEVBackbone
from .sub_modules.downsample_conv import DownsampleConv
from .heter_common import HeterFront, add_heads, center_crop_nhwc, modality_names


def modality_of(data_dict):
    """The modality of a single-agent batch, parsed as the reference does: its one `inputs_*` key through
    `str.lstrip('inputs_')` (which strips a character set, not a prefix: `inputs_m1` -> `m1`)."""
    names = [x for x in data_dict.keys() if x.startswith("inputs_")]
    if len(names) != 1:
        raise ValueError(f"a single-agent batch has exactly one inputs_* key, got {names}")
    return names[0].lstrip('inputs_')


def batch_inputs(inputs):
    """Several cavs' `inputs_<m>` dicts (each one agent) -> one dict of len(inputs) agents in the layout the encoders read from
    the intermediate datasets: voxels concatenated with the agent index in voxel_coords[:, 0] (and `batch_size` set, so the
    encoder needs no host sync), raw clouds concatenated with running `agent_offsets`, camera tensors concatenated on dim 0."""
    if len(inputs) == 1:
        return inputs[0]
    first = inputs[0]
    if 'voxel_features' in first:
        coords = []
        for j, d in enumerate(inputs):
            c = d['voxel_coords'].clone()
            c[:, 0] = j
            coords.append(c)
        return {'voxel_features': torch.cat([d['voxel_features'] for d in inputs], 0),
                'voxel_num_points': torch.cat([d['voxel_num_points'] for d in inputs], 0),
                'voxel_coords': torch.cat(coords, 0), 'batch_size': len(inputs)}
    if 'points' in first:
        out = {k: v for k, v in first.items() if not torch.is_tensor(v)}
        offs, base = [first['agent_offsets'][:1]], 0
        for d in inputs:
            if d['agent_offsets'].numel() != 2:
                raise ValueError("a late-fusion cav carries one cloud (agent_offsets of length 2)")
            offs.append(d['agent_offsets'][1:] + base)
            base += d['points'].shape[0]
        out['points'] = torch.cat([d['points'] for d in inputs], 0)
        out['agent_offsets'] = torch.cat(offs, 0)
        return out
    return {k: torch.cat([d[k] for d in inputs], 0) for k, v in first.items() if torch.is_tensor(v)}


def _slice_cav(v, j, n):
    """Cav j's share of a batched per-cav output: image rows [j*k, (j+1)*k) of every tensor, k = rows / n."""
    if torch.is_tensor(v):
        k = v.shape[0] // n
        return v[j * k:(j + 1) * k]
    if isinstance(v, (list, tuple)):
        return type(v)(_slice_cav(x, j, n) for x in v)
    return v


class LateForward:
    """Late-fusion forward of a single-agent model.  Subclasses provide `_heads_act(data_dict, m, extras, out=None)`: the batched
    forward of modality m up to the fused heads, an f32 Act (n,H,W,A+7A+bins*A) (written into `out` when given), with per-batch
    extra outputs (depth items, occupancy maps) added to `extras`."""

    def late_heads(self, batch_data):
        """-> (cav ids in batch_data order, fused heads Act (n_cav,H,W,S) in that order, {cav_id: extra outputs}).  One forward per
        modality present."""
        require_eval(self)
        cavs = list(batch_data.keys())
        groups = OrderedDict()
        for i, c in enumerate(cavs):
            groups.setdefault(modality_of(batch_data[c]), []).append(i)
        inputs = {m: batch_inputs([batch_data[cavs[i]][f"inputs_{m}"] for i in idx]) for m, idx in groups.items()}
        y, ext = self.grouped_heads(groups, inputs, len(cavs))
        extras = {}
        for m, idx in groups.items():
            for j, i in enumerate(idx):
                extras[cavs[i]] = {k: _slice_cav(v, j, len(idx)) for k, v in ext[m].items()}
        return cavs, y, extras

    def grouped_heads(self, groups, inputs, n_cav):
        """groups {modality: cav positions}, inputs {modality: that group's batched `inputs_<m>`} -> (heads Act (n_cav,H,W,S) with
        image i = cav position i, {modality: batched extra outputs}).  A group whose cavs form one contiguous run writes its heads
        straight into the shared buffer; an interleaved group's heads are copied there per cav (device copies, no host sync)."""
        shared, ext = None, {}
        for m, idx in groups.items():
            ext[m] = {}
            run = shared is not None and idx == list(range(idx[0], idx[-1] + 1))
            y = self._heads_act({f"inputs_{m}": inputs[m]}, m, ext[m], out=shared.images(idx[0], idx[-1] + 1) if run else None)
            if len(groups) == 1:
                return y, ext
            if shared is None:
                shared = ops.act_empty(n_cav, y.H, y.W, y.C, "f32", y.device)
            if not run:
                if (y.H, y.W, y.C) != (shared.H, shared.W, shared.C):
                    raise ValueError(f"modality {m}: heads {(y.H, y.W, y.C)} differ from {(shared.H, shared.W, shared.C)}; "
                                     "late fusion needs one anchor grid")
                for j, i in enumerate(idx):
                    shared.t[i].copy_(y.t[j])
        return shared, ext

    def _split(self, y):
        # every modality's heads have the same A / 7A / bins*A channels (one anchor_number and dir_args per model)
        cls, reg, dirp = self._any_heads().split(y)
        return {'cls_preds': cls, 'reg_preds': reg, 'dir_preds': dirp}

    def forward_late(self, batch_data):
        """`{cav_id: cav_content}` -> OrderedDict `{cav_id: output_dict}` in batch_data order, each as `self(cav_content)` returns
        it (what the reference's inference_late_fusion builds with one model call per cav)."""
        cavs, y, extras = self.late_heads(batch_data)
        out = OrderedDict()
        for j, c in enumerate(cavs):
            out[c] = dict(self._base_output())
            out[c].update(extras[c])
            out[c].update(self._split(y.t[j:j + 1]))
        return out

    def _base_output(self):
        return {}

    def forward(self, data_dict):
        require_eval(self)
        m = modality_of(data_dict)
        ext = {}
        y = self._heads_act(data_dict, m, ext)
        out = dict(self._base_output())
        out.update(ext)
        out.update(self._split(y.t))
        return out


class HeterModelLate(LateForward, HeterFront, nn.Module):
    def __init__(self, args):
        super().__init__()
        self.modality_name_list = modality_names(args)
        self.cav_range = args['lidar_range']
        self.sensor_type_dict = OrderedDict()
        self._heads = {}
        for m in self.modality_name_list:
            setting = args[m]
            self._add_modality(m, setting, ResNetBEVBackbone(setting['backbone_args']))
            setattr(self, f"layers_{m}", ResNetBEVBackbone(setting['layers_args']))
            setattr(self, f"layers_num_{m}", len(setting['layers_args']['num_upsample_filter']))
            setattr(self, f"shrink_conv_{m}", DownsampleConv(setting['shrink_header']))
            self._heads[m] = add_heads(self, setting['head_args']['in_head'], args, f"_{m}")

    def _any_heads(self):
        return next(iter(self._heads.values()))

    def _heads_act(self, data_dict, m, extras, out=None):
        f, crop = self._agent_feature(data_dict, m, extras)
        if crop is not None:
            f = center_crop_nhwc(f, *crop)
        # layer0 of layers_{m} never runs: the backbone's output is the first scale (heter_model_late.py:91-98)
        layers = getattr(self, f"layers_{m}")
        feats = [f]
        for i in range(1, getattr(self, f"layers_num_{m}")):
            for blk in getattr(layers.resnet, f"layer{i}"):
                f = blk.forward_nhwc(f)
            feats.append(f)
        f = getattr(self, f"shrink_conv_{m}").forward_nhwc(layers.decode_nhwc(feats))
        return self._heads[m].act(f, out=out)
