"""GPU mirror of opencood/data_utils/post_processor/voxel_postprocessor.py (VoxelPostprocessor, inference side).

Same constructor (`anchor_params`, `train`), `generate_anchor_box()` and `post_process(data_dict, output_dict)` as the reference
(:26-83, :245-405); the decode / filter / rotated-NMS chain runs in one C-ABI call (heal_box_decode_nms, csrc/postprocess.cu) on the
head outputs where they already live -- the reference copies them to the host and loops over shapely polygons.
`generate_label` (training targets) is out of scope and raises."""
from __future__ import annotations

import math

import numpy as np
import torch

from ... import ops

TOP = 1000          # decode capacity: the best-scoring candidates kept for NMS (box_utils.nms_rotated's `top`)


def decode_kwargs(params, has_dir: bool):
    """The keyword arguments ops.box_decode_nms, box_decode_nms_multi and box_decode_nms_late take from a `postprocess:` block:
    thresholds, box order, range mask, capacity TOP, and the direction-bin correction of `dir_args` when the heads have a dir
    head."""
    dargs = params.get('dir_args', {}) if has_dir else {}
    return dict(score_threshold=params['target_args']['score_threshold'], nms_threshold=params['nms_thresh'],
                dir_offset=dargs.get('dir_offset', 0.0), num_bins=dargs.get('num_bins', 2), order=params['order'],
                gt_range=params['gt_range'], top=TOP)


class VoxelPostprocessor:
    def __init__(self, anchor_params, train):
        self.params = anchor_params
        self.train = train
        self.anchor_num = self.params['anchor_args']['num']
        self._buffers = {}
        self._anchors_dev = {}

    # -- voxel_postprocessor.py:30-83 -----------------------------------------------------------
    def generate_anchor_box(self):
        aa = self.params['anchor_args']
        W, H = aa['W'], aa['H']
        r = [math.radians(e) for e in aa['r']]
        assert self.anchor_num == len(r)
        vh, vw = aa['vh'], aa['vw']
        xrange = [aa['cav_lidar_range'][0], aa['cav_lidar_range'][3]]
        yrange = [aa['cav_lidar_range'][1], aa['cav_lidar_range'][4]]
        stride = aa.get('feature_stride', 2)
        x = np.linspace(xrange[0] + vw, xrange[1] - vw, W // stride)
        y = np.linspace(yrange[0] + vh, yrange[1] - vh, H // stride)
        cx, cy = np.meshgrid(x, y)
        cx = np.tile(cx[..., np.newaxis], self.anchor_num)
        cy = np.tile(cy[..., np.newaxis], self.anchor_num)
        cz = np.ones_like(cx) * -1.0
        w, l, h = np.ones_like(cx) * aa['w'], np.ones_like(cx) * aa['l'], np.ones_like(cx) * aa['h']
        r_ = np.ones_like(cx)
        for i in range(self.anchor_num):
            r_[..., i] = r[i]
        if self.params['order'] == 'hwl':
            return np.stack([cx, cy, cz, h, w, l, r_], axis=-1)
        if self.params['order'] == 'lhw':
            return np.stack([cx, cy, cz, l, h, w, r_], axis=-1)
        raise ValueError('Unknown bbx order.')

    def generate_label(self, **kwargs):
        raise NotImplementedError("heal_b200 covers the inference path; training targets stay in opencood")

    # -- voxel_postprocessor.py:245-405 ---------------------------------------------------------
    def _decode_many(self, data_dict, output_dict):
        """several cavs (late fusion) and / or iou_preds: heal_box_decode_nms_multi"""
        cavs, dirs = [], []
        for cav, out in output_dict.items():
            cls = out.get('cls_preds', out.get('psm'))
            reg = out.get('reg_preds', out.get('rm'))
            if reg.dim() != 4:
                raise NotImplementedError("anchor-free (CenterPoint) heads are not part of the GPU post-processor")
            dirp = out.get('dir_preds', out.get('dm'))
            dirs.append(dirp is not None)
            cavs.append({"cls": cls, "reg": reg, "dir": dirp, "iou": out.get('iou_preds'),
                         "anchors": self._device_anchors(data_dict[cav]['anchor_box'], cls.device),
                         "transform": data_dict[cav]['transformation_matrix']})
        A, H, W = cavs[0]["cls"].shape[1], cavs[0]["cls"].shape[2], cavs[0]["cls"].shape[3]
        bkey = (H * len(cavs), W, A, str(cavs[0]["cls"].device))
        if bkey not in self._buffers:
            self._buffers[bkey] = ops.PostprocessBuffers(H * len(cavs), W, A, TOP, cavs[0]["cls"].device)
        return ops.box_decode_nms_multi(cavs, **decode_kwargs(self.params, any(dirs)), buffers=self._buffers[bkey])

    def _decode_one(self, cav_content, out):
        cls = out.get('cls_preds', out.get('psm'))
        reg = out.get('reg_preds', out.get('rm'))
        dirp = out.get('dir_preds', out.get('dm'))
        if 'iou_preds' in out:
            raise NotImplementedError("use _decode_many for iou_preds rescoring")
        if reg.dim() != 4:
            raise NotImplementedError("anchor-free (CenterPoint) heads are not part of the GPU post-processor")
        dev = cls.device
        anchors = self._device_anchors(cav_content['anchor_box'], dev)
        A, H, W = cls.shape[1], cls.shape[2], cls.shape[3]
        bkey = (H, W, A, str(dev))
        if bkey not in self._buffers:
            self._buffers[bkey] = ops.PostprocessBuffers(H, W, A, TOP, dev)
        return ops.box_decode_nms(cls, reg, dirp, anchors, cav_content['transformation_matrix'],
                                  **decode_kwargs(self.params, dirp is not None), buffers=self._buffers[bkey])

    def _device_anchors(self, anchor, dev):
        """fp32 device copy of the anchor grid, cached per (shape, device).  The reference's collate builds a NEW anchor tensor for
        every batch (intermediate_heter_fusion_dataset.py:704), so neither its data_ptr nor its id identifies the contents: the
        cache keeps the source values and re-uploads when they differ (one small host compare per frame, no unbounded growth)."""
        src = torch.as_tensor(anchor)
        key = (tuple(src.shape), str(dev))
        hit = self._anchors_dev.get(key)
        if hit is not None:
            same = (hit[0] is src) or (hit[0].device == src.device and hit[0].dtype == src.dtype and torch.equal(hit[0], src))
            if same:
                return hit[1]
        devt = src.to(device=dev, dtype=torch.float32).contiguous()
        self._anchors_dev[key] = (src.detach().clone(), devt)
        return devt

    def post_process(self, data_dict, output_dict):
        """Returns (pred_box3d_tensor (K,8,3), scores (K,)) on the device, or (None, None).  One cav (early / intermediate fusion:
        the ego) or several (late fusion: every cav's boxes projected to ego, one NMS over all of them), with optional iou_preds."""
        cavs = list(output_dict.keys())
        assert all(c in data_dict for c in cavs)
        if len(cavs) != 1 or 'iou_preds' in output_dict[cavs[0]]:
            buf = self._decode_many(data_dict, output_dict)          # late fusion: NMS across all cavs' boxes; iou rescoring
        else:
            buf = self._decode_one(data_dict[cavs[0]], output_dict[cavs[0]])
        # the only host sync of the call: box count + candidate count in ONE device-to-host copy (the reference-shaped return
        # needs the box count; the 4x4 transform is host metadata in the reference's collate and is read before the launch)
        k, above = torch.cat([buf.count, buf.stats[:1]]).tolist()
        if above == 0:                               # nothing above the score threshold (voxel_postprocessor.py:351-352)
            return None, None
        return buf.boxes[:k].clone(), buf.scores[:k].clone()


def make_reference_subclass(ref_cls):
    """Build the class the registry hook installs: a SUBCLASS of the reference's own VoxelPostprocessor (so the datasets keep
    generate_label / generate_gt_bbx / generate_object_center* / collate_batch, which they call on the inference path too:
    intermediate_heter_fusion_dataset.py:179,458,537,666,781; opv2v_basedataset.py:435) whose `post_process` runs on the GPU
    when it can (anchor-based heads of equal geometry on a CUDA device: one cav, or several = late fusion, with or without
    iou_preds) and defers to the reference implementation otherwise (CPU tensors, anchor-free heads)."""
    gpu = VoxelPostprocessor

    class GpuVoxelPostprocessor(ref_cls):
        def __init__(self, anchor_params, train):
            super().__init__(anchor_params, train)
            self._gpu = gpu(anchor_params, train)

        @staticmethod
        def _gpu_eligible(output_dict):
            if not (1 <= len(output_dict) <= 16):
                return False
            shape = None
            for out in output_dict.values():
                cls = out.get('cls_preds', out.get('psm'))
                reg = out.get('reg_preds', out.get('rm'))
                if not (torch.is_tensor(cls) and cls.is_cuda and torch.is_tensor(reg) and reg.dim() == 4):
                    return False
                if shape is not None and tuple(cls.shape) != shape:
                    return False                      # cavs with different head geometry: reference path
                shape = tuple(cls.shape)
            return True

        def post_process(self, data_dict, output_dict):
            if self._gpu_eligible(output_dict):
                return self._gpu.post_process(data_dict, output_dict)
            return super().post_process(data_dict, output_dict)

    GpuVoxelPostprocessor.__name__ = "VoxelPostprocessor"
    return GpuVoxelPostprocessor
