"""Per-modality encoders with the reference's `(data_dict, modality_name) -> (n,C,H,W)` signature
(opencood/models/heter_encoders.py:22-301).  PointPillar runs PillarVFE + scatter as one kernel; Lift-Splat-Shoot builds either of
the reference's camera encoders (`camera_encoder: EfficientNet` -> CamEncode, `Resnet101` -> CamEncode_Resnet101)."""
import os as _os

import numpy as np
import torch
import torch.nn as nn

from .. import ops
from ..engine import require_eval
from .sub_modules.pillar_vfe import PillarVFE
from .sub_modules.point_pillar_scatter import PointPillarScatter


class PointPillar(nn.Module):
    """heter_encoders.py:22-50.  If `inputs_<m>` holds raw points (`points`, `agent_offsets`) instead of
    CPU-voxelised tensors, voxelisation runs on the GPU first (SURVEY.md 7.2 'Boundary vs DataLoader workers')."""

    def __init__(self, args):
        super().__init__()
        grid_size = (np.array(args['lidar_range'][3:6]) - np.array(args['lidar_range'][0:3])) / np.array(args['voxel_size'])
        grid_size = np.round(grid_size).astype(np.int64)
        args['point_pillar_scatter']['grid_size'] = grid_size
        self.pillar_vfe = PillarVFE(args['pillar_vfe'], num_point_features=4, voxel_size=args['voxel_size'],
                                    point_cloud_range=args['lidar_range'])
        self.scatter = PointPillarScatter(args['point_pillar_scatter'])
        self.voxel_size = [float(v) for v in args['voxel_size']]
        self.lidar_range = [float(v) for v in args['lidar_range']]
        self.voxelize_args = args.get('voxelize', {'max_points_per_voxel': 32, 'max_voxels': 70000})

    def forward(self, data_dict, modality_name):
        """reference signature: returns the (n, C, ny, nx) BEV map (logical NCHW, physically channels-last fp32)."""
        return ops.act_to_nchw(self.forward_act(data_dict, modality_name, fmt="f32", sparse=False))

    def forward_act(self, data_dict, modality_name, fmt=None, sparse=None):
        """internal path: the canvas as an `Act` in the conv engine's activation format (no conversion pass), or - when the
        sparse stem is on - as an `ops.SparseCanvas` (pillar features + id map) that the first residual block consumes."""
        from .. import engine
        from ..engine import act_fmt
        fmt = fmt or act_fmt()
        sparse = engine.SPARSE_STEM if sparse is None else sparse
        require_eval(self)
        inp = data_dict[f'inputs_{modality_name}']
        nvox_dev = None
        if 'voxel_features' in inp:
            vf, vc, vn = inp['voxel_features'], inp['voxel_coords'], inp['voxel_num_points']
            batch_size = inp.get('batch_size')
            if batch_size is None:
                batch_size = int(vc[:, 0].max().item()) + 1     # host sync, as the reference (scatter.py:45)
        else:
            pts, offs = ops.raw_points_of(inp, self.lidar_range)
            vf, vc, vn, nvox_dev = ops.voxelize(pts, offs, self.lidar_range, self.voxel_size,
                                                int(inp.get('max_points_per_voxel', self.voxelize_args['max_points_per_voxel'])),
                                                int(inp.get('max_voxels', self.voxelize_args['max_voxels'])))
            batch_size = offs.numel() - 1
        w, b = self.pillar_vfe.folded()
        if sparse:
            return ops.pillar_vfe_sparse(vf, vn, vc, w, b, self.voxel_size, self.lidar_range, nx=self.scatter.nx,
                                         ny=self.scatter.ny, batch_size=batch_size, num_voxels_dev=nvox_dev,
                                         want_split_rows=(ops.STEM_GATHER_TC and fmt == "split"))
        _, canvas = ops.pillar_vfe_scatter(vf, vn, vc, w, b, self.voxel_size, self.lidar_range,
                                           nx=self.scatter.nx, ny=self.scatter.ny, batch_size=batch_size,
                                           num_voxels_dev=nvox_dev, canvas_fmt=fmt)
        return canvas


# ---------------------------------------------------------------------------------------------------------
# Lift-Splat-Shoot camera encoder
# ---------------------------------------------------------------------------------------------------------
def gen_dx_bx(xbound, ybound, zbound):
    """opencood/utils/camera_utils.py:129-134 (fp32 tensors, same construction)."""
    dx = torch.Tensor([row[2] for row in [xbound, ybound, zbound]])
    bx = torch.Tensor([row[0] + row[2] / 2.0 for row in [xbound, ybound, zbound]])
    nx = torch.LongTensor([(row[1] - row[0]) / row[2] for row in [xbound, ybound, zbound]])
    return dx, bx, nx


def depth_discretization(depth_min, depth_max, num_bins, mode):
    """opencood/utils/camera_utils.py:187-196."""
    if mode == "UD":
        return depth_min + (depth_max - depth_min) / num_bins * np.arange(num_bins)
    if mode == "LID":
        bin_size = 2 * (depth_max - depth_min) / (num_bins * (1 + num_bins))
        return depth_min + bin_size * (np.arange(num_bins) * np.arange(1, 1 + num_bins)) / 2
    raise NotImplementedError(mode)


class CamEncode_Resnet101(nn.Module):
    """Image trunk + depth / image heads (opencood/models/sub_modules/lss_submodule.py:140-233), same attribute
    names -> same state-dict keys (the torchvision modules are parameter containers).  `heads_nhwc` runs the whole trunk on
    the conv engine (SURVEY.md 8f-2):
      conv1 7x7/2 + bn1 + ReLU   as a 3x3 convolution on the 4x4 space-to-depth image (3 -> 64 input channels, 4 output phases
                                 x 64 channels): a wgmma shape instead of a K = 3 stem; exact re-indexing of the same sums
      maxpool 3x3/2              heal_maxpool3x3s2 reading the phase-major stem output directly
      layer1, layer2             torchvision Bottlenecks: 1x1 / 3x3 (stride) / 1x1 + residual, each conv+BN(+ReLU) one kernel
      depth_head | image_head    one fused 1x1 convolution 512 -> D + C, fp32 channels-last output
    The depth softmax (x) feature outer product that follows is NOT computed here - it is fused into the BEV-pool kernel.
    `heads` keeps the plain torch path (CPU-capable; the tests' oracle trunk)."""

    def __init__(self, D, C, downsample, ddiscr, mode, use_gt_depth=False, depth_supervision=True):
        super().__init__()
        from torchvision.models.resnet import resnet101
        self.D, self.C, self.downsample = D, C, downsample
        self.d_min, self.d_max, self.num_bins = ddiscr[0], ddiscr[1], ddiscr[2]
        self.mode, self.use_gt_depth, self.depth_supervision = mode, use_gt_depth, depth_supervision
        trunk = resnet101(weights=None, zero_init_residual=True)
        self.conv1, self.bn1, self.relu, self.maxpool = trunk.conv1, trunk.bn1, nn.ReLU(), trunk.maxpool
        self.layer1, self.layer2, self.layer3 = trunk.layer1, trunk.layer2, nn.Identity()
        if use_gt_depth:
            raise NotImplementedError("use_depth_gt is a training-time option outside the inference hot path")
        self.depth_head = nn.Conv2d(512, self.D, kernel_size=1, padding=0)
        self.image_head = nn.Conv2d(512, self.C, kernel_size=1, padding=0)

    def heads(self, x):
        """x (BN, 3|4, H, W) -> (depth_logits (BN,D,fH,fW), feat (BN,C,fH,fW))"""
        f = self.layer2(self.layer1(self.maxpool(self.relu(self.bn1(self.conv1(x[:, :3].clone()))))))
        return self.depth_head(f), self.image_head(f)

    # ---- conv-engine path -------------------------------------------------------------------------------------------
    def _stem_as_s2d_conv(self):
        """conv1 (64,3,7,7, stride 2, pad 3) + bn1 folded -> Conv2d(64, 256, 3, pad 1, bias) acting on pixel_unshuffle(x, 4):
        input channel = c*16 + dy*4 + dx (c < 3; c == 3 is zero padding), output channel = (py*2 + px)*64 + co where the
        output pixel is (2Y + py, 2X + px).  out(2Y+py, 2X+px) = sum_{r,s} W[r,s] in(4Y + 2py - 3 + r, 4X + 2px - 3 + s):
        with block offset b in {-1,0,1} and in-block row d, r = 4b + d - 2py + 3."""
        from ..engine import _sig
        sig = _sig(self.conv1, self.bn1)
        hit = getattr(self, "_stem_cache", None)
        if hit is not None and hit[0] == sig:
            return hit[1]
        w = self.conv1.weight.detach().double().cpu()                       # (64, 3, 7, 7)
        bn = self.bn1
        scale = bn.weight.detach().double().cpu() / torch.sqrt(bn.running_var.detach().double().cpu() + bn.eps)
        shift = bn.bias.detach().double().cpu() - bn.running_mean.detach().double().cpu() * scale
        w = w * scale[:, None, None, None]
        wn = torch.zeros((4, 64, 4, 16, 3, 3), dtype=torch.float64)          # (phase, co, c, dy*4+dx, by, bx)
        for py in range(2):
            for px in range(2):
                for by in range(3):
                    for dy in range(4):
                        r = 4 * (by - 1) + dy - 2 * py + 3
                        if not (0 <= r < 7):
                            continue
                        for bx in range(3):
                            for dx in range(4):
                                q = 4 * (bx - 1) + dx - 2 * px + 3
                                if 0 <= q < 7:
                                    wn[py * 2 + px, :, :3, dy * 4 + dx, by, bx] = w[:, :, r, q]
        conv = nn.Conv2d(64, 256, 3, padding=1, bias=True)
        with torch.no_grad():
            conv.weight.copy_(wn.reshape(256, 64, 3, 3).float())
            conv.bias.copy_(shift.repeat(4).float())
        conv = conv.to(self.conv1.weight.device)
        self.__dict__["_stem_cache"] = (sig, conv)                            # not a registered submodule: no state-dict keys
        return conv

    def _fused_heads(self):
        from ..engine import _sig
        sig = _sig(self.depth_head, self.image_head)
        hit = getattr(self, "_heads_cache", None)
        if hit is not None and hit[0] == sig:
            return hit[1]
        conv = nn.Conv2d(512, self.D + self.C, 1).to(self.depth_head.weight.device)
        with torch.no_grad():
            conv.weight.copy_(torch.cat([self.depth_head.weight, self.image_head.weight], 0))
            conv.bias.copy_(torch.cat([self.depth_head.bias, self.image_head.bias], 0))
        self.__dict__["_heads_cache"] = (sig, conv)
        return conv

    @staticmethod
    def _bottleneck_nhwc(blk, x):
        """torchvision.models.resnet.Bottleneck.forward on the conv engine (stride on the 3x3, ResNet v1.5)."""
        from ..engine import conv_bn_act
        idt = x
        if blk.downsample is not None:
            idt = conv_bn_act(x, blk.downsample[0], blk.downsample[1], relu=False)
        y = conv_bn_act(x, blk.conv1, blk.bn1, relu=True)
        y = conv_bn_act(y, blk.conv2, blk.bn2, relu=True)
        return conv_bn_act(y, blk.conv3, blk.bn3, relu=True, residual=idt)

    def heads_nhwc(self, x, plan=None):
        """x (BN, 3|4, H, W) fp32 CUDA -> Act f32 (BN, H/8, W/8, D + C): [depth logits | image features] per pixel.  With a `plan`
        (data_utils.camera_input.inference_plan), x is raw uint8 frames (BN, H0, W0, 3): heal_camera_input resizes, crops and
        normalises them straight into the stem's space-to-depth layout."""
        from ..engine import conv_bn_act
        if plan is not None:
            H, W = plan.final_dim
            if (H % 8) or (W % 8):
                raise NotImplementedError("image sides must be multiples of 8 (the LSS yamls use img_downsample 8)")
            a = ops.camera_input(x, plan, "s2d")                                # (BN, H/4, W/4, 64)
        else:
            BN, Cx, H, W = x.shape
            if (H % 8) or (W % 8):
                raise NotImplementedError("image sides must be multiples of 8 (the LSS yamls use img_downsample 8)")
            x4 = torch.zeros((BN, 4, H, W), dtype=torch.float32, device=x.device)
            x4[:, :3] = x[:, :3]
            a = ops.to_act(torch.nn.functional.pixel_unshuffle(x4, 4))      # (BN, H/4, W/4, 64): layout plumbing of the raw image
        y = conv_bn_act(a, self._stem_as_s2d_conv(), None, relu=True)         # phase-major (BN, H/4, W/4, 4*64) = logical (BN, H/2, W/2, 64)
        y = ops.maxpool3x3s2(y, depth_to_space_in=True)                       # (BN, H/4, W/4, 64)
        for blk in self.layer1:
            y = self._bottleneck_nhwc(blk, y)
        for blk in self.layer2:
            y = self._bottleneck_nhwc(blk, y)
        return conv_bn_act(y, self._fused_heads(), None, relu=False, out_fmt="f32")


class Up(nn.Module):
    """lss_submodule.py:17-36: bilinear x2 (align_corners=True) of x1, cat([x2, x1_up]), two conv3x3 + BN + ReLU.  `forward_nhwc`
    writes the concatenation once, in the conv engine's activation format with the channel count rounded up to a multiple of 64
    (heal_upsample2x_concat), so both convolutions are tensor-core shapes."""

    def __init__(self, in_channels, out_channels, scale_factor=2):
        super().__init__()
        self.up = nn.Upsample(scale_factor=scale_factor, mode='bilinear', align_corners=True)
        self.conv = nn.Sequential(
            nn.Conv2d(in_channels, out_channels, kernel_size=3, padding=1, bias=False), nn.BatchNorm2d(out_channels), nn.ReLU(inplace=True),
            nn.Conv2d(out_channels, out_channels, kernel_size=3, padding=1, bias=False), nn.BatchNorm2d(out_channels), nn.ReLU(inplace=True))

    def forward(self, x1, x2):
        return self.conv(torch.cat([x2, self.up(x1)], dim=1))

    def _first_conv_padded(self):
        """conv[0] with zero weights for the input channels that pad the concatenation to a multiple of 64."""
        from ..engine import _sig
        src = self.conv[0]
        sig = _sig(src)
        hit = self.__dict__.get("_conv0_cache")
        if hit is not None and hit[0] == sig:
            return hit[1]
        cin = (src.in_channels + 63) // 64 * 64
        conv = nn.Conv2d(cin, src.out_channels, 3, padding=1, bias=False).to(src.weight.device)
        with torch.no_grad():
            conv.weight.zero_()
            conv.weight[:, :src.in_channels].copy_(src.weight)
        self.__dict__["_conv0_cache"] = (sig, conv)                          # not a registered submodule: no state-dict keys
        return conv

    def forward_nhwc(self, x1, x2):
        from ..engine import act_fmt, conv_bn_act
        y = ops.upsample2x_concat(x1, x2, act_fmt())
        y = conv_bn_act(y, self._first_conv_padded(), self.conv[1], relu=True)
        return conv_bn_act(y, self.conv[3], self.conv[4], relu=True)


class CamEncode(nn.Module):
    """EfficientNet-B0 trunk + two `Up` stages + depth / image heads (opencood/models/sub_modules/lss_submodule.py:39-138), same
    attribute names -> same state-dict keys; `trunk` holds efficientnet_pytorch's key names (sub_modules/efficientnet_b0.py).
    `heads_nhwc` is the GPU path:
      trunk                     stem, depthwise and pointwise kernels of csrc/mbconv.cu (fp32 channels-last; BN folded; the SE
                                multiply applied inside the project conv)
      up1, up2                  heal_upsample2x_concat, then both 3x3 convs + BN + ReLU on the conv engine (wgmma)
      depth_head | image_head   one fused 1x1 convolution 512 -> D + C, fp32 channels-last output
    `heads` keeps the plain torch path (CPU-capable; the tests' oracle-side restatement)."""

    def __init__(self, D, C, downsample, ddiscr, mode, use_gt_depth=False, depth_supervision=True):
        super().__init__()
        from .sub_modules.efficientnet_b0 import EfficientNetB0
        self.D, self.C, self.downsample = D, C, downsample
        self.d_min, self.d_max, self.num_bins = ddiscr[0], ddiscr[1], ddiscr[2]
        self.mode, self.use_gt_depth, self.depth_supervision = mode, use_gt_depth, depth_supervision
        if downsample not in (8, 16):
            raise NotImplementedError(f"img_downsample {downsample}: the EfficientNet encoder produces /8 or /16 feature maps")
        self.trunk = EfficientNetB0()
        self.up1 = Up(320 + 112, 512)
        if downsample == 8:
            self.up2 = Up(512 + 40, 512)
        if use_gt_depth:
            raise NotImplementedError("use_depth_gt is a training-time option outside the inference hot path")
        self.depth_head = nn.Conv2d(512, self.D, kernel_size=1, padding=0)
        self.image_head = nn.Conv2d(512, self.C, kernel_size=1, padding=0)

    def _check_sides(self, H, W):
        """`Up` concatenates the x2-upsampled coarser map with the finer one (lss_submodule.py:108-110); each stride-2 stage maps a
        side s to s // 2, so the two only agree when no halving that `Up` undoes dropped a row or column."""
        for name, s in (("height", H), ("width", W)):
            r = [s]
            for _ in range(5):
                r.append(r[-1] // 2)
            pairs = [(r[5], r[4])] + ([(r[4], r[3])] if self.downsample == 8 else [])
            for coarse, fine in pairs:
                if coarse < 1 or 2 * coarse != fine:
                    raise ValueError(f"image {name} {s}: the EfficientNet feature maps have {name}s {r[3]} (/8), {r[4]} (/16), {r[5]} (/32), "
                                     f"and {coarse} upsampled x2 does not match {fine}; use image sides that are multiples of 32")

    def heads(self, x):
        """x (BN, 3|4, H, W) -> (depth_logits (BN,D,fH,fW), feat (BN,C,fH,fW))"""
        self._check_sides(x.shape[2], x.shape[3])
        ep = self.trunk.endpoints(x[:, :3])
        f = self.up1(ep['reduction_5'], ep['reduction_4'])
        if self.downsample == 8:
            f = self.up2(f, ep['reduction_3'])
        return self.depth_head(f), self.image_head(f)

    _fused_heads = CamEncode_Resnet101._fused_heads

    def heads_nhwc(self, x, plan=None):
        """x (BN, 3|4, H, W) fp32 CUDA -> Act f32 (BN, H/ds, W/ds, D + C): [depth logits | image features] per pixel.  With a `plan`
        (data_utils.camera_input.inference_plan), x is raw uint8 frames (BN, H0, W0, 3), resized, cropped and normalised to NCHW fp32
        by heal_camera_input first."""
        from ..engine import conv_bn_act
        if plan is not None:
            x = ops.camera_input(x, plan, "nchw")
        self._check_sides(x.shape[2], x.shape[3])
        r3, r4, r5 = self.trunk.endpoints_nhwc(x.float().contiguous())
        f = self.up1.forward_nhwc(r5, r4)
        if self.downsample == 8:
            f = self.up2.forward_nhwc(f, r3)
        return conv_bn_act(f, self._fused_heads(), None, relu=False, out_fmt="f32")


class LiftSplatShoot(nn.Module):
    """opencood/models/heter_encoders.py:83-241 with the reference's ctor argument and forward signature."""

    def __init__(self, args):
        super().__init__()
        self.grid_conf = args['grid_conf']
        self.data_aug_conf = args['data_aug_conf']
        dx, bx, nx = gen_dx_bx(self.grid_conf['xbound'], self.grid_conf['ybound'], self.grid_conf['zbound'])
        self.register_buffer("dx", dx.clone(), persistent=False)
        self.register_buffer("bx", bx.clone(), persistent=False)
        self.register_buffer("nx", nx.clone(), persistent=False)
        # host copies of the grid constants: the kernels take them as host arguments, and reading the (device) buffers back would
        # be a synchronising copy per frame that a CUDA graph capture rejects
        self._lower_host = (bx - dx / 2.).tolist()
        self._dx_host = dx.tolist()
        self._nx_host = [int(v) for v in nx.tolist()]
        self.depth_supervision = args['depth_supervision']
        self.downsample = args['img_downsample']
        self.camC = args['img_features']
        self.register_buffer("frustum", self.create_frustum(), persistent=False)
        self.D = self.frustum.shape[0]
        self.camera_encoder_type = args['camera_encoder']
        encoders = {'EfficientNet': CamEncode, 'Resnet101': CamEncode_Resnet101}
        if self.camera_encoder_type not in encoders:
            raise NotImplementedError(f"camera_encoder '{self.camera_encoder_type}': the reference builds 'EfficientNet' or 'Resnet101' "
                                      "(opencood/models/heter_encoders.py:103-108)")
        self.camencode = encoders[self.camera_encoder_type](self.D, self.camC, self.downsample, self.grid_conf['ddiscr'],
                                                            self.grid_conf['mode'], args['use_depth_gt'], args['depth_supervision'])
        if self._nx_host[2] != 1:
            raise NotImplementedError("heal_lss_pool supports a single z slice (every HEAL yaml uses zbound with nz == 1)")

    def create_frustum(self):
        ogfH, ogfW = self.data_aug_conf['final_dim']
        fH, fW = ogfH // self.downsample, ogfW // self.downsample
        ds = torch.tensor(depth_discretization(*self.grid_conf['ddiscr'], self.grid_conf['mode']), dtype=torch.float) \
            .view(-1, 1, 1).expand(-1, fH, fW)
        D = ds.shape[0]
        xs = torch.linspace(0, ogfW - 1, fW, dtype=torch.float).view(1, 1, fW).expand(D, fH, fW)
        ys = torch.linspace(0, ogfH - 1, fH, dtype=torch.float).view(1, fH, 1).expand(D, fH, fW)
        return torch.stack((xs, ys, ds), -1).contiguous()

    def bev_from_heads(self, depth_logits, feat, rots, trans, intrins, post_rots, post_trans):
        """The kernel part: geometry -> cell index -> fused softmax (x) feat -> BEV pool.  Returns Act f32 (B,ny,nx,C)."""
        B, N = trans.shape[:2]
        post_inv, combine = ops.lss_camera_matrices(rots, intrins, post_rots)      # the reference's 3x3 algebra (:135,:142), capturable
        cell = ops.lss_cell_index(self.frustum, post_inv, post_trans.reshape(B * N, 3), combine, trans.reshape(B * N, 3),
                                  self._lower_host, self._dx_host, self._nx_host)
        return ops.lss_pool(depth_logits, feat, cell, N, self._nx_host[0], self._nx_host[1])

    def cell_index(self, rots, trans, intrins, post_rots, post_trans):
        B, N = trans.shape[:2]
        post_inv, combine = ops.lss_camera_matrices(rots, intrins, post_rots)      # the reference's 3x3 algebra (:135,:142), capturable
        return ops.lss_cell_index(self.frustum, post_inv, post_trans.reshape(B * N, 3), combine, trans.reshape(B * N, 3),
                                  self._lower_host, self._dx_host, self._nx_host)

    def camera_plan(self, H0, W0):
        """The reference's inference resize / crop of a raw (H0, W0) frame for this encoder's data_aug_conf (cached per size).  The
        batch's post_rots / post_trans are still what the geometry uses."""
        from ..data_utils.camera_input import inference_plan
        plans = self.__dict__.setdefault("_camera_plans", {})
        if (H0, W0) not in plans:
            plans[(H0, W0)] = inference_plan(self.data_aug_conf, H0, W0)
        return plans[(H0, W0)]

    def forward_act(self, data_dict, modality_name, fmt=None):
        """image trunk + heads on the conv engine -> frustum cell index -> deterministic sorted BEV pooling
        (heal_lss_pool_sorted reads logits and features straight from the fused heads' channels-last output)."""
        from ..engine import act_fmt
        require_eval(self)
        d = data_dict[f'inputs_{modality_name}']
        x = d['imgs']
        plan = None
        if x.dtype == torch.uint8:                                        # raw sensor frames (B, N, H0, W0, 3), resampled on the GPU
            B, N, H0, W0, _ = x.shape
            plan = self.camera_plan(H0, W0)
            x = x.reshape(B * N, H0, W0, 3)
        else:                                                             # images the reference's DataLoader already normalised
            B, N, C, imH, imW = x.shape
            x = x.view(B * N, C, imH, imW)
        if _os.environ.get("HEAL_CAM_TRUNK_TORCH", "0") == "1":           # A/B hook: torch / cuDNN trunk + atomic pooling (round 1)
            depth_logits, feat = self.camencode.heads(x if plan is None else ops.camera_input(x, plan, "nchw"))
            if self.depth_supervision:
                self.depth_items = (depth_logits, None)
            return self.bev_from_heads(depth_logits, feat, d['rots'], d['trans'], d['intrins'], d['post_rots'], d['post_trans'])
        y = self.camencode.heads_nhwc(x, plan)                            # Act f32 (BN, fH, fW, D + camC)
        D, camC, fH, fW = self.D, self.camC, y.H, y.W
        S, HW = D + camC, y.H * y.W
        if self.depth_supervision:
            self.depth_items = (y.t[..., :D].permute(0, 3, 1, 2), None)
        cell = self.cell_index(d['rots'], d['trans'], d['intrins'], d['post_rots'], d['post_trans'])
        return ops.lss_pool_sorted(y.t, (HW * S, 1, S), y.t[..., D:], (HW * S, 1, S), cell, N, D, camC, fH, fW,
                                   self._nx_host[0], self._nx_host[1], out_fmt=fmt or act_fmt())

    def forward(self, data_dict, modality_name):
        return ops.act_to_nchw(self.forward_act(data_dict, modality_name))


class LiftSplatShootVoxel(LiftSplatShoot):
    """heter_encoders.py:244-301: max over z instead of concat; identical for the single-slice grids HEAL uses."""


# ---------------------------------------------------------------------------------------------------------
# SECOND
# ---------------------------------------------------------------------------------------------------------
class SECOND(nn.Module):
    """heter_encoders.py:52-81: MeanVFE -> VoxelBackBone8x (sparse 3-D convs) -> HeightCompression."""

    def __init__(self, args):
        super().__init__()
        from .sub_modules.mean_vfe import MeanVFE
        from .sub_modules.sparse_backbone_3d import VoxelBackBone8x
        from .sub_modules.height_compression import HeightCompression
        lidar_range = np.array(args['lidar_range'])
        grid_size = np.round((lidar_range[3:6] - lidar_range[:3]) / np.array(args['voxel_size'])).astype(np.int64)
        self.vfe = MeanVFE(args['mean_vfe'], args['mean_vfe']['num_point_features'])
        self.spconv_block = VoxelBackBone8x(args['spconv'], input_channels=args['spconv']['num_features_in'], grid_size=grid_size)
        self.map_to_bev = HeightCompression(args['map2bev'])
        self.voxel_size = [float(v) for v in args['voxel_size']]
        self.lidar_range = [float(v) for v in args['lidar_range']]
        self.voxelize_args = args.get('voxelize', {'max_points_per_voxel': 5, 'max_voxels': 70000})

    def forward_act(self, data_dict, modality_name, fmt=None):
        require_eval(self)
        inp = data_dict[f'inputs_{modality_name}']
        rows_dev = None
        if 'voxel_features' in inp:
            vf, vc, vn = inp['voxel_features'], inp['voxel_coords'], inp['voxel_num_points']
            batch_size = inp.get('batch_size')
            if batch_size is None:
                batch_size = int(vc[:, 0].max().item()) + 1          # host sync, as the reference (heter_encoders.py:70)
        else:
            pts, offs = ops.raw_points_of(inp, self.lidar_range)
            vf, vc, vn, nvox = ops.voxelize(pts, offs, self.lidar_range, self.voxel_size,
                                            int(inp.get('max_points_per_voxel', self.voxelize_args['max_points_per_voxel'])),
                                            int(inp.get('max_voxels', self.voxelize_args['max_voxels'])))
            rows_dev = nvox[0:1]
            batch_size = inp['agent_offsets'].numel() - 1
        feats = ops.mean_vfe(vf.contiguous(), vn)
        out, _ = self.spconv_block.forward_sparse(feats, vc, batch_size, rows_dev)
        return self.map_to_bev.forward_act(out)

    def forward(self, data_dict, modality_name):
        return ops.act_to_nchw(self.forward_act(data_dict, modality_name))
