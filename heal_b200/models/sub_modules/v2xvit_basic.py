"""Parameter containers of opencood/models/sub_modules/v2xvit_basic.py (V2XFusionBlock, V2XTEncoder, V2XTransformer) with
the reference's submodule names, so that the state-dict keys match.  STTF has no parameters; RTE is only built with
use_RTE, which V2XViTFusion refuses.  V2XViTFusion (fuse_modules/fusion_in_one.py) runs the encoder."""
import torch
import torch.nn as nn
import torch.nn.functional as F

from .base_transformer import FeedForward, PreNorm
from .hmsa import HGTCavAttention
from .mswin import PyramidWindowAttention


class STTF(nn.Module):
    def __init__(self, args):
        super().__init__()
        self.discrete_ratio = args['voxel_size'][0]
        self.downsample_rate = args['downsample_rate']

    def theta(self, H, W):
        """(2, 3) fp32: the matrix STTF.forward hands F.affine_grid for a non-ego agent with the identity spatial correction
        V2XViTFusion passes, by the reference's own fp32 chain (get_discretized_transformation_matrix ->
        get_transformation_matrix -> warp_affine's homography, normalize_homography and inverse).  Its rounding makes it only
        nearly the identity, so the warp is applied, not skipped."""
        m = torch.eye(4).reshape(1, 1, 4, 4)
        m = m[:, :, [0, 1], :][:, :, :, [0, 1, 3]]
        m[:, :, :, -1] = m[:, :, :, -1] / (self.discrete_ratio * self.downsample_rate)
        M = m.reshape(-1, 2, 3).float()
        center = torch.Tensor([W / 2, H / 2]).unsqueeze(0)
        shift_m = torch.eye(3)[None].repeat(1, 1, 1)
        shift_m[:, :2, 2] = center
        shift_m_inv = torch.eye(3)[None].repeat(1, 1, 1)
        shift_m_inv[:, :2, 2] = -center
        rotat_m = torch.eye(3)[None].repeat(1, 1, 1)
        rotat_m[:, :2, :2] = M[:, :2, :2]
        T = (shift_m @ rotat_m @ shift_m_inv)[:, :2, :]
        T[..., 2] += M[..., 2]
        H3 = F.pad(T, [0, 0, 0, 1], "constant", value=0.0)
        H3[..., -1, -1] += 1.0

        def norm_pix(h, w):
            tr = torch.tensor([[1.0, 0.0, -1.0], [0.0, 1.0, -1.0], [0.0, 0.0, 1.0]])
            tr[0, 0] = tr[0, 0] * 2.0 / (1e-14 if w == 1 else w - 1.0)
            tr[1, 1] = tr[1, 1] * 2.0 / (1e-14 if h == 1 else h - 1.0)
            return tr.unsqueeze(0)

        src_pix_trans_src_norm = torch.inverse(norm_pix(H, W))
        dst_norm_trans_src_norm = norm_pix(H, W) @ (H3 @ src_pix_trans_src_norm)
        return torch.inverse(dst_norm_trans_src_norm)[0, :2, :].contiguous()


class V2XFusionBlock(nn.Module):
    def __init__(self, num_blocks, cav_att_config, pwindow_config):
        super().__init__()
        self.layers = nn.ModuleList([])
        self.num_blocks = num_blocks
        for _ in range(num_blocks):
            att = HGTCavAttention(cav_att_config['dim'], heads=cav_att_config['heads'], dim_head=cav_att_config['dim_head'],
                                  dropout=cav_att_config['dropout'])
            self.layers.append(nn.ModuleList([
                PreNorm(cav_att_config['dim'], att),
                PreNorm(cav_att_config['dim'],
                        PyramidWindowAttention(pwindow_config['dim'], heads=pwindow_config['heads'],
                                               dim_heads=pwindow_config['dim_head'], drop_out=pwindow_config['dropout'],
                                               window_size=pwindow_config['window_size'],
                                               relative_pos_embedding=pwindow_config['relative_pos_embedding'],
                                               fuse_method=pwindow_config['fusion_method']))]))


class V2XTEncoder(nn.Module):
    def __init__(self, args):
        super().__init__()
        cav_att_config = args['cav_att_config']
        pwindow_att_config = args['pwindow_att_config']
        feed_config = args['feed_forward']
        num_blocks = args['num_blocks']
        depth = args['depth']
        mlp_dim = feed_config['mlp_dim']
        dropout = feed_config['dropout']
        self.downsample_rate = args['sttf']['downsample_rate']
        self.discrete_ratio = args['sttf']['voxel_size'][0]
        self.use_roi_mask = args['use_roi_mask']
        self.use_RTE = cav_att_config['use_RTE']
        self.RTE_ratio = cav_att_config['RTE_ratio']
        self.sttf = STTF(args['sttf'])
        # the prior encoding (velocity, time delay, infra) would enter through prior_feed; V2XViTFusion feeds zeros and the
        # reference never applies it, so it is kept for the state dict only
        self.prior_feed = nn.Linear(cav_att_config['dim'] + 3, cav_att_config['dim'])
        self.layers = nn.ModuleList([])
        for _ in range(depth):
            self.layers.append(nn.ModuleList([
                V2XFusionBlock(num_blocks, cav_att_config, pwindow_att_config),
                PreNorm(cav_att_config['dim'], FeedForward(cav_att_config['dim'], mlp_dim, dropout=dropout))
            ]))


class V2XTransformer(nn.Module):
    def __init__(self, args):
        super().__init__()
        self.encoder = V2XTEncoder(args['encoder'])
