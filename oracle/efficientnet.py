"""ORACLE — TEST INFRASTRUCTURE ONLY.  EfficientNet-B0 as the reference's CamEncode uses it
(opencood/models/sub_modules/lss_submodule.py:53 `EfficientNet.from_pretrained("efficientnet-b0")`, :87-107).

The `efficientnet_pytorch` package is not installed, so (a) this file restates its efficientnet-b0 in plain torch with the package's
state-dict key names, written for clarity (explicit F.pad, conv2d with padding 0), and (b) `install()` registers a stand-in module
named `efficientnet_pytorch` exposing `EfficientNet.from_pretrained(name)` (randomly initialised: no download).  With it the
UNMODIFIED reference CamEncode and LiftSplatShoot run on the CPU (oracle/make_golden_efficientnet.py), so endpoint selection, `Up`,
the heads and everything downstream are pinned to reference code; only the inside of the trunk is a restatement.  Its topology is
cross-checked against torchvision's efficientnet_b0 in tests/test_oracle_efficientnet.py; its padding and BN epsilon are restated
from the package's documentation of `Conv2dStaticSamePadding` (image_size 224) and are NOT pinned against the real package
(SURVEY.md 8c).  Nothing here imports heal_b200.

Architecture ("efficientnet-b0", width 1.0, depth 1.0): stem conv 3x3/2 3 -> 32, BN, swish; 16 MBConv blocks from 7 stages
(kernel, stride, expand ratio, in, out, repeats); every BN has eps 1e-3; SE squeeze width max(1, int(block input channels / 4)).
"""
import sys
import types

import torch
import torch.nn as nn
import torch.nn.functional as F

from workloads import procedural

STAGES = [  # k, s, e, i, o, r
    (3, 1, 1, 32, 16, 1),
    (3, 2, 6, 16, 24, 2),
    (5, 2, 6, 24, 40, 2),
    (3, 2, 6, 40, 80, 3),
    (5, 1, 6, 80, 112, 3),
    (5, 2, 6, 112, 192, 4),
    (3, 1, 6, 192, 320, 1),
]
NOMINAL_IMAGE = 224
EPS = 1e-3


def static_same_pad(size, k, s):
    """Conv2dStaticSamePadding for one axis of nominal length `size`: total = max((ceil(size/s) - 1) * s + k - size, 0), split
    (total // 2, total - total // 2).  Returns ((before, after), output length at the nominal size)."""
    out = -(-size // s)
    total = max((out - 1) * s + k - size, 0)
    return (total // 2, total - total // 2), out


class Swish(nn.Module):
    def forward(self, x):
        return x * torch.sigmoid(x)


class StaticPadConv(nn.Conv2d):
    """Conv2d whose zero padding (left, right, top, bottom) was fixed from the nominal image size at construction."""

    def __init__(self, cin, cout, k, stride, groups, bias, nominal):
        super().__init__(cin, cout, k, stride=stride, padding=0, groups=groups, bias=bias)
        (a, b), self.nominal_out = static_same_pad(nominal, k, stride)
        self.static_pad = (a, b, a, b)

    def forward(self, x):
        return F.conv2d(F.pad(x, self.static_pad), self.weight, self.bias, self.stride, 0, 1, self.groups)


class Block(nn.Module):
    def __init__(self, k, s, e, cin, cout, nominal):
        super().__init__()
        mid = cin * e
        self.has_expand = e != 1
        if self.has_expand:
            self._expand_conv = StaticPadConv(cin, mid, 1, 1, 1, False, nominal)
            self._bn0 = nn.BatchNorm2d(mid, eps=EPS)
        self._depthwise_conv = StaticPadConv(mid, mid, k, s, mid, False, nominal)
        self._bn1 = nn.BatchNorm2d(mid, eps=EPS)
        squeezed = max(1, int(cin * 0.25))
        self._se_reduce = StaticPadConv(mid, squeezed, 1, 1, 1, True, 1)
        self._se_expand = StaticPadConv(squeezed, mid, 1, 1, 1, True, 1)
        self._project_conv = StaticPadConv(mid, cout, 1, 1, 1, False, self._depthwise_conv.nominal_out)
        self._bn2 = nn.BatchNorm2d(cout, eps=EPS)
        self._swish = Swish()
        self.identity_skip = s == 1 and cin == cout
        self.nominal_out = self._depthwise_conv.nominal_out

    def forward(self, inputs, drop_connect_rate=None):
        x = inputs
        if self.has_expand:
            x = self._swish(self._bn0(self._expand_conv(x)))
        x = self._swish(self._bn1(self._depthwise_conv(x)))
        squeezed = F.adaptive_avg_pool2d(x, 1)
        squeezed = self._se_expand(self._swish(self._se_reduce(squeezed)))
        x = torch.sigmoid(squeezed) * x
        x = self._bn2(self._project_conv(x))
        if self.identity_skip:
            assert not self.training, "drop-connect is the identity in eval mode only"
            x = x + inputs
        return x


class EfficientNet(nn.Module):
    def __init__(self):
        super().__init__()
        size = NOMINAL_IMAGE
        self._conv_stem = StaticPadConv(3, 32, 3, 2, 1, False, size)
        size = self._conv_stem.nominal_out
        self._bn0 = nn.BatchNorm2d(32, eps=EPS)
        blocks = []
        for k, s, e, cin, cout, r in STAGES:
            for j in range(r):
                blocks.append(Block(k, s if j == 0 else 1, e, cin if j == 0 else cout, cout, size))
                size = blocks[-1].nominal_out
        self._blocks = nn.ModuleList(blocks)
        self._conv_head = StaticPadConv(320, 1280, 1, 1, 1, False, size)
        self._bn1 = nn.BatchNorm2d(1280, eps=EPS)
        self._fc = nn.Linear(1280, 1000)
        self._swish = Swish()
        self._global_params = types.SimpleNamespace(drop_connect_rate=0.2, batch_norm_epsilon=EPS, image_size=NOMINAL_IMAGE)

    @classmethod
    def from_pretrained(cls, model_name, **kwargs):
        if model_name != "efficientnet-b0":
            raise NotImplementedError(model_name)
        return cls()


def install():
    """Register the stand-in as `efficientnet_pytorch`.  Call BEFORE oracle.ref_shim.install() (which only stubs absent modules)
    and before anything imports opencood.models.sub_modules.lss_submodule."""
    mod = types.ModuleType("efficientnet_pytorch")
    mod.EfficientNet = EfficientNet
    sys.modules["efficientnet_pytorch"] = mod
    return mod


# ---------------------------------------------------------------------------------------------------------------------------
# shared by oracle/make_golden_efficientnet.py and the tests: weights, configs, seeded inputs
# ---------------------------------------------------------------------------------------------------------------------------
def state_dict_of(shapes, seed=1234):
    """SURVEY.md 8d weight recipe (procedural.make_state_dict: randomised BN statistics) with wide squeeze-and-excitation biases,
    so that the gates spread over (0, 1) instead of sitting near 0.5."""
    sd = procedural.make_state_dict(shapes, seed)
    for k in sd:
        if k.endswith("_se_expand.bias"):
            sd[k] = sd[k] * 20.0
        elif k.endswith("_se_reduce.bias"):
            sd[k] = sd[k] * 10.0
    return sd


TRUNK_D, TRUNK_C = 16, 32
TRUNK_DDISCR = [2, 30, 16]


def trunk_images():
    """(2, 4, 64, 96) seeded: two cameras, RGB + a depth plane the encoder must ignore."""
    return torch.randn(2, 4, 64, 96, generator=torch.Generator().manual_seed(61))


def lss_cfg():
    return {"grid_conf": {"xbound": [-12.8, 12.8, 0.4], "ybound": [-12.8, 12.8, 0.4], "zbound": [-10, 10, 20.0],
                          "ddiscr": [2, 30, 16], "mode": "LID"},
            "data_aug_conf": {"final_dim": [64, 128]}, "img_downsample": 8, "img_features": 32,
            "camera_encoder": "EfficientNet", "use_depth_gt": False, "depth_supervision": False}


def cam_inputs(seed=53):
    """One agent, two 64 x 128 cameras, seeded; goldens do not store them."""
    from workloads import synth
    rots, trans, intr, post_rots, post_trans = [torch.from_numpy(a) for a in synth.camera_rig(1, 2, 64, 128)]
    imgs = torch.randn(1, 2, 3, 64, 128, generator=torch.Generator().manual_seed(seed))
    return {"imgs": imgs, "rots": rots, "trans": trans, "intrins": intr, "post_rots": post_rots, "post_trans": post_trans}


def collab_args():
    """make_golden.small_model_args() (m1 PointPillar) plus the m2 block of opv2v/MoreModality/HEAL/stage1/m2_pyramid.yaml
    (Lift-Splat-Shoot, EfficientNet) scaled down: camera grid +-19.2 m against the +-12.8 m lidar range, so the camera map
    (96 x 96 cells, 48 x 48 after the stride-2 backbone) is center-cropped to the lidar map's 32 x 32."""
    from oracle import make_golden
    a = make_golden.small_model_args()
    enc = lss_cfg()
    enc["grid_conf"]["xbound"] = [-19.2, 19.2, 0.4]
    enc["grid_conf"]["ybound"] = [-19.2, 19.2, 0.4]
    enc["img_features"] = 64
    a["m2"] = {"core_method": "lift_splat_shoot", "sensor_type": "camera", "encoder_args": enc,
               "camera_mask_args": {"grid_conf": enc["grid_conf"]},
               "backbone_args": {"layer_nums": [3], "layer_strides": [2], "num_filters": [64], "inplanes": 64},
               "aligner_args": {"core_method": "identity"}}
    return a


COLLAB_AML = ["m1", "m2", "m1"]


def collab_data():
    """Agents [m1, m2, m1]: lidar agents and poses as make_golden_coalign.hetero_data(), the camera agent from cam_inputs()."""
    from oracle import make_golden
    lidar = make_golden.small_scene(seed=11, n_agents=2)
    return {"inputs_m1": lidar["inputs_m1"], "inputs_m2": cam_inputs(), "agent_modality_list": list(COLLAB_AML),
            "record_len": torch.tensor([3], dtype=torch.long),
            "pairwise_t_matrix": make_golden.small_scene(seed=11, n_agents=3)["pairwise_t_matrix"]}
