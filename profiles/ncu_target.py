"""Stand-alone launcher of the four dominant conv shapes of the C2 frame, for `ncu --set full` captures
(keeps the report small; the launch list of the full frame comes from `bench.py --no-graph`).
  1. shrink conv 3x3 384->256 @256x256 (N=1)        k_conv2d_tc<128,3,1>
  2. per-agent ResNet conv 3x3 64->64 @256x256 (N=1) k_conv2d_tc<64,2,2> (halo)
  3. ResNeXt level-0 conv1 1x1 64->128 @256x256      k_conv2d_tc<128,2,2>
  4. ResNeXt level-0 grouped 3x3 (32 groups, 128 ch) k_gconv3x3_ring (k_conv2d_tc<64,3,2,false,true> with HEAL_TC_RING=0)
(template arguments: BLOCK_N, STAGES, staging buffers[, GELU, GROUPED])
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from heal_b200 import ops  # noqa: E402


def run(cin, cout, k, groups, N=1, H=256, W=256, reps=3):
    conv = torch.nn.Conv2d(cin, cout, k, padding=k // 2, groups=groups, bias=False)
    bn = torch.nn.BatchNorm2d(cout).eval()
    pc = ops.pack_conv_tc(conv, bn, True, planes=2).to("cuda")
    x = ops.convert(ops.to_act(torch.randn(N, cin, H, W, device="cuda")), "split")
    for _ in range(reps):
        ops.conv2d_tc(x, pc)
    torch.cuda.synchronize()


if __name__ == "__main__":
    run(384, 256, 3, 1)
    run(64, 64, 3, 1)
    run(64, 128, 1, 1)
    run(128, 128, 3, 32)
