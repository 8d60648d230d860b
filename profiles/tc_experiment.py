"""Timing experiment for the wgmma conv: where does a tile's time go?  HEAL_TC_DBG bits (results invalid, timing only):
1 = skip the epilogue's global stores, 2 = skip the weight (B) TMA loads, 4 = skip the activation (A) TMA loads,
8 = skip the residual loads, 16 = skip the MMAs."""
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SHAPES = [("shrink3x3_384_256_n1", 384, 256, 3, 1, 1), ("shrink3x3_256_256_n1", 256, 256, 3, 1, 1),
          ("res3x3_64_64_n5", 64, 64, 3, 1, 5), ("res3x3_64_64_n5_res", 64, 64, 3, 1, 5), ("l0_1x1_64_128_n5", 64, 128, 1, 1, 5),
          ("l0_1x1_128_64_n5_res", 128, 64, 1, 1, 5), ("l0_grouped_128_n5", 128, 128, 3, 32, 5), ("l1_1x1_256_128_n5_128px_res", 256, 128, 1, 1, 5),
          ("l1_grouped_256_n5_128px", 256, 256, 3, 32, 5),
          ("l2_1x1_256_512_n5_64px", 256, 512, 1, 1, 5), ("l2_1x1_512_256_n5_64px_res", 512, 256, 1, 1, 5), ("l2_grouped_512_n5_64px", 512, 512, 3, 32, 5)]


def main():
    from heal_b200 import ops
    only = os.environ.get("TC_EXP_ONLY")
    for name, cin, cout, k, groups, N in SHAPES:
        if only and only not in name:
            continue
        H = W = 64 if "64px" in name else (128 if "128px" in name else 256)
        conv = torch.nn.Conv2d(cin, cout, k, padding=k // 2, groups=groups, bias=False)
        pc = ops.pack_conv_tc(conv, torch.nn.BatchNorm2d(cout).eval(), True, planes=2).to("cuda")
        x = ops.convert(ops.to_act(torch.randn(N, cin, H, W, device="cuda")), "split")
        out = ops.act_empty(N, H, W, cout, "split", "cuda")
        res = ops.convert(ops.to_act(torch.randn(N, cout, H, W, device="cuda")), "split") if name.endswith("_res") else None
        for _ in range(3):
            ops.conv2d_tc(x, pc, out=out, residual=res)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(20):
            ops.conv2d_tc(x, pc, out=out, residual=res)
        b.record()
        torch.cuda.synchronize()
        us = a.elapsed_time(b) / 20 * 1e3
        fl = 2.0 * N * H * W * cout * (cin // groups) * k * k
        print(f"dbg={os.environ.get('HEAL_TC_DBG', '0')} {name}: {us:8.1f} us  {fl / us / 1e6:7.1f} TF/s")


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "all":
        for d in ("0", "1", "8", "16", "6", "22", "31"):
            subprocess.run([sys.executable, __file__], env={**os.environ, "HEAL_TC_DBG": d})
    else:
        main()
