"""Feature compression (`compressor:`): which path the first decoder conv (Conv3x3(c -> C) + BN + ReLU on the compressed map,
c = C // ratio < 64) should take, and what the compressor costs in a frame.

1. The first decoder conv, three ways, alternating in one run (CUDA events after warm-up, tc32 and bf16):
     narrow:  heal_conv3x3_narrow_tc (K = 9 * c, rounded up to 16)
     padded:  heal_conv2d_tc on the map zero-padded to 64 channels (K = 9 * 64), timed with the zero fill of the padded map
              (NaiveCompressor allocates it zeroed each frame and the encoder writes its c channels)
     simt:    heal_conv2d_simt (fp32 CUDA cores; tc32 only)
   at the HEAL shape (5 x 64 x 256^2, ratios 2..32) and the baseline shapes (5 x 256 x 256^2 and 128^2, ratios 8..32), with the
   narrow and padded outputs compared.
2. The whole NaiveCompressor.forward_nhwc per ratio at the same shapes.
3. The C2 HeterPyramidCollab frame (graph replay) without and with a compressor (input_dim 64).
Prints the card's name and power limit first; --out DIR writes the records as DIR/compressor.json."""
import argparse
import copy
import json
import os
import sys

import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))

from bottleneck_experiment import card, time_us  # noqa: E402
from fusion_methods_experiment import frame_inputs, load_procedural  # noqa: E402

SHAPES = [("heal 5x64x256^2", 5, 64, 256, (2, 4, 8, 16, 32)),
          ("baseline 5x256x256^2", 5, 256, 256, (8, 16, 32)),
          ("baseline 5x256x128^2", 5, 256, 128, (8, 16, 32))]


def conv_bn(cin, cout, seed):
    torch.manual_seed(seed)
    conv, bn = nn.Conv2d(cin, cout, 3, padding=1), nn.BatchNorm2d(cout, eps=1e-3)
    with torch.no_grad():
        bn.running_var.uniform_(0.5, 1.5)
        bn.running_mean.normal_(0, 0.1)
    return conv.eval(), bn.eval()


def padded_conv(conv, cin_to):
    p = nn.Conv2d(cin_to, conv.out_channels, 3, padding=1)
    with torch.no_grad():
        p.weight.zero_()
        p.weight[:, :conv.in_channels] = conv.weight
        p.bias.copy_(conv.bias)
    return p.eval()


def first_decoder_conv(iters, rounds):
    from heal_b200 import engine, ops
    recs = []
    for name, N, C, HW, ratios in SHAPES:
        for r in ratios:
            c = C // r
            conv, bn = conv_bn(c, C, r)
            pconv = padded_conv(conv, 64).cuda()
            conv, bn = conv.cuda(), bn.cuda()
            x32 = torch.relu(torch.randn(N, HW, HW, c, device="cuda"))
            xp32 = torch.zeros(N, HW, HW, 64, device="cuda")
            xp32[..., :c] = x32
            pn = ops.pack_conv3x3_narrow(conv, bn, True).to("cuda")
            pt = engine.packed(pconv, bn, True, kind="tc2")
            ps = engine.packed(conv, bn, True, kind="simt" if c % 4 == 0 else "simt_cin4")
            xs32 = x32 if c % 4 == 0 else xp32[..., :(c + 3) // 4 * 4].contiguous()
            flops = 2.0 * N * HW * HW * C * c * 9
            for fmt, planes in (("split", 2), ("bf16", 1)):
                x = ops.convert(ops.Act(x32, "f32"), fmt)
                xp = ops.convert(ops.Act(xp32, "f32"), fmt)
                xp_data = xp.t.clone()
                variants = {"narrow": lambda: ops.conv3x3_narrow_tc(x, pn, planes, out_fmt=fmt),
                            "padded": lambda: (xp.t.zero_(), ops.conv2d_tc(xp, pt)[0])[1]}
                if fmt == "split":
                    variants["simt"] = lambda: ops.conv2d_simt(ops.Act(xs32, "f32"), ps, out_fmt="split")
                outs = {k: ops.act_to_nchw(f()) for k, f in variants.items() if k != "padded"}
                outs["padded"] = ops.act_to_nchw(ops.conv2d_tc(ops.Act(xp_data, fmt), pt)[0])
                diff = (outs["narrow"] - outs["padded"]).abs().max().item() / max(outs["padded"].abs().max().item(), 1.0)
                times = {k: [] for k in variants}
                for f in variants.values():
                    time_us(f, 3)
                for _ in range(rounds):
                    for k, f in variants.items():
                        times[k].append(time_us(f, iters))
                rec = {"shape": name, "ratio": r, "c": c, "fmt": fmt, "narrow_vs_padded_rel": diff,
                       "us": {k: sorted(v) for k, v in times.items()},
                       "tflops_narrow": flops / min(times["narrow"]) / 1e6}
                recs.append(rec)
                print(json.dumps(rec), flush=True)
    return recs


def whole_compressor(iters):
    from heal_b200 import engine, ops
    from heal_b200.models.sub_modules.naive_compress import NaiveCompressor
    from workloads import procedural
    recs = []
    for prec in ("tc32", "bf16"):
        engine.set_precision(prec)
        for name, N, C, HW, ratios in SHAPES:
            x = ops.convert(ops.Act(torch.relu(torch.randn(N, HW, HW, C, device="cuda")), "f32"), engine.act_fmt())
            for r in ratios:
                m = NaiveCompressor(C, r).eval()
                m.load_state_dict(procedural.make_state_dict(procedural.shapes_of(m)), strict=True)
                m = m.cuda()
                with torch.no_grad():
                    f = lambda: m.forward_nhwc(x)
                    time_us(f, 3)
                    us = sorted(time_us(f, iters) for _ in range(3))
                rec = {"compressor": name, "ratio": r, "precision": prec, "us": us}
                recs.append(rec)
                print(json.dumps(rec), flush=True)
    engine.set_precision("tc32")
    return recs


def frames(iters):
    from heal_b200 import engine
    from heal_b200.graph import FrameGraph
    from heal_b200.models.heter_pyramid_collab import HeterPyramidCollab
    from workloads import configs as wcfg
    pts, offs, pw = frame_inputs(5)
    cap = (pts.shape[0] + 4095) // 4096 * 4096
    recs = []
    for prec in ("tc32", "bf16"):
        engine.set_precision(prec)
        graphs = {}
        for ratio in (None, 2, 8, 32):
            args = copy.deepcopy(wcfg.c2_args())
            if ratio:
                args["compressor"] = {"input_dim": 64, "compress_ratio": ratio}
            m = load_procedural(HeterPyramidCollab(args).eval()).cuda()
            fg = FrameGraph(m, 5, cap, pw.shape)
            fg.load(pts, offs, pw)
            graphs[ratio] = (m, fg)
        times = {k: [] for k in graphs}
        for _ in range(3):
            for k, (_, fg) in graphs.items():
                times[k].append(time_us(fg.replay, iters))
        for k, v in times.items():
            rec = {"frame": "C2 HeterPyramidCollab, 5 agents", "precision": prec, "compress_ratio": k, "us": sorted(v)}
            recs.append(rec)
            print(json.dumps(rec), flush=True)
        del graphs
        torch.cuda.empty_cache()
    engine.set_precision("tc32")
    return recs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    opt = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    c = card()
    print("card:", c, flush=True)
    res = {"card": c, "first_decoder_conv": first_decoder_conv(opt.iters, opt.rounds),
           "compressor": whole_compressor(opt.iters), "frames": frames(max(opt.iters // 2, 10))}
    if opt.out:
        os.makedirs(opt.out, exist_ok=True)
        with open(os.path.join(opt.out, "compressor.json"), "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
