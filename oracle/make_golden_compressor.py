"""Golden vectors for feature compression (`compressor:`, TEST INFRASTRUCTURE ONLY): the UNMODIFIED reference NaiveCompressor
(opencood/models/sub_modules/naive_compress.py:5-31), HeterPyramidCollab and HeterModelBaseline with a `compressor:` entry, run on
the CPU with procedural weights.

    python -m oracle.make_golden_compressor        (needs the reference package: oracle/_ref or HEAL_REFERENCE_ROOT)

Writes
  tests/golden/compressor_c64.pt.xz, compressor_c256.pt.xz       NaiveCompressor(C, ratio) for ratio in RATIOS on the seeded
                                                                  module_x(C) (not stored): every 4th (C = 64) or 16th (C = 256)
                                                                  output channel
  tests/golden/heter_pyramid_collab_compress_small.pt.xz          make_golden.small_model_args() + compressor (64, ratio 8) on
                                                                  make_golden.small_scene()
  tests/golden/heter_pyramid_collab_hetero_compress_small.pt.xz   efficientnet.collab_args() + compressor (64, ratio 8), agents
                                                                  [m1 PointPillar, m2 LSS-EfficientNet, m1] (efficientnet.collab_data)
  tests/golden/heter_model_baseline_compress_small.pt.xz          make_golden.baseline_att_args() + compressor (256, ratio 32) +
                                                                  supervise_single on make_golden.small_scene()"""
import copy
import os

import torch

from oracle import efficientnet

efficientnet.install()          # before ref_shim.install(): the stand-in takes the place of the MagicMock stub

from oracle import golden, make_golden, procedural, ref_shim  # noqa: E402
from oracle.make_golden_coalign import _cuda_moves_stay_on_cpu  # noqa: E402

OUT = make_golden.OUT
RATIOS = (1, 2, 4, 8, 16, 32)
SAMPLE = {64: 4, 256: 16}       # output channel sampling step per input width (each file stays under 1 MB)
HEADS = ("cls_preds", "reg_preds", "dir_preds")


def module_x(C, seed=11):
    """Seeded (2, C, 37, 53) input: odd sides, so the 8 x 16 output tiles of the narrow conv end inside the map.  Non-negative,
    as the features after the aligner / shrinker ReLUs are."""
    g = torch.Generator().manual_seed(seed + C)
    return torch.relu(torch.randn(2, C, 37, 53, generator=g))


def collab_compress_args():
    args = make_golden.small_model_args()
    args["compressor"] = {"input_dim": 64, "compress_ratio": 8}
    return args


def hetero_compress_args():
    args = efficientnet.collab_args()
    args["compressor"] = {"input_dim": 64, "compress_ratio": 8}
    return args


def baseline_compress_args():
    args = make_golden.baseline_att_args()
    args["compressor"] = {"input_dim": 256, "compress_ratio": 32}
    args["supervise_single"] = True
    args["in_head_single"] = 256
    return args


def module_goldens():
    from opencood.models.sub_modules.naive_compress import NaiveCompressor
    for C in (64, 256):
        x = module_x(C)
        outs = {}
        for r in RATIOS:
            m = NaiveCompressor(C, r).eval()
            shapes = procedural.shapes_of(m)
            m.load_state_dict(procedural.make_state_dict(shapes), strict=True)
            with torch.no_grad():
                y = m(x)
            outs[r] = {"shapes": shapes, "out_s": y[:, ::SAMPLE[C]].contiguous()}
            print(f"NaiveCompressor({C}, {r}):", tuple(y.shape), float(y.abs().max()), float((y > 0).float().mean()))
        golden.save({"C": C, "step": SAMPLE[C], "ratios": outs}, os.path.join(OUT, f"compressor_c{C}.pt"))


def model_golden(cls, args, data, name, keys, state_dict_of=procedural.make_state_dict):
    with _cuda_moves_stay_on_cpu():
        m = cls(copy.deepcopy(args)).eval()
    shapes = procedural.shapes_of(m)
    m.load_state_dict(state_dict_of(shapes), strict=True)
    with torch.no_grad():
        out = m(copy.deepcopy(data))
    golden.save({"args": args, "shapes": shapes, "out": {k: out[k] for k in keys}}, os.path.join(OUT, name + ".pt"))
    print(name, {k: (tuple(out[k].shape), float(out[k].abs().max())) for k in keys})


def main():
    ref_shim.install()
    torch.set_num_threads(8)
    from opencood.models.heter_model_baseline import HeterModelBaseline
    from opencood.models.heter_pyramid_collab import HeterPyramidCollab
    module_goldens()
    data = make_golden.small_scene()
    model_golden(HeterPyramidCollab, collab_compress_args(), data, "heter_pyramid_collab_compress_small", HEADS)
    model_golden(HeterPyramidCollab, hetero_compress_args(), efficientnet.collab_data(),
                 "heter_pyramid_collab_hetero_compress_small", HEADS, state_dict_of=efficientnet.state_dict_of)
    model_golden(HeterModelBaseline, baseline_compress_args(), data, "heter_model_baseline_compress_small",
                 HEADS + ("cls_preds_single", "reg_preds_single", "dir_preds_single"))
    for f in ("compressor_c64", "compressor_c256", "heter_pyramid_collab_compress_small",
              "heter_pyramid_collab_hetero_compress_small", "heter_model_baseline_compress_small"):
        print(f, os.path.getsize(os.path.join(OUT, f + ".pt.xz")) // 1024, "KiB")


if __name__ == "__main__":
    main()
