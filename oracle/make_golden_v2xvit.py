"""Golden vectors for V2X-ViT (TEST INFRASTRUCTURE ONLY): the UNMODIFIED reference V2XViTFusion (fusion_in_one.py:320-372) and
HeterModelBaseline with fusion_method v2xvit, run on CPU with procedural weights.

    python -m oracle.make_golden_v2xvit        (needs the reference package: oracle/_ref or HEAL_REFERENCE_ROOT)

Writes tests/golden/fusion_v2xvit.pt.xz (module level: the cases of v2xvit.module_cases(), seeded inputs not stored, outputs
stored as channel samples to keep the file small) and heter_model_baseline_v2xvit_small.pt.xz (the lidar_v2xvit.yaml block on
make_golden.small_scene(), a 32 x 32 fused map)."""
import copy
import os

import torch

from oracle import golden, make_golden, procedural, ref_shim, v2xvit

OUT = make_golden.OUT
STRIDE = 8      # channel sampling of the stored module outputs


def load_procedural(module):
    shapes = procedural.shapes_of(module)
    module.load_state_dict(procedural.make_state_dict(shapes), strict=True)
    return shapes


def baseline_v2xvit_args():
    """make_golden.baseline_att_args with the `v2xvit:` block of opv2v/LiDAROnly/lidar_v2xvit.yaml (max_cav 5)."""
    args = make_golden.baseline_att_args()
    args["fusion_method"] = "v2xvit"
    del args["att"]
    args["v2xvit"] = v2xvit.v2xvit_args()
    return args


def main():
    ref_shim.install()
    torch.set_num_threads(8)
    from opencood.models.fuse_modules.fusion_in_one import V2XViTFusion
    from opencood.models.heter_model_baseline import HeterModelBaseline
    cases = {}
    for name, (args, _, _, _, L) in v2xvit.module_cases().items():
        x, rl, pw = v2xvit.case_inputs(name)
        aff = v2xvit.case_affine(pw)
        m = V2XViTFusion(copy.deepcopy(args)).eval()
        shapes = load_procedural(m)
        with torch.no_grad():
            y = m(x, rl, aff)
        cases[name] = {"args": args, "shapes": shapes, "record_len": rl, "pairwise_t_matrix": pw, "affine": aff,
                       "stride": STRIDE, "out_s": y[:, ::STRIDE].contiguous()}
        print(f"v2xvit {name}:", tuple(y.shape), float(y.abs().max()))
    golden.save(cases, os.path.join(OUT, v2xvit.MODULE_GOLDEN))
    data = make_golden.small_scene()
    bargs = baseline_v2xvit_args()
    bm = HeterModelBaseline(copy.deepcopy(bargs)).eval()
    shapes = load_procedural(bm)
    with torch.no_grad():
        bout = bm(copy.deepcopy(data))
    golden.save({"args": bargs, "shapes": shapes, "data": data,
                 "out": {k: bout[k] for k in ("cls_preds", "reg_preds", "dir_preds")}},
                os.path.join(OUT, "heter_model_baseline_v2xvit_small.pt"))
    print("heter_model_baseline_v2xvit_small:", {k: tuple(v.shape) for k, v in bout.items() if torch.is_tensor(v)})
    for f in ("fusion_v2xvit.pt.xz", "heter_model_baseline_v2xvit_small.pt.xz"):
        print(f, os.path.getsize(os.path.join(OUT, f)) // 1024, "KiB")


if __name__ == "__main__":
    main()
