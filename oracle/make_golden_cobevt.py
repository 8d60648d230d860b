"""Golden vectors for CoBEVT (TEST INFRASTRUCTURE ONLY): the UNMODIFIED reference CoBEVT (fusion_in_one.py:374-429) and
HeterModelBaseline with fusion_method cobevt, run on CPU with procedural weights.

    python -m oracle.make_golden_cobevt        (needs the reference package: oracle/_ref or HEAL_REFERENCE_ROOT)

relative_position_index is an int64 buffer of the state dict: every float key gets its procedural value and the module keeps
its own index.  Writes tests/golden/fusion_cobevt.pt.xz (module level: the cases of cobevt.module_cases(), seeded inputs not
stored, outputs stored as channel samples to keep the file small) and heter_model_baseline_cobevt_small.pt.xz (the
lidar_cobevt.yaml block on make_golden.small_scene(), a 32 x 32 fused map)."""
import copy
import os

import torch

from oracle import cobevt, golden, make_golden, procedural, ref_shim

OUT = make_golden.OUT
STRIDE = {"c64": 4, "c256": 8, "l2": 4}      # channel sampling of the stored outputs


def load_procedural(module):
    """Procedural values for every float key; the module's own relative_position_index buffers stay."""
    shapes = procedural.shapes_of(module)
    sd = module.state_dict()
    sd.update(procedural.make_state_dict(cobevt.float_shapes(shapes)))
    module.load_state_dict(sd, strict=True)
    return shapes


def baseline_cobevt_args():
    """make_golden.baseline_att_args with the `cobevt:` block of opv2v/LiDAROnly/lidar_cobevt.yaml (max_cav 5)."""
    args = make_golden.baseline_att_args()
    args["fusion_method"] = "cobevt"
    del args["att"]
    args["cobevt"] = cobevt.cobevt_args(256, 3, 5)
    return args


def main():
    ref_shim.install()
    torch.set_num_threads(8)
    from opencood.models.fuse_modules.fusion_in_one import CoBEVT
    from opencood.models.heter_model_baseline import HeterModelBaseline
    cases = {}
    for name, (args, _, _, _, L) in cobevt.module_cases().items():
        x, rl, pw = cobevt.case_inputs(name)
        aff = cobevt.case_affine(pw)
        m = CoBEVT(copy.deepcopy(args)).eval()
        shapes = load_procedural(m)
        with torch.no_grad():
            y = m(x, rl, aff)
        idx = m.layers[0].window_attention.fn.relative_position_index.clone()
        cases[name] = {"args": args, "shapes": shapes, "record_len": rl, "pairwise_t_matrix": pw, "affine": aff,
                       "index": idx, "stride": STRIDE[name], "out_s": y[:, ::STRIDE[name]].contiguous()}
        print(f"cobevt {name}:", tuple(y.shape), float(y.abs().max()))
    golden.save(cases, os.path.join(OUT, cobevt.MODULE_GOLDEN))
    data = make_golden.small_scene()
    bargs = baseline_cobevt_args()
    bm = HeterModelBaseline(copy.deepcopy(bargs)).eval()
    shapes = load_procedural(bm)
    with torch.no_grad():
        bout = bm(copy.deepcopy(data))
    golden.save({"args": bargs, "shapes": shapes, "data": data,
                 "out": {k: bout[k] for k in ("cls_preds", "reg_preds", "dir_preds")}},
                os.path.join(OUT, "heter_model_baseline_cobevt_small.pt"))
    print("heter_model_baseline_cobevt_small:", {k: tuple(v.shape) for k, v in bout.items() if torch.is_tensor(v)})
    for f in ("fusion_cobevt.pt.xz", "heter_model_baseline_cobevt_small.pt.xz"):
        print(f, os.path.getsize(os.path.join(OUT, f)) // 1024, "KiB")


if __name__ == "__main__":
    main()
