"""Golden vectors for MaxFusion / V2VNetFusion (TEST INFRASTRUCTURE ONLY): the UNMODIFIED reference modules
(fusion_in_one.py:87-124, :203-318) and HeterModelBaseline with fusion_method max / v2vnet, run on CPU with procedural weights.

    python -m oracle.make_golden_fusion_methods        (needs the reference package: oracle/_ref or HEAL_REFERENCE_ROOT)

Writes tests/golden/fusion_max_v2vnet.pt.xz (module level; the seeded input fusion_methods.fusion_x() is not stored, and the
outputs are stored as channel samples to keep the file under 1 MB) and heter_model_baseline_{max,v2vnet}_small.pt.xz."""
import copy
import os

import numpy as np
import torch

from oracle import fusion_methods, golden, make_golden, procedural, ref_shim

OUT = make_golden.OUT
V2V_VARIANTS = [("avg", True), ("max", True), ("avg", False), ("max", False)]


def v2vnet_args(C, H, W, agg="avg", gru=True, iterations=2):
    """`v2vnet:` block of opv2v/LiDAROnly/lidar_v2vnet.yaml with the channel count and map size of the test."""
    return {"num_iteration": iterations, "in_channels": C, "gru_flag": gru, "agg_operator": agg,
            "conv_gru": {"H": H, "W": W, "num_layers": 1, "kernel_size": [[3, 3]]}}


def fusion_scenes():
    """Two scenes, record_len [3, 2], max_cav 5, on a 9.6 m x 16 m (24 x 40) map: rotated and translated agents with parts of
    their maps out of the ego's view, and one sub-pixel translation (fractional V2VNet masks on the border)."""
    from workloads import synth
    scenes = [[[0, 0, 0, 0, 0, 0], [3.0, -1.5, 0, 0, 35, 0], [-4.0, 2.5, 0, 0, -120, 0]],
              [[0, 0, 0, 0, 0, 0], [0.07, 0.05, 0, 0, 0, 0]]]
    pw = np.stack([synth.pairwise_t_matrix(p, 5) for p in scenes])
    return torch.tensor([3, 2]), torch.from_numpy(pw)


def baseline_fusion_args(method):
    """make_golden.baseline_att_args with fusion_method `method` (small_scene: 64 x 64 pillars -> 32 x 32 fused map)."""
    args = make_golden.baseline_att_args()
    args["fusion_method"] = method
    del args["att"]
    if method == "v2vnet":
        args["v2vnet"] = v2vnet_args(256, 32, 32)
    return args


def main():
    ref_shim.install()
    torch.set_num_threads(8)
    from opencood.models.fuse_modules.fusion_in_one import MaxFusion, V2VNetFusion
    from opencood.models.heter_model_baseline import HeterModelBaseline
    from opencood.utils.transformation_utils import normalize_pairwise_tfm
    record_len, pw = fusion_scenes()
    aff = normalize_pairwise_tfm(pw.clone(), 9.6, 16.0, 1)
    x = fusion_methods.fusion_x()
    C, H, W = x.shape[1:]
    with torch.no_grad():
        mx = MaxFusion()(x, record_len, aff)
    v2v = {}
    for agg, gru in V2V_VARIANTS:
        a = v2vnet_args(C, H, W, agg, gru)
        m = V2VNetFusion(copy.deepcopy(a)).eval()
        shapes = procedural.shapes_of(m)
        m.load_state_dict(procedural.make_state_dict(shapes), strict=True)
        with torch.no_grad():
            y = m(x, record_len, aff)
        v2v[f"{agg}_gru{int(gru)}"] = {"args": a, "shapes": shapes, "out_s": y[:, ::4].contiguous()}
        print(f"v2vnet {agg} gru={gru}:", tuple(y.shape), float(y.abs().max()))
    golden.save({"record_len": record_len, "pairwise_t_matrix": pw, "H": 9.6, "W": 16.0, "affine": aff,
                 "max_s": mx[:, ::2].contiguous(), "v2vnet": v2v}, os.path.join(OUT, fusion_methods.MODULE_GOLDEN))
    print("fusion_max_v2vnet: max", tuple(mx.shape), float(mx.abs().max()))
    data = make_golden.small_scene()
    for method in ("max", "v2vnet"):
        bargs = baseline_fusion_args(method)
        bm = HeterModelBaseline(copy.deepcopy(bargs)).eval()
        shapes = procedural.shapes_of(bm)
        bm.load_state_dict(procedural.make_state_dict(shapes), strict=True)
        with torch.no_grad():
            bout = bm(copy.deepcopy(data))
        golden.save({"args": bargs, "shapes": shapes, "data": data,
                     "out": {k: bout[k] for k in ("cls_preds", "reg_preds", "dir_preds")}},
                    os.path.join(OUT, f"heter_model_baseline_{method}_small.pt"))
        print(f"heter_model_baseline_{method}_small:", {k: tuple(v.shape) for k, v in bout.items() if torch.is_tensor(v)})
    for f in ("fusion_max_v2vnet.pt.xz", "heter_model_baseline_max_small.pt.xz", "heter_model_baseline_v2vnet_small.pt.xz"):
        print(f, os.path.getsize(os.path.join(OUT, f)) // 1024, "KiB")


if __name__ == "__main__":
    main()
