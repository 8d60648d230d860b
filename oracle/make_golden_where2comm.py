"""Golden vectors for Where2commFusion / Who2comFusion (TEST INFRASTRUCTURE ONLY): the UNMODIFIED reference modules
(fusion_in_one.py:431-539, where2comm_attn.py EncodeLayer) and HeterModelBaseline with fusion_method where2comm / who2com, run
on CPU with procedural weights.

    python -m oracle.make_golden_where2comm        (needs the reference package: oracle/_ref or HEAL_REFERENCE_ROOT)

where2comm_attn.py imports `turtle` (unused) at module top; without tkinter that import fails, so a stub stands in for it.

Writes tests/golden/fusion_where2comm_who2com.pt.xz (module level; the seeded input where2comm.fusion_x() is not stored, and the
outputs are stored as every 16th channel to keep the file small) and heter_model_baseline_{where2comm,who2com}_small.pt.xz."""
import copy
import os
import sys
from unittest.mock import MagicMock

import numpy as np
import torch

from oracle import golden, make_golden, make_golden_fusion_methods as mgf, procedural, ref_shim, where2comm

OUT = make_golden.OUT
METHODS = ("where2comm", "who2com")


def install_reference():
    """ref_shim.install() with a stub for the `turtle` import of where2comm_attn.py when the real one cannot be imported."""
    try:
        import turtle  # noqa: F401
    except Exception:
        m = MagicMock(name="turtle")
        m.__spec__ = None
        sys.modules["turtle"] = m
    return ref_shim.install()


def fusion_scenes():
    """make_golden_fusion_methods.fusion_scenes() (record_len [3, 2]) plus a third scene of two agents whose ego-to-ego transform
    affine[2, 0, 0] is not the identity (a 7 degree turn and a shift), which tells the warped ego from the unwarped one."""
    rl, pw = mgf.fusion_scenes()
    from workloads import synth
    third = synth.pairwise_t_matrix([[0, 0, 0, 0, 0, 0], [-2.0, 1.2, 0, 0, 60, 0]], pw.shape[1])
    a = np.radians(7.0)
    third[0, 0] = np.array([[np.cos(a), -np.sin(a), 0, 0.9], [np.sin(a), np.cos(a), 0, -0.45], [0, 0, 1, 0], [0, 0, 0, 1]])
    return torch.cat([rl, torch.tensor([2])]), torch.cat([pw, torch.from_numpy(third)[None]])


def baseline_args(method):
    """make_golden.baseline_att_args with fusion_method `method` and its `method: 256` entry."""
    args = make_golden.baseline_att_args()
    args["fusion_method"] = method
    del args["att"]
    args[method] = 256
    return args


def main():
    install_reference()
    torch.set_num_threads(8)
    from opencood.models.fuse_modules.fusion_in_one import Where2commFusion, Who2comFusion
    from opencood.models.heter_model_baseline import HeterModelBaseline
    from opencood.utils.transformation_utils import normalize_pairwise_tfm
    record_len, pw = fusion_scenes()
    aff = normalize_pairwise_tfm(pw.clone(), 9.6, 16.0, 1)
    x = where2comm.fusion_x()
    d = {"record_len": record_len, "pairwise_t_matrix": pw, "H": 9.6, "W": 16.0, "affine": aff}
    for method, cls in zip(METHODS, (Where2commFusion, Who2comFusion)):
        m = cls(256).eval()
        shapes = procedural.shapes_of(m)
        m.load_state_dict(procedural.make_state_dict(shapes), strict=True)
        with torch.no_grad():
            y = m(x, record_len, aff)
        d[method] = {"shapes": shapes, "out_s": y[:, ::16].contiguous()}
        print(f"{method}:", tuple(y.shape), float(y.abs().max()))
    golden.save(d, os.path.join(OUT, where2comm.MODULE_GOLDEN))
    data = make_golden.small_scene()
    for method in METHODS:
        bargs = baseline_args(method)
        bm = HeterModelBaseline(copy.deepcopy(bargs)).eval()
        shapes = procedural.shapes_of(bm)
        bm.load_state_dict(procedural.make_state_dict(shapes), strict=True)
        with torch.no_grad():
            bout = bm(copy.deepcopy(data))
        golden.save({"args": bargs, "shapes": shapes, "data": data,
                     "out": {k: bout[k] for k in ("cls_preds", "reg_preds", "dir_preds")}},
                    os.path.join(OUT, f"heter_model_baseline_{method}_small.pt"))
        print(f"heter_model_baseline_{method}_small:", {k: tuple(v.shape) for k, v in bout.items() if torch.is_tensor(v)})
    for f in (where2comm.MODULE_GOLDEN, *(f"heter_model_baseline_{m}_small.pt" for m in METHODS)):
        print(f + ".xz", os.path.getsize(os.path.join(OUT, f + ".xz")) // 1024, "KiB")


if __name__ == "__main__":
    main()
