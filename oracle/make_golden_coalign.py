"""Golden vectors for HeterModelBaselineMs (TEST INFRASTRUCTURE ONLY): the UNMODIFIED reference model
(opencood/models/heter_model_baseline_ms.py:26-220) run on CPU with procedural weights.

    python -m oracle.make_golden_coalign        (needs the reference package: oracle/_ref or HEAL_REFERENCE_ROOT)

Writes tests/golden/heter_model_baseline_ms_{att_small,max_small,att_two_scenes,att_hetero}.pt.xz:
  att_small       att, PointPillar, make_golden.small_scene() (3 agents), supervise_single (in_head_single 64)
  max_small       max, the same scene
  att_two_scenes  att, two scenes in one batch (record_len [3, 2])
  att_hetero      att, agents [m1, m4, m1]: PointPillar + Lift-Splat-Shoot (Resnet101) with a camera grid wider than the lidar
                  range, so that the camera map is center-cropped (the seeded images of coalign.hetero_cam_inputs() are not stored)
The reference's LiftSplatShoot constructor moves its grid tensors to "cuda"; while the model is built here those moves stay on
the CPU (the reference source is not edited)."""
import contextlib
import copy
import os

import numpy as np
import torch

from oracle import coalign, golden, make_golden, procedural, ref_shim

OUT = make_golden.OUT


@contextlib.contextmanager
def _cuda_moves_stay_on_cpu():
    to = torch.Tensor.to

    def cpu_to(self, *a, **k):
        a = tuple(torch.device("cpu") if isinstance(v, torch.device) and v.type == "cuda" else v for v in a)
        if isinstance(k.get("device"), torch.device) and k["device"].type == "cuda":
            k["device"] = torch.device("cpu")
        return to(self, *a, **k)
    torch.Tensor.to = cpu_to
    try:
        yield
    finally:
        torch.Tensor.to = to


def two_scene_data():
    """5 PointPillar agents of make_golden.small_scene(seed 9) split into scenes of 3 and 2 (max_cav 5)."""
    from workloads import synth
    d = make_golden.small_scene(seed=9, n_agents=5)
    rng = np.random.default_rng(13)
    pw = []
    for n in (3, 2):
        poses = [[0, 0, 0, 0, 0, 0]] + [[rng.uniform(-5, 5), rng.uniform(-5, 5), 0, 0, rng.uniform(-180, 180), 0]
                                        for _ in range(n - 1)]
        pw.append(synth.pairwise_t_matrix(poses, 5))
    d["record_len"] = torch.tensor([3, 2], dtype=torch.long)
    d["pairwise_t_matrix"] = torch.from_numpy(np.stack(pw))
    return d


def hetero_data():
    """Agents [m1, m4, m1]: the lidar agents are the two of make_golden.small_scene(seed 11, 2 agents), the poses those of
    small_scene(seed 11, 3 agents)."""
    lidar = make_golden.small_scene(seed=11, n_agents=2)
    return {"inputs_m1": lidar["inputs_m1"], "inputs_m4": coalign.hetero_cam_inputs(),
            "agent_modality_list": list(coalign.HETERO_AML), "record_len": torch.tensor([3], dtype=torch.long),
            "pairwise_t_matrix": make_golden.small_scene(seed=11, n_agents=3)["pairwise_t_matrix"]}


def cases():
    return {"att_small": (coalign.coalign_args("att", supervise_single=True), make_golden.small_scene()),
            "max_small": (coalign.coalign_args("max"), make_golden.small_scene()),
            "att_two_scenes": (coalign.coalign_args("att"), two_scene_data()),
            "att_hetero": (coalign.hetero_args(), hetero_data())}


def main():
    ref_shim.install()
    torch.set_num_threads(8)
    from opencood.models.heter_model_baseline_ms import HeterModelBaselineMs
    for name, (args, data) in cases().items():
        with _cuda_moves_stay_on_cpu():
            m = HeterModelBaselineMs(copy.deepcopy(args)).eval()
        shapes = procedural.shapes_of(m)
        m.load_state_dict(procedural.make_state_dict(shapes), strict=True)
        with torch.no_grad():
            out = m(copy.deepcopy(data))
        keys = [k for k in ("cls_preds", "reg_preds", "dir_preds", "cls_preds_single", "reg_preds_single", "dir_preds_single")
                if k in out]
        stored = dict(data)
        stored.pop("inputs_m4", None)
        path = os.path.join(OUT, f"heter_model_baseline_ms_{name}.pt")
        golden.save({"args": args, "shapes": shapes, "data": stored, "out": {k: out[k] for k in keys}}, path)
        print(f"heter_model_baseline_ms_{name}: {len(shapes)} state-dict keys,", {k: tuple(out[k].shape) for k in keys},
              os.path.getsize(path + ".xz") // 1024, "KiB")


if __name__ == "__main__":
    main()
