"""Golden vectors for tests/test_gpu_fullsize.py: the UNMODIFIED reference models (oracle/ref_runner.py) at full size on CPU.

The heads of a full-size frame hold millions of values, so each head is stored as a fixed, seeded sample of its flattened
elements (indices + values) together with its shape and max |value| (the scale of the relative tolerance).  The inputs are
not stored: the test regenerates the same scene / cloud from the seeds below, and the weights are the procedural ones
(workloads/procedural.py) that depend only on the {key: shape} table.

    python -m oracle.make_golden_fullsize        (needs the reference package: oracle/_ref or HEAL_REFERENCE_ROOT)
"""
import os

import numpy as np

from workloads import configs as wcfg, synth

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
HEADS = ("cls_preds", "reg_preds", "dir_preds")
SAMPLES = 16384
C2_SCENE_SEED, C2_AGENTS = 321, 5
C1_CLOUD_SEED = 77


def c2_scene():
    return synth.scene(C2_SCENE_SEED, n_agents=C2_AGENTS, max_cav=max(5, C2_AGENTS), rings=64, azimuth=1024)


def c1_cloud():
    return synth.lidar_cloud(np.random.default_rng(C1_CLOUD_SEED), rings=20, azimuth=1000)


def _sample(ref, seed):
    rng = np.random.default_rng(seed)
    rec = {}
    for i, k in enumerate(HEADS):
        a = ref[k].detach().float().cpu().numpy()
        idx = np.sort(rng.choice(a.size, size=min(SAMPLES, a.size), replace=False)).astype(np.int32)
        rec[f"{k}.shape"] = np.asarray(a.shape, dtype=np.int64)
        rec[f"{k}.index"] = idx
        rec[f"{k}.value"] = a.reshape(-1)[idx].astype(np.float32)
        rec[f"{k}.max_abs"] = np.float32(np.abs(a).max())
    return rec


def main():
    from oracle import ref_runner
    assert ref_runner.available(), "the reference package is needed (python -m oracle.build_ref)"
    sc = c2_scene()
    model, _ = ref_runner.build_model("heter_pyramid_collab", wcfg.c2_args())
    data, _ = ref_runner.c2_data({"clouds": sc["points"], "pairwise": sc["pairwise_t_matrix"]}, C2_AGENTS)
    np.savez_compressed(os.path.join(OUT, "fullsize_c2.npz"), **_sample(ref_runner.forward(model, data), 2))
    cloud = c1_cloud()
    model, _ = ref_runner.build_model("point_pillar", wcfg.c1_args())
    data, _ = ref_runner.c1_data(cloud)
    np.savez_compressed(os.path.join(OUT, "fullsize_c1.npz"), **_sample(ref_runner.forward(model, data), 1))


if __name__ == "__main__":
    main()
