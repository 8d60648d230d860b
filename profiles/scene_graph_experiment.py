"""A mixed-modality intermediate-fusion scene served three ways: the eager forward, SceneGraph.replay() (one captured graph) and
FramePipeline.for_scene (pinned host inputs in, results out, frames overlapped).  The scene has the shape of
opv2v/MoreModality/HEAL/final_infer/m1m2m3m4.yaml: HeterPyramidCollab with m1 PointPillars, m2 Lift-Splat-Shoot EfficientNet,
m3 SECOND and m4 Lift-Splat-Shoot ResNet101, ConvNeXt aligners, 5 agents [m1, m2, m3, m4, m1] over +-102.4 m (256 x 256
fusion map), four 256 x 704 cameras per camera agent on a +-51.2 m grid (zero-padded to the lidar range), tc32, procedural
weights, synthetic 64-ring clouds.  Also times the agent assembly alone, the convert / crop / torch.cat sequence the forwards
ran before against one heal_agent_stack launch, and counts the bytes a frame copies back with boxes and with heads.  Needs a
GPU; prints the card and its power limit, which belong beside every number taken from the output.

    python profiles/scene_graph_experiment.py [--reps 5] [--iters 20] [--out DIR]

Times are CUDA events around blocks of `--iters` frames (ten times as many assembly calls), and for the pipeline a host clock
around `--iters` submits and the drain that brings the last result to the host; the arms alternate for `--reps` rounds after
warm-up and the table gives the median round.  The eager and graph arms read device-resident inputs; the pipeline reads pinned host
inputs and ends with the results on the host.  Before timing, the graph's heads are checked bit for bit against the eager ones.
"""
import argparse
import copy
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

AML = ["m1", "m2", "m3", "m4", "m1"]
CAMS, IMG_H, IMG_W = 4, 256, 704
CONVNEXT = {"core_method": "convnext", "spatial_align": False, "args": {"num_of_blocks": 3, "dim": 64}}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()


def scene_args():
    from workloads import configs
    a = configs.c4_args()                                   # m1 PointPillars + m2 LSS-ResNet101 at the yaml's sizes
    cam_backbone = a["m2"]["backbone_args"]
    m4 = a.pop("m2")
    m4["aligner_args"] = copy.deepcopy(CONVNEXT)
    m2 = copy.deepcopy(m4)
    m2["encoder_args"]["camera_encoder"] = "EfficientNet"
    a["m1"]["aligner_args"] = copy.deepcopy(CONVNEXT)
    a["m2"] = m2
    a["m3"] = {"core_method": "second", "sensor_type": "lidar", "encoder_args": configs.second_encoder_args(),
               "backbone_args": dict(cam_backbone, layer_strides=[1]), "aligner_args": copy.deepcopy(CONVNEXT)}
    a["m4"] = m4
    return a


def scene_batch(seed):
    from workloads import synth
    sc = synth.scene(seed, n_agents=len(AML))
    batch = {"agent_modality_list": list(AML), "record_len": torch.tensor([len(AML)]),
             "pairwise_t_matrix": torch.from_numpy(sc["pairwise_t_matrix"])}
    for m in ("m1", "m3"):
        clouds = [sc["points"][i] for i, a in enumerate(AML) if a == m]
        offs = np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds])]).astype(np.int32)
        batch[f"inputs_{m}"] = {"points": torch.from_numpy(np.concatenate(clouds)), "agent_offsets": torch.from_numpy(offs)}
    for m in ("m2", "m4"):
        rots, trans, intr, post_rots, post_trans = [torch.from_numpy(a) for a in synth.camera_rig(1, CAMS, IMG_H, IMG_W)]
        imgs = torch.randn(1, CAMS, 3, IMG_H, IMG_W, generator=torch.Generator().manual_seed(seed * 10 + int(m[1])))
        batch[f"inputs_{m}"] = {"imgs": imgs, "rots": rots, "trans": trans, "intrins": intr, "post_rots": post_rots,
                                "post_trans": post_trans}
    return batch


def to(d, fn):
    if torch.is_tensor(d):
        return fn(d)
    if isinstance(d, dict):
        return {k: to(v, fn) for k, v in d.items()}
    return d


def timed(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for i in range(iters):
        fn(i)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def legacy_stack(feats, aml, crops):
    """The agent assembly the forwards ran before heal_agent_stack: convert, CenterCrop with torch pad / slicing, torch.cat."""
    from heal_b200 import ops
    from heal_b200.models.heter_common import crop_tensor
    f32 = {m: ops.convert(f, "f32").t for m, f in feats.items()}
    f32 = {m: crop_tensor(f, *crops[m]) if m in crops else f for m, f in f32.items()}
    cnt = {m: 0 for m in f32}
    rows = []
    for m in aml:
        rows.append(f32[m][cnt[m]:cnt[m] + 1])
        cnt[m] += 1
    return ops.Act(torch.cat(rows, 0), "f32")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    opt = ap.parse_args()
    from heal_b200 import engine, ops
    from heal_b200.graph import FramePipeline, SceneGraph
    from heal_b200.models.heter_pyramid_collab import HeterPyramidCollab
    from oracle import make_golden
    from workloads import configs, procedural
    engine.set_precision("tc32")
    who = card()
    print(f"card: {who}")
    model = HeterPyramidCollab(scene_args()).eval()
    model.load_state_dict(procedural.make_state_dict(procedural.shapes_of(model)), strict=True)
    model = model.cuda()
    params = make_golden.postprocess_params(rng=tuple(configs.RANGE))
    host = [to(scene_batch(s), lambda t: t.pin_memory()) for s in (1, 2, 3)]
    dev = [to(h, lambda t: t.cuda()) for h in host]
    caps = {m: (max(int(h[f"inputs_{m}"]["points"].shape[0]) for h in host) + 4095) // 4096 * 4096 for m in ("m1", "m3")}
    caps.update({"m2": (CAMS, IMG_H, IMG_W), "m4": (CAMS, IMG_H, IMG_W)})
    pw_shape = tuple(host[0]["pairwise_t_matrix"].shape)

    def eager(i):
        return model(dev[i % 3])

    with torch.no_grad():
        for i in range(3):
            eager(i)
        graph = SceneGraph(model, AML, caps, pw_shape, params)
        for i in range(3):                                  # the graph's heads are the eager ones, bit for bit
            want = eager(i)
            graph.load(dev[i])
            got = graph.replay()
            torch.cuda.synchronize()
            assert all(torch.equal(got[k], want[k]) for k in ("cls_preds", "reg_preds", "dir_preds")), i
        pipes = {"boxes": FramePipeline.for_scene(model, AML, caps, pw_shape, postprocess_params=params),
                 "heads": FramePipeline.for_scene(model, AML, caps, pw_shape)}

        def replay(i):
            graph.load(dev[i % 3])
            return graph.replay()

        def piped(pipe):
            def run(iters):                                 # host clock: the last result is on the host when it stops
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for i in range(iters):
                    pipe.submit(host[i % 3])
                pipe.drain()
                return (time.perf_counter() - t0) * 1e3 / iters
            return run

        # the agent assembly alone, on the scene's own post-aligner maps (engine formats)
        feats, crops = {}, {}
        d = dev[0]
        for m in ("m1", "m2", "m3", "m4"):
            feats[m], crop = model._agent_feature(d, m, {})
            if crop is not None:
                crops[m] = crop
        assert torch.equal(ops.agent_stack(feats, AML, crops).t, legacy_stack(feats, AML, crops).t)
        arms = {"eager": lambda n: timed(eager, n), "scene_graph": lambda n: timed(replay, n),
                "pipeline_boxes": piped(pipes["boxes"]), "pipeline_heads": piped(pipes["heads"]),
                "assembly_old": lambda n: timed(lambda i: legacy_stack(feats, AML, crops), 10 * n),
                "assembly_agent_stack": lambda n: timed(lambda i: ops.agent_stack(feats, AML, crops), 10 * n)}
        for fn in arms.values():                            # warm-up
            fn(3)
        runs = {name: [] for name in arms}
        for _ in range(opt.reps):
            for name, fn in arms.items():
                runs[name].append(fn(opt.iters))
    med = {k: statistics.median(v) for k, v in runs.items()}
    feats_bytes = {m: f.N * f.H * f.W * f.C * ops.BPE[f.fmt] for m, f in feats.items()}
    res = {"card": who, "precision": "tc32", "agents": AML, "point_capacity": caps["m1"],
           "ms": med, "ms_all": runs,
           "frames_per_s": {k: 1e3 / med[k] for k in ("eager", "scene_graph", "pipeline_boxes", "pipeline_heads")},
           "kernels_per_replay": graph.kernels_per_replay,
           "d2h_bytes_per_frame": {k: p.d2h_bytes for k, p in pipes.items()},
           "h2d_bytes_per_frame": pipes["boxes"].h2d_bytes,
           "assembly_input_bytes": feats_bytes,
           "assembly_formats": {m: f.fmt for m, f in feats.items()}}
    print(f"{'arm':<22}{'ms':>10}{'frames/s':>12}")
    for k in ("eager", "scene_graph", "pipeline_boxes", "pipeline_heads"):
        print(f"{k:<22}{med[k]:>10.3f}{1e3 / med[k]:>12.1f}")
    for k in ("assembly_old", "assembly_agent_stack"):
        print(f"{k:<22}{med[k]:>10.3f}")
    print(f"D2H bytes per frame: boxes {pipes['boxes'].d2h_bytes}, heads {pipes['heads'].d2h_bytes}; "
          f"H2D bytes per frame {pipes['boxes'].h2d_bytes}; {graph.kernels_per_replay} kernels per replay")
    if opt.out:
        os.makedirs(opt.out, exist_ok=True)
        with open(os.path.join(opt.out, "scene_graph_experiment.json"), "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
