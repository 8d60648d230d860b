"""A stream of mixed-modality scenes whose agent list changes from frame to frame, served by SceneStream (one captured graph per
agent list and pipeline slot) against the eager forward on the same frames.  The model is the full-size m1m2m3m4 model of
scene_graph_experiment.py (HeterPyramidCollab: m1 PointPillars, m2 Lift-Splat-Shoot EfficientNet, m3 SECOND, m4 Lift-Splat-Shoot
ResNet101, ConvNeXt aligners, 256 x 256 fusion map, four 256 x 704 cameras per camera agent, tc32, procedural weights).  A
seeded generator draws `--lists` agent lists of 1 to 5 agents over the four modalities and a stream of `--frames` frames over
them.  Needs a GPU; prints the card and its power limit, which belong beside every number taken from the output.

    python profiles/scene_stream_experiment.py [--lists 6] [--frames 48] [--reps 3] [--out DIR]

It records:
- memory: `torch.cuda.memory_reserved()` growth of capturing every list into one slot (SceneStream, depth 1) against one
  stand-alone SceneGraph per list; each frame's boxes from the stream are compared bit for bit with its list's SceneGraph;
- capture time per new list: `SceneStream.capture(list)` at depth 2 (two graphs, one per slot), host clock around a
  device synchronise;
- frames/s: the stream (depth 2, pinned host inputs, boxes back on the host; host clock around the submits and the drain that
  brings the last result back) against the eager forward on the same frames (device-resident inputs, CUDA events), alternating
  for `--reps` rounds after a warm-up round; the median round is reported.
"""
import argparse
import gc
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import scene_graph_experiment as sge  # noqa: E402

MODALITIES = ("m1", "m2", "m3", "m4")
CAMS, IMG_H, IMG_W = sge.CAMS, sge.IMG_H, sge.IMG_W


def agent_lists(n, seed=5):
    """`n` distinct ordered agent lists of 1 to 5 agents (the ego first), every size present when n >= 5."""
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < n:
        size = len(out) % 5 + 1
        aml = [str(m) for m in rng.choice(MODALITIES, size)]
        if aml not in out:
            out.append(aml)
    return out


def scene_batch(aml, seed):
    """The collated ego batch of one frame of agent list `aml` (host tensors): 64-ring clouds, camera rigs, fp32 images."""
    from workloads import synth
    sc = synth.scene(seed, n_agents=len(aml))
    batch = {"agent_modality_list": list(aml), "record_len": torch.tensor([len(aml)]),
             "pairwise_t_matrix": torch.from_numpy(sc["pairwise_t_matrix"])}
    for m in dict.fromkeys(aml):
        k = aml.count(m)
        if m in ("m1", "m3"):
            clouds = [sc["points"][i] for i, a in enumerate(aml) if a == m]
            offs = np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds])]).astype(np.int32)
            batch[f"inputs_{m}"] = {"points": torch.from_numpy(np.concatenate(clouds)), "agent_offsets": torch.from_numpy(offs)}
        else:
            rots, trans, intr, post_rots, post_trans = [torch.from_numpy(a) for a in synth.camera_rig(k, CAMS, IMG_H, IMG_W)]
            imgs = torch.randn(k, CAMS, 3, IMG_H, IMG_W, generator=torch.Generator().manual_seed(seed * 10 + int(m[1])))
            batch[f"inputs_{m}"] = {"imgs": imgs, "rots": rots, "trans": trans, "intrins": intr, "post_rots": post_rots,
                                    "post_trans": post_trans}
    return batch


def settled():
    torch.cuda.synchronize()
    gc.collect()
    torch.cuda.empty_cache()
    return torch.cuda.memory_reserved()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lists", type=int, default=6)
    ap.add_argument("--frames", type=int, default=48)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    opt = ap.parse_args()
    from heal_b200 import engine
    from heal_b200.graph import SceneGraph, SceneStream
    from heal_b200.models.heter_pyramid_collab import HeterPyramidCollab
    from oracle import make_golden
    from workloads import configs, procedural
    engine.set_precision("tc32")
    who = sge.card()
    print(f"card: {who}")
    model = HeterPyramidCollab(sge.scene_args()).eval()
    model.load_state_dict(procedural.make_state_dict(procedural.shapes_of(model)), strict=True)
    model = model.cuda()
    params = make_golden.postprocess_params(rng=tuple(configs.RANGE))
    lists = agent_lists(opt.lists)
    uniq = [(aml, scene_batch(aml, 10 * i + r)) for i, aml in enumerate(lists) for r in range(2)]     # two frames per list
    order = np.random.default_rng(7).integers(0, len(uniq), opt.frames)
    host = [sge.to(b, lambda t: t.pin_memory()) for _, b in uniq]
    dev = [sge.to(h, lambda t: t.cuda()) for h in host]
    caps = {m: (max([int(h[f"inputs_{m}"]["points"].shape[0]) for h in host if f"inputs_{m}" in h] + [1]) + 4095) // 4096 * 4096
            for m in ("m1", "m3")}
    caps.update({"m2": (CAMS, IMG_H, IMG_W), "m4": (CAMS, IMG_H, IMG_W)})
    pw_shape = tuple(host[0]["pairwise_t_matrix"].shape)
    print(f"lists: {lists}; {opt.frames} frames over {len(uniq)} distinct scenes; capacities {caps}")

    with torch.no_grad():
        for d in dev:                                           # weight caches exist before any memory is measured
            model(d)
        # memory: every list captured into one slot, against a SceneGraph per list; the stream's boxes are the graphs' bits
        r0 = settled()
        one = SceneStream(model, caps, pw_shape, postprocess_params=params, depth=1)
        for aml in lists:
            one.capture(aml)
        shared = settled() - r0
        got = [{k: (v.clone() if torch.is_tensor(v) else v) for k, v in one.submit(h).items()} for h in host]
        del one
        r1 = settled()
        graphs = {tuple(aml): SceneGraph(model, aml, caps, pw_shape, params) for aml in lists}
        alone = settled() - r1
        for (aml, _), d, r in zip(uniq, dev, got):
            g = graphs[tuple(aml)]
            g.load(d)
            out = g.replay().get("postprocess")
            n = int(out.count.item())
            assert r["agent_modality_list"] == aml and int(r["count"][0]) == n, aml
            assert torch.equal(r["boxes"][:n], out.boxes[:n].cpu()) and torch.equal(r["scores"][:n], out.scores[:n].cpu()), aml
        kernels = {" ".join(k): g.kernels_per_replay for k, g in graphs.items()}
        del graphs
        settled()

        stream = SceneStream(model, caps, pw_shape, postprocess_params=params, depth=2)
        capture_ms = {}
        for aml in lists:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            stream.capture(aml)
            torch.cuda.synchronize()
            capture_ms[" ".join(aml)] = (time.perf_counter() - t0) * 1e3

        def eager():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for i in order:
                model(dev[i])
            b.record()
            torch.cuda.synchronize()
            return a.elapsed_time(b) / len(order)

        def streamed():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for i in order:
                stream.submit(host[i])
            stream.drain()
            return (time.perf_counter() - t0) * 1e3 / len(order)

        arms = {"eager": eager, "scene_stream": streamed}
        for fn in arms.values():                                # warm-up round
            fn()
        runs = {k: [] for k in arms}
        for _ in range(opt.reps):
            for k, fn in arms.items():
                runs[k].append(fn())
        assert stream.captures == 2 * len(lists)                # the timed rounds captured nothing
    med = {k: statistics.median(v) for k, v in runs.items()}
    res = {"card": who, "precision": "tc32", "lists": lists, "frames": int(opt.frames),
           "agents_per_frame": [len(uniq[i][0]) for i in order], "capacities": {m: list(v) if isinstance(v, tuple) else v
                                                                                for m, v in caps.items()},
           "ms_per_frame": med, "ms_per_frame_all": runs, "frames_per_s": {k: 1e3 / v for k, v in med.items()},
           "capture_ms_per_list_two_slots": capture_ms, "kernels_per_replay": kernels,
           "reserved_bytes": {"one_slot_all_lists": shared, "scene_graph_per_list": alone}}
    print(f"{'arm':<16}{'ms/frame':>10}{'frames/s':>10}")
    for k, v in med.items():
        print(f"{k:<16}{v:>10.3f}{1e3 / v:>10.1f}")
    for k, v in capture_ms.items():
        print(f"capture {k:<24}{v:>10.1f} ms (two slots)")
    print(f"reserved: one slot, all {len(lists)} lists {shared / 2**20:.1f} MiB; a SceneGraph per list {alone / 2**20:.1f} MiB")
    if opt.out:
        os.makedirs(opt.out, exist_ok=True)
        with open(os.path.join(opt.out, "scene_stream_experiment.json"), "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
