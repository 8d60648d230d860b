"""heal_agent_stack (csrc/agent_stack.cu): the agent assembly of a heterogeneous scene against a float64 restatement (zero-pad,
then slice, then stack: torchvision CenterCrop as the reference's forwards apply it), bit for bit; its refusals; and the three
heterogeneous forwards against the convert / crop / torch.cat sequence they ran before, on the hetero goldens."""
import copy
import os

import pytest
import torch
import torch.nn.functional as F

from oracle import golden

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _restore_precision():
    from heal_b200 import engine
    saved = engine.PRECISION
    yield
    engine.set_precision(saved)


def _map(n, h, w, c, fmt, seed, coffset=0, extra=0):
    """(n, h, w, c) seeded values as an Act in `fmt`, optionally a channel slice [coffset, coffset + c) of a wider map; also
    returns the float64 values the Act holds."""
    from heal_b200 import ops
    g = torch.Generator().manual_seed(seed)
    full = torch.randn(n, h, w, coffset + c + extra, generator=g) * 3
    full[..., ::7] = -0.0
    if fmt == "f32":
        t = full.cuda()
        held = full.double()
    else:
        t = ops.split_bf16(full, 2 if fmt == "split" else 1)
        held = (t[0].float() + t[1].float() if fmt == "split" else t[0].float()).double()     # hi + lo in fp32, -0.0 kept
        t = t.cuda()
    a = ops.Act(t, fmt)
    if coffset or extra:
        a = ops.Act(t[..., coffset:coffset + c], fmt)
    return a, held[..., coffset:coffset + c]


def _center(x, th, tw):
    """torchvision CenterCrop on (n, h, w, c): pad (left/top (t - s) // 2, right/bottom (t - s + 1) // 2) where the target is
    larger, then the window at int(round((s - t) / 2.0))."""
    n, h, w, c = x.shape
    if th > h or tw > w:
        ph, pw = max(th - h, 0), max(tw - w, 0)
        x = F.pad(x, (0, 0, pw // 2, (pw + 1) // 2, ph // 2, (ph + 1) // 2))
        n, h, w, c = x.shape
    top, left = int(round((h - th) / 2.0)), int(round((w - tw) / 2.0))
    return x[:, top:top + th, left:left + tw]


def _reference(held, aml, crops, H, W):
    cnt = {m: 0 for m in held}
    rows = []
    for m in aml:
        x = held[m][cnt[m]:cnt[m] + 1]
        rows.append(_center(x, *crops[m]) if m in crops else x)
        cnt[m] += 1
    return torch.cat(rows).float()


def _as_fmt(ref32, fmt):
    from heal_b200 import ops
    return ref32 if fmt == "f32" else ops.split_bf16(ref32, 2 if fmt == "split" else 1)


# (name, {m: (images, h, w, fmt, crop target or None)}, agent_modality_list, channels)
CASES = [
    ("f32_crop_odd", {"m1": (2, 20, 24, "f32", None), "m2": (1, 27, 31, "f32", (20, 24))}, ["m1", "m2", "m1"], 64),
    ("bf16_pad_odd", {"m1": (2, 20, 24, "bf16", None), "m2": (2, 13, 15, "bf16", (20, 24))}, ["m2", "m1", "m2", "m1"], 64),
    ("split_crop_pad", {"m1": (1, 20, 24, "split", None), "m3": (2, 25, 17, "split", (20, 24))}, ["m3", "m1", "m3"], 64),
    # mixed formats in one call, modality agents not adjacent, crop differences 1, 3, 5, 7 (round-half-even offsets)
    ("mixed_formats", {"m1": (2, 16, 16, "split", None), "m2": (1, 17, 19, "bf16", (16, 16)), "m3": (1, 21, 23, "f32", (16, 16)),
                       "m4": (2, 8, 12, "f32", (16, 16))}, ["m1", "m4", "m2", "m1", "m3", "m4"], 32),
    ("single_modality_lidar", {"m1": (3, 12, 10, "bf16", None)}, ["m1", "m1", "m1"], 64),
    ("single_modality_camera", {"m2": (2, 11, 14, "split", (16, 12))}, ["m2", "m2"], 64),
    ("scalar_channels", {"m1": (1, 9, 9, "f32", None), "m2": (1, 12, 6, "bf16", (9, 9))}, ["m2", "m1"], 6),
    ("pad_one_axis_crop_other", {"m1": (1, 10, 10, "f32", None), "m2": (1, 7, 14, "split", (10, 10))}, ["m1", "m2"], 8),
]


@pytest.mark.parametrize("name,maps,aml,C", CASES, ids=[c[0] for c in CASES])
@pytest.mark.parametrize("out_fmt", ["f32", "bf16", "split"])
def test_agent_stack_equals_pad_slice_stack(name, maps, aml, C, out_fmt):
    from heal_b200 import ops
    feats, held, crops = {}, {}, {}
    for i, (m, (n, h, w, fmt, crop)) in enumerate(maps.items()):
        feats[m], held[m] = _map(n, h, w, C, fmt, seed=11 * i + len(name))
        if crop is not None:
            crops[m] = crop
    H, W = next((maps[m][1], maps[m][2]) for m in maps if maps[m][4] is None) if len(crops) < len(maps) else \
        next(iter(crops.values()))
    out = ops.agent_stack(feats, aml, crops, fmt=out_fmt)
    torch.cuda.synchronize()
    ref = _as_fmt(_reference(held, aml, crops, H, W), out_fmt)
    assert out.t.shape == ref.shape
    assert torch.equal(out.t.cpu().view(torch.int16 if out_fmt != "f32" else torch.int32),
                       ref.view(torch.int16 if out_fmt != "f32" else torch.int32)), name


def test_agent_stack_reads_channel_slices_and_writes_into_a_wider_map():
    """Views with a channel offset (the scalar path: offset 2) and the vector path (offset 4), into a channel slice of a wider
    output whose other channels stay untouched."""
    from heal_b200 import ops
    for co in (2, 4):
        a, ha = _map(2, 12, 12, 16, "split", 5, coffset=co, extra=4)
        b, hb = _map(1, 15, 13, 16, "f32", 6, coffset=co, extra=4)
        wide = torch.full((3, 12, 12, 24), 7.0, device="cuda")
        out = ops.Act(wide[..., 4:20], "f32")
        ops.agent_stack({"m1": a, "m2": b}, ["m1", "m2", "m1"], {"m2": (12, 12)}, out=out)
        torch.cuda.synchronize()
        ref = _reference({"m1": ha, "m2": hb}, ["m1", "m2", "m1"], {"m2": (12, 12)}, 12, 12)
        assert torch.equal(wide[..., 4:20].cpu().view(torch.int32), ref.view(torch.int32))
        assert (wide[..., :4] == 7).all() and (wide[..., 20:] == 7).all()


def test_agent_stack_python_checks():
    from heal_b200 import ops
    a, _ = _map(2, 8, 8, 16, "f32", 1)
    b, _ = _map(1, 9, 9, 16, "f32", 2)
    with pytest.raises(ValueError, match="scene is"):
        ops.agent_stack({"m1": a, "m2": b}, ["m1", "m2"])                 # an uncropped map of another size
    with pytest.raises(ValueError, match="3 m1 agents"):
        ops.agent_stack({"m1": a}, ["m1", "m1", "m1"])


REFUSALS = [
    ("no_sources", "HEAL_ERR_ARG"),
    ("no_agents", "HEAL_ERR_ARG"),
    ("nine_sources", "HEAL_ERR_UNSUPPORTED"),
    ("65_agents", "HEAL_ERR_UNSUPPORTED"),
    ("source_index", "HEAL_ERR_ARG"),
    ("image_index", "HEAL_ERR_ARG"),
    ("uncropped_size", "HEAL_ERR_ARG"),
    ("format", "HEAL_ERR_ARG"),
    ("null_source", "HEAL_ERR_ARG"),
    ("null_dst", "HEAL_ERR_ARG"),
    ("narrow_cstride", "HEAL_ERR_ARG"),
]


@pytest.mark.parametrize("what, error", REFUSALS)
def test_refusals(what, error):
    """Each bad call is refused by name, and nothing is launched."""
    from heal_b200 import ops
    from heal_b200._lib import lib, HealAct, HealStackSource
    buf = torch.zeros(1 << 16, dtype=torch.float32, device="cuda")
    C, H, W = 8, 4, 4

    def src(**kw):
        d = dict(data=buf.data_ptr(), fmt=0, cstride=C, images=2, height=H, width=W, center_crop=0)
        d.update(kw)
        return HealStackSource(HealAct(d["data"], d["fmt"], d["cstride"], 0, 0), d["images"], d["height"], d["width"],
                               d["center_crop"])

    n_src = {"no_sources": 0, "nine_sources": 9}.get(what, 1)
    srcs = (HealStackSource * 9)(*[src(fmt=3 if what == "format" else 0, data=0 if what == "null_source" else buf.data_ptr(),
                                       cstride=4 if what == "narrow_cstride" else C,
                                       height=H + 1 if what == "uncropped_size" else H) for _ in range(9)])
    n_agents = {"no_agents": 0, "65_agents": 65}.get(what, 2)
    agent_src = [1 if what == "source_index" else 0] * 65
    agent_img = [2 if what == "image_index" else 0] * 65
    dst = HealAct(0 if what == "null_dst" else buf.data_ptr(), 0, C, 0, 0)
    torch.cuda.synchronize()
    before = lib.heal_launch_count()
    with pytest.raises(RuntimeError, match=f"heal_agent_stack failed: {error}"):
        ops._call("heal_agent_stack", srcs, n_src, ops._host_i32(agent_src), ops._host_i32(agent_img), n_agents, C, dst, H, W)
    torch.cuda.synchronize()
    assert lib.heal_launch_count() == before


# ------------------------------------------------------------------------------------------------ the forwards, unchanged bits
def _legacy_stack(feats, aml, crops=None, fmt="f32", out=None):
    """The sequence the forwards ran before heal_agent_stack: convert to fp32, CenterCrop with torch pad / slicing, torch.cat."""
    from heal_b200 import ops
    from heal_b200.models.heter_pyramid_collab import HeterPyramidCollab
    crops = crops or {}
    f32 = {m: ops.convert(f, "f32").t for m, f in feats.items()}
    f32 = {m: HeterPyramidCollab._crop_tensor(f, *crops[m]) if m in crops else f for m, f in f32.items()}
    cnt = {m: 0 for m in f32}
    rows = []
    for m in aml:
        rows.append(f32[m][cnt[m]:cnt[m] + 1])
        cnt[m] += 1
    return ops.Act(torch.cat(rows, 0), "f32")


def _cuda(d):
    if torch.is_tensor(d):
        return d.cuda()
    if isinstance(d, dict):
        return {k: _cuda(v) for k, v in d.items()}
    return d


def _hetero_cases(golden_dir):
    """(name, model, data) of the hetero goldens: HeterPyramidCollab [m1, m2 EfficientNet, m1] and with a compressor,
    HeterModelBaselineMs [m1, m4 Resnet101, ...] and HeterModelBaseline att with a zero-padded LSS agent."""
    from heal_b200.models.heter_pyramid_collab import HeterPyramidCollab
    from heal_b200.models.heter_model_baseline_ms import HeterModelBaselineMs
    from oracle import efficientnet as oe, coalign, procedural
    out = []
    g = golden.load(os.path.join(golden_dir, "heter_pyramid_collab_effnet_small.pt"))
    m = HeterPyramidCollab(copy.deepcopy(g["args"])).eval()
    m.load_state_dict(oe.state_dict_of(g["shapes"]), strict=True)
    out.append(("collab_effnet", m.cuda(), _cuda(oe.collab_data())))
    g = coalign.load_golden(golden_dir, "att_hetero")
    m = HeterModelBaselineMs(copy.deepcopy(g["args"])).eval()
    m.load_state_dict(procedural.make_state_dict(g["shapes"]), strict=True)
    out.append(("baseline_ms_att_hetero", m.cuda(), _cuda(g["data"])))
    from scene_fixtures import baseline_camera_model, scene_batch
    m = baseline_camera_model()
    out.append(("baseline_att_lidar_camera", m, scene_batch("baseline", 1)))
    return out


@pytest.mark.parametrize("prec", ["fp32", "tc32", "bf16"])
def test_forwards_give_the_bits_of_the_convert_crop_cat_sequence(golden_dir, prec, monkeypatch):
    from heal_b200 import engine, ops
    engine.set_precision(prec)
    for name, m, data in _hetero_cases(golden_dir):
        with torch.no_grad():
            new = {k: v.clone() for k, v in m(data).items() if k.endswith("_preds")}
            with monkeypatch.context() as mp:
                mp.setattr(ops, "agent_stack", _legacy_stack)
                old = {k: v for k, v in m(data).items() if k.endswith("_preds")}
        torch.cuda.synchronize()
        for k in old:
            assert torch.equal(new[k], old[k]), (name, prec, k)
