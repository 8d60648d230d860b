"""HeterModelBaselineMs (`core_method: heter_model_baseline_ms`, the CoAlign configs) on the GPU: the mirror against goldens of the
reference's own model in three precisions, the full-size lidar_coalign fusion stage against the oracle on the GPU, CUDA-graph
replay of a frame, and the reference's create_model returning the mirror once it is installed."""
import copy
import sys

import numpy as np
import pytest
import torch

from oracle import coalign, nets, procedural, ref_shim

pytestmark = pytest.mark.gpu

BF16_TOL = 2.5e-2
PREC = [("fp32", 1e-3), ("tc32", 1e-3), ("bf16", BF16_TOL)]


@pytest.fixture(autouse=True)
def _restore_precision():
    from heal_b200 import engine
    old = engine.PRECISION
    yield
    engine.set_precision(old)


def _tol_check(got, ref, tol, name):
    err = (got.float().cpu() - ref.float().cpu()).abs().max().item()
    scale = max(ref.abs().max().item(), 1.0)
    print(f"{name}: max|ref|={scale:.3f} max_abs_err={err:.3e}")
    assert err < tol * scale, (name, err, scale)


def _to_cuda(d):
    if torch.is_tensor(d):
        return d.cuda()
    if isinstance(d, dict):
        return {k: _to_cuda(v) for k, v in d.items()}
    return d


def _model(args, shapes):
    from heal_b200.models.heter_model_baseline_ms import HeterModelBaselineMs
    m = HeterModelBaselineMs(copy.deepcopy(args)).eval()
    m.load_state_dict(procedural.make_state_dict(shapes), strict=True)
    return m.cuda()


@pytest.mark.parametrize("name", coalign.GOLDENS)
@pytest.mark.parametrize("prec,tol", PREC)
def test_heter_model_baseline_ms_vs_reference_golden(golden_dir, name, prec, tol):
    from heal_b200 import engine
    engine.set_precision(prec)
    g = coalign.load_golden(golden_dir, name)
    m = _model(g["args"], g["shapes"])
    data = _to_cuda(g["data"])
    data["record_len"] = g["data"]["record_len"]
    with torch.no_grad():
        out = m(data)
    for k, ref in g["out"].items():
        assert out[k].shape == ref.shape, k
        _tol_check(out[k], ref, tol, f"{name}/{prec}/{k}")


def _fullsize_scene(n=5):
    """lidar_coalign.yaml: 5 agents on the +-102.4 m range, within 40 m of the ego, any heading."""
    from heal_b200 import synth
    g = torch.Generator().manual_seed(29)
    poses = [[0, 0, 0, 0, 0, 0]] + [[float(v) for v in ((torch.rand(2, generator=g) - 0.5) * 80).tolist()] +
                                    [0, 0, float(torch.rand(1, generator=g) * 360 - 180), 0] for _ in range(n - 1)]
    pw = torch.from_numpy(synth.pairwise_t_matrix(poses, n)[None])
    return torch.tensor([n]), nets.normalize_pairwise_tfm(pw, 204.8, 204.8, 1)


@pytest.mark.parametrize("method", ["att", "max"])
def test_fullsize_fusion_stage_vs_oracle_on_gpu(method):
    """The fusion stage of a lidar_coalign frame (5 agents; 256^2 x 64, 128^2 x 128 and 64^2 x 256 level maps) in tc32 against the
    oracle run by PyTorch on the GPU in fp32 with TF32 off."""
    from heal_b200 import engine, ops
    from heal_b200.models.fuse_modules.fusion_in_one import AttFusion, MaxFusion
    engine.set_precision("tc32")
    rl, aff = _fullsize_scene()
    aff = aff.cuda()
    g = torch.Generator().manual_seed(31)
    tf32 = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    args = coalign.coalign_args(method)
    try:
        for i, (C, hw) in enumerate(((64, 256), (128, 128), (256, 64))):
            x = (torch.randn(5, C, hw, hw, generator=g) * 0.5).cuda()
            xa = ops.convert(ops.to_act(x), engine.act_fmt())           # the level map as the conv engine hands it over
            xr = ops.act_to_nchw(xa).contiguous()                        # the values the kernel reads
            fuse = AttFusion(C) if method == "att" else MaxFusion()
            with torch.no_grad():
                ref = coalign.fuse_levels([xr] * (i + 1), args, rl, aff)[i]
                got = ops.act_to_nchw(fuse.forward_nhwc(xa, rl, aff))
            _tol_check(got, ref, 1e-3, f"fullsize/{method}/level{i} ({hw}^2 x {C})")
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32


def test_graph_replay_is_bit_identical():
    """A HeterModelBaselineMs frame (3 agents, att) captured in a FrameGraph replays bit for bit what the eager forward gives."""
    from heal_b200 import engine, synth
    from heal_b200.graph import FrameGraph
    engine.set_precision("tc32")
    args = coalign.coalign_args("att", supervise_single=True)
    from heal_b200.models.heter_model_baseline_ms import HeterModelBaselineMs
    m = _model(args, procedural.shapes_of(HeterModelBaselineMs(copy.deepcopy(args))))
    sc = synth.scene(3, n_agents=3, rings=16, azimuth=256)
    pts = torch.from_numpy(np.concatenate(sc["points"])).cuda()
    offs = torch.from_numpy(np.concatenate([[0], np.cumsum([p.shape[0] for p in sc["points"]])]).astype(np.int32)).cuda()
    pw = torch.from_numpy(sc["pairwise_t_matrix"]).cuda()
    fg = FrameGraph(m, 3, pts.shape[0] + 64, pw.shape)
    fg.load(pts, offs, pw)
    out = fg.replay()
    torch.cuda.synchronize()
    got = {k: v.clone() for k, v in out.items() if torch.is_tensor(v)}
    data = {"inputs_m1": {"points": pts, "agent_offsets": offs}, "agent_modality_list": ["m1"] * 3, "record_len": [3],
            "pairwise_t_matrix": pw}
    with torch.no_grad():
        eager = m(data)
    torch.cuda.synchronize()
    assert set(got) == {k for k, v in eager.items() if torch.is_tensor(v)}
    for k, v in got.items():
        assert torch.equal(v, eager[k]), k
    assert fg.replay() is out
    torch.cuda.synchronize()
    for k, v in got.items():
        assert torch.equal(out[k], v), k


@pytest.fixture
def _isolate_opencood_modules():
    before = {k: v for k, v in sys.modules.items() if k.startswith(("opencood", "shapely"))}
    yield
    for k in [k for k in sys.modules if k.startswith(("opencood", "shapely"))]:
        del sys.modules[k]
    sys.modules.update(before)


def test_create_model_returns_the_mirror(golden_dir, _isolate_opencood_modules):
    """After install_into_opencood(), the reference's own train_utils.create_model builds the mirror from a coalign `model:` block,
    and the reference-keyed checkpoint loads strictly."""
    if not ref_shim.available():
        pytest.skip("oracle/_ref not built")
    import types
    from unittest.mock import MagicMock
    from oracle import postprocess as opp
    sg = types.ModuleType("shapely.geometry")
    sg.Polygon, sg.Point, sg.MultiPoint = opp.QuadPolygon, MagicMock(), MagicMock()
    sh = types.ModuleType("shapely")
    sh.geometry = sg
    sys.modules["shapely"], sys.modules["shapely.geometry"] = sh, sg
    sys.modules.setdefault("opencood.utils.box_overlaps", MagicMock())
    ref_shim.install()
    from heal_b200 import install
    done = install.install_into_opencood()
    assert "opencood.models.heter_model_baseline_ms" in done
    from opencood.tools.train_utils import create_model
    g = coalign.load_golden(golden_dir, "att_small")
    model = create_model({"model": {"core_method": "heter_model_baseline_ms", "args": copy.deepcopy(g["args"])}})
    assert type(model).__module__ == "heal_b200.models.heter_model_baseline_ms"
    assert type(model).__name__ == "HeterModelBaselineMs"
    res = model.load_state_dict(procedural.make_state_dict(g["shapes"]), strict=True)
    assert not res.missing_keys and not res.unexpected_keys
