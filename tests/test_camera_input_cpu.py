"""CPU checks of the camera input stage: oracle/camera_input.py against PIL + torchvision bit for bit, the host plan and the
coefficient tables against the reference and the oracle, the dataset hook, and the wrapper's argument checks."""
import dataclasses
import glob
import os
import sys
from unittest.mock import MagicMock

import numpy as np
import pytest
import torch

from oracle import camera_input as oci
from oracle import ref_shim

# (frame H0 x W0, resize_dims (W, H), crop box): the four shipped inference shapes, an upscale, odd sizes, one axis unchanged
# (each way), and crops past each edge of the resized frame
CASES = [
    ((600, 800), (512, 384), (0, -10, 512, 374)),
    ((600, 800), (448, 336), (0, -9, 448, 327)),
    ((1080, 1920), (512, 288), (0, -8, 512, 280)),
    ((600, 800), (704, 528), (0, 258, 704, 514)),
    ((50, 70), (134, 96), (3, -5, 120, 91)),
    ((37, 53), (29, 21), (1, 2, 28, 19)),
    ((40, 56), (56, 24), (4, 0, 52, 24)),
    ((40, 56), (32, 40), (0, 4, 32, 36)),
    ((33, 47), (40, 24), (-5, 0, 35, 24)),
    ((33, 47), (40, 24), (8, 0, 48, 24)),
    ((33, 47), (40, 24), (0, -6, 40, 18)),
    ((33, 47), (40, 24), (0, 8, 40, 32)),
    ((33, 47), (40, 24), (-9, -7, 49, 33)),
]


def _frame(H0, W0, seed):
    return np.random.default_rng(seed).integers(0, 256, (H0, W0, 3), dtype=np.uint8)


@pytest.mark.parametrize("case", range(len(CASES)))
def test_oracle_equals_pil_and_torchvision(case):
    Image = pytest.importorskip("PIL.Image")
    tv = pytest.importorskip("torchvision")
    (H0, W0), dims, box = CASES[case]
    norm = tv.transforms.Compose((tv.transforms.ToTensor(),
                                  tv.transforms.Normalize(mean=[0.485, 0.456, 0.406], std=[0.229, 0.224, 0.225])))
    f = _frame(H0, W0, 10 + case)
    ref = norm(Image.fromarray(f).resize(dims).crop(box)).numpy()
    got = oci.camera_input(f, dims, box)
    assert got.shape == ref.shape and got.dtype == np.float32
    assert np.array_equal(got.view(np.int32), ref.view(np.int32))


@pytest.mark.parametrize("case", range(len(CASES)))
def test_coefficient_tables_equal_the_oracle(case):
    from heal_b200.data_utils.camera_input import axis_table, span_rows, TILE_ROWS
    (H0, W0), (W, H), (l, t, r, b) = CASES[case]
    for in_size, out_size, first, n in ((W0, W, l, r - l), (H0, H, t, b - t)):
        tab = axis_table(in_size, out_size, first, n)
        assert tab.dtype == np.int32 and tab.shape[0] == n
        ref = oci.coefficients(in_size, out_size) if in_size != out_size else \
            [(i, np.array([1 << oci.PRECISION_BITS])) for i in range(out_size)]
        for i in range(n):
            o = first + i
            if not 0 <= o < out_size:
                assert tab[i, 1] == 0
                continue
            start, w = ref[o]
            assert (tab[i, 0], tab[i, 1]) == (start, len(w))
            assert np.array_equal(tab[i, 2:2 + len(w)], w) and not tab[i, 2 + len(w):].any()
    rows = axis_table(H0, H, t, b - t)
    need = 1
    for y0 in range(0, b - t, TILE_ROWS):
        idx = [y for y in range(y0, min(y0 + TILE_ROWS, b - t)) if rows[y, 1] > 0]
        if idx:
            need = max(need, max(rows[y, 0] + rows[y, 1] for y in idx) - min(rows[y, 0] for y in idx))
    assert span_rows(rows) == need


def _shipped_confs():
    if not ref_shim.available():
        pytest.skip("reference package not available")
    import yaml
    confs = {}

    def walk(o):
        if isinstance(o, dict):
            if "data_aug_conf" in o and isinstance(o["data_aug_conf"], dict):
                c = o["data_aug_conf"]
                confs[repr(sorted(c.items()))] = c
            for v in o.values():
                walk(v)
        elif isinstance(o, list):
            for v in o:
                walk(v)

    for p in glob.glob(os.path.join(ref_shim.REFERENCE_ROOT, "opencood", "hypes_yaml", "**", "*.yaml"), recursive=True):
        try:
            with open(p) as fh:
                walk(yaml.load(fh, Loader=yaml.Loader))
        except yaml.YAMLError:
            continue
    return list(confs.values())


def _camera_utils():
    ref_shim.install()
    import opencood.utils.camera_utils as cu
    return cu


def test_inference_plan_equals_the_reference_for_every_shipped_conf():
    from heal_b200.data_utils.camera_input import inference_plan
    confs = _shipped_confs()
    assert len(confs) >= 3
    cu = _camera_utils()
    seen = set()
    for conf in confs:
        for H0, W0 in ((conf["H"], conf["W"]), (conf["H"] + 7, conf["W"] - 5)):
            resize, dims, crop, flip, rotate = cu.sample_augmentation(conf, False)
            _, post_rot, post_tran = cu.img_transform([], torch.eye(2), torch.zeros(2), resize=resize, resize_dims=dims, crop=crop,
                                                      flip=flip, rotate=rotate)
            plan = inference_plan(conf, H0, W0)
            assert (plan.resize, plan.resize_dims, plan.crop) == (resize, tuple(dims), tuple(crop))
            assert plan.final_dim == tuple(conf["final_dim"]) and (plan.H0, plan.W0) == (H0, W0)
            assert plan.post_rot.dtype == post_rot.dtype and torch.equal(plan.post_rot, post_rot)
            assert plan.post_tran.dtype == post_tran.dtype and torch.equal(plan.post_tran, post_tran)
            seen.add((tuple(conf["final_dim"]), tuple(dims), tuple(crop)))
    # the shipped shapes of the issue's table: every one crops above the top of the resized frame
    assert {((384, 512), (512, 384), (0, -10, 512, 374)), ((336, 448), (448, 336), (0, -9, 448, 327)),
            ((288, 512), (512, 288), (0, -8, 512, 280))} <= seen
    plan = inference_plan({"H": 600, "W": 800, "final_dim": [256, 704], "bot_pct_lim": [0.0, 0.05]}, 600, 800)
    assert (plan.resize_dims, plan.crop) == ((704, 528), (0, 258, 704, 514))
    with pytest.raises(ValueError, match="bot_pct_lim"):
        inference_plan({"H": 600, "W": 800, "final_dim": [256, 704]}, 600, 800)


def test_hook_pair_ships_the_frame_and_the_reference_matrices():
    Image = pytest.importorskip("PIL.Image")
    from heal_b200.data_utils.camera_input import reference_pair
    cu = _camera_utils()
    img_transform, normalize_img = reference_pair(cu.img_transform, cu.normalize_img)
    conf = {"H": 60, "W": 80, "final_dim": [40, 48], "bot_pct_lim": [0.0, 0.05]}
    f = _frame(60, 80, 7)
    resize, dims, crop, flip, rotate = cu.sample_augmentation(conf, False)
    out, pr, pt = img_transform([Image.fromarray(f)], torch.eye(2), torch.zeros(2), resize=resize, resize_dims=dims, crop=crop,
                                flip=flip, rotate=rotate)
    _, rr, rt = cu.img_transform([Image.fromarray(f)], torch.eye(2), torch.zeros(2), resize=resize, resize_dims=dims, crop=crop,
                                 flip=flip, rotate=rotate)
    assert len(out) == 1 and out[0].dtype == torch.uint8 and torch.equal(out[0], torch.from_numpy(f))
    assert torch.equal(pr, rr) and torch.equal(pt, rt)
    assert normalize_img(out[0]) is out[0]
    # flip, rotate, a depth image or a non-RGB image: the reference's functions
    for kw, src in ((dict(flip=True, rotate=0), [Image.fromarray(f)]), (dict(flip=False, rotate=5.0), [Image.fromarray(f)]),
                    (dict(flip=False, rotate=0), [Image.fromarray(f), Image.fromarray(f[..., 0])]),
                    (dict(flip=False, rotate=0), [Image.fromarray(f[..., 0])])):
        got, gr, gt = img_transform(list(src), torch.eye(2), torch.zeros(2), resize=resize, resize_dims=dims, crop=crop, **kw)
        exp, er, et = cu.img_transform(list(src), torch.eye(2), torch.zeros(2), resize=resize, resize_dims=dims, crop=crop, **kw)
        assert all(isinstance(g, Image.Image) and g.size == e.size and g.tobytes() == e.tobytes() for g, e in zip(got, exp))
        assert torch.equal(gr, er) and torch.equal(gt, et)
    pil = cu.img_transform([Image.fromarray(f)], torch.eye(2), torch.zeros(2), resize=resize, resize_dims=dims, crop=crop,
                           flip=False, rotate=0)[0][0]
    assert torch.equal(normalize_img(pil), cu.normalize_img(pil))


def test_install_rebinds_the_six_dataset_modules():
    from heal_b200 import install
    ref_shim.install()
    added = []
    for name in ("pypcd", "opencood.utils.box_overlaps"):            # absent here; unused by the camera branch
        if name not in sys.modules:
            try:
                __import__(name)
            except ImportError:
                m = MagicMock(name=name)
                m.__path__, m.__spec__ = [], None
                sys.modules[name] = m
                added.append(name)
    try:
        done = install.install_gpu_camera_input()
        assert len(done) == 6
        for name in done:
            mod = sys.modules[name]
            assert mod.img_transform.reference is sys.modules["opencood.utils.camera_utils"].img_transform
            assert mod.normalize_img.reference is sys.modules["opencood.utils.camera_utils"].normalize_img
        assert install.install_gpu_camera_input() == done                # installing twice wraps the originals, not the hook
        for name in done:
            assert sys.modules[name].img_transform.reference is sys.modules["opencood.utils.camera_utils"].img_transform
    finally:
        for name in install.CAMERA_DATASETS:                              # stock datasets again for the tests that follow
            mod = sys.modules.get(name)
            if mod is not None and hasattr(mod.img_transform, "reference"):
                mod.img_transform, mod.normalize_img = mod.img_transform.reference, mod.normalize_img.reference
        for name in added:
            sys.modules.pop(name, None)


def test_wrapper_refuses_malformed_input():
    from heal_b200 import ops
    from heal_b200.data_utils.camera_input import inference_plan
    plan = inference_plan({"H": 60, "W": 80, "final_dim": [40, 48], "bot_pct_lim": [0.0, 0.05]}, 60, 80)
    ok = torch.zeros((2, 60, 80, 3), dtype=torch.uint8)
    with pytest.raises(TypeError, match="uint8"):
        ops.camera_input(ok.float(), plan)
    with pytest.raises(ValueError, match="RGB"):
        ops.camera_input(torch.zeros((2, 60, 80, 4), dtype=torch.uint8), plan)
    with pytest.raises(ValueError, match="contiguous"):
        ops.camera_input(torch.zeros((2, 80, 60, 3), dtype=torch.uint8).transpose(1, 2), plan)
    with pytest.raises(ValueError, match="plan was made"):
        ops.camera_input(torch.zeros((2, 61, 80, 3), dtype=torch.uint8), plan)
    with pytest.raises(ValueError, match="final_dim"):
        ops.camera_input(ok, dataclasses.replace(plan, crop=(2, -1, 50, 40)))
    with pytest.raises(ValueError, match="layout"):
        ops.camera_input(ok, plan, "nhwc")
    odd = inference_plan({"H": 60, "W": 80, "final_dim": [36, 48], "bot_pct_lim": [0.0, 0.05]}, 60, 80)
    with pytest.raises(ValueError, match="multiples of 8"):
        ops.camera_input(ok, odd, "s2d")
    with pytest.raises(RuntimeError, match="CUDA"):                      # no CPU fallback
        ops.camera_input(ok, plan)
