"""CPU-only checks of ops.box_decode_nms_late's argument validation: every malformed call is refused by name before anything is
launched, and the wrapper carries the device guard."""
import pytest
import torch


def _act(N, H, W, C, fmt="f32"):
    from heal_b200 import ops
    a = object.__new__(ops.Act)          # an Act without a device buffer: validation reads only the geometry
    a.t, a.fmt, a.N, a.H, a.W, a.C = torch.zeros(0), fmt, N, H, W, C
    return a


@pytest.fixture
def no_cuda_check(monkeypatch):
    from heal_b200 import ops
    monkeypatch.setattr(ops, "_need_cuda", lambda *t: None)
    monkeypatch.setattr(ops, "_call", lambda *a: pytest.fail("launched"))


def _anchors(H=4, W=5, A=2):
    return torch.zeros((H, W, A, 7), dtype=torch.float32)


def test_is_device_guarded_and_listed_as_a_launcher():
    from heal_b200 import ops
    assert hasattr(ops.box_decode_nms_late, "device_arg")
    assert "heal_box_decode_nms_late" in open(ops.__file__).read()


@pytest.mark.parametrize("case,match", [
    ("bf16_heads", "fp32 heads"), ("bad_tensor", r"\(n_cav, C, H, W\)"), ("too_many_cavs", "1 to 16"),
    ("anchor_grid", "anchors must be"), ("reg_channels", "reg_preds needs 14 channels"),
    ("dir_offset", "dir_preds needs 4 channels from offset 2"), ("reg_batch", "reg_preds is"), ("transforms_cpu", "transforms must"),
    ("transforms_shape", "transforms must"), ("transforms_f64", "transforms must")])
def test_malformed_calls_are_refused(no_cuda_check, case, match):
    from heal_b200 import ops
    n, H, W, A = 3, 4, 5, 2
    cls, reg, dirp, anchors = _act(n, H, W, A), _act(n, H, W, 7 * A), _act(n, H, W, 2 * A), _anchors(H, W, A)
    T = torch.zeros((n, 4, 4))
    kw = {}
    if case == "bf16_heads":
        cls = _act(n, H, W, A, "bf16")
    elif case == "bad_tensor":
        cls = torch.zeros((n, A, H), dtype=torch.float32)
    elif case == "too_many_cavs":
        cls = _act(17, H, W, A)
    elif case == "anchor_grid":
        anchors = _anchors(H, W + 1, A)
    elif case == "reg_channels":
        reg = _act(n, H, W, 7 * A - 1)
    elif case == "dir_offset":
        kw["coffsets"] = (0, 0, 2)
    elif case == "reg_batch":
        reg = _act(n - 1, H, W, 7 * A)
    elif case == "transforms_shape":
        T = torch.zeros((n, 3, 4))
    elif case == "transforms_f64":
        T = torch.zeros((n, 4, 4), dtype=torch.float64)
    with pytest.raises(ValueError, match=match):
        ops.box_decode_nms_late(cls, reg, dirp, anchors, T, 0.2, 0.15, **kw)


def test_cpu_tensors_are_refused():
    from heal_b200 import ops
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.box_decode_nms_late(torch.zeros((2, 2, 4, 5)), torch.zeros((2, 14, 4, 5)), None, _anchors(), torch.zeros((2, 4, 4)),
                                0.2, 0.15)
