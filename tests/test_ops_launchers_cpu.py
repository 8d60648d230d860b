"""CPU-only checks of heal_b200.ops as the C-ABI boundary: every public wrapper that launches carries the device guard, the
multi-cav post-processing takes its device from the anchors, and every launch goes through `_call`."""
import inspect
import os
import re

import torch


def _launchers(ops):
    """Module-level functions of ops whose own source calls the library."""
    out = {}
    for name, fn in vars(ops).items():
        if inspect.isfunction(fn) and fn.__module__ == ops.__name__:
            src = inspect.getsource(inspect.unwrap(fn))
            if "_call(" in src or "lib.heal_" in src:
                out[name] = fn
    return out


def test_every_public_launcher_is_device_guarded():
    from heal_b200 import ops
    launchers = _launchers(ops)
    assert {"conv2d_tc", "swap_attention", "window_attention", "box_decode_nms_multi"} <= set(launchers)
    unguarded = sorted(n for n, fn in launchers.items() if not n.startswith("_") and not hasattr(fn, "device_arg"))
    assert not unguarded, f"public ops wrappers without @_guard: {unguarded}"


def test_guard_resolves_the_first_device_argument():
    from heal_b200 import ops
    # _device_of ignores CPU tensors, so the resolver is checked for which argument it picks, with a stand-in for _device_of
    cuda_like = torch.zeros(1)
    assert ops._first_device_arg(1, None, "x") is None
    saved = ops._device_of
    try:
        ops._device_of = lambda a: torch.device("cuda", 0) if a is cuda_like else None
        assert ops._first_device_arg(3, cuda_like, torch.zeros(1)) is cuda_like
        assert ops._first_device_arg(3, out=cuda_like) is cuda_like
    finally:
        ops._device_of = saved


def test_box_decode_nms_multi_takes_its_device_from_the_anchors():
    from heal_b200 import ops
    anchors, cls = torch.zeros(7), torch.zeros(1)
    cavs = [{"cls": cls, "reg": cls, "anchors": anchors}, {"cls": cls, "reg": cls, "anchors": torch.zeros(7)}]
    resolve = ops.box_decode_nms_multi.device_arg
    assert resolve(cavs, 0.2, 0.15) is anchors
    assert resolve(cavs=cavs, score_threshold=0.2, nms_threshold=0.15) is anchors
    assert resolve([], 0.2, 0.15) is None


def test_every_launch_goes_through_call():
    from heal_b200 import ops
    src = open(os.path.join(os.path.dirname(ops.__file__), "ops.py")).read()
    assert "ctypes.byref" not in src
    assert not re.search(r"\bcheck\(rc,", src)
    # the only library calls outside _call are workspace / table-size queries and the profiler's launch counter
    direct = set(re.findall(r"\blib\.(heal_\w+)\(", src))
    assert all(s.endswith(("_workspace", "_table_size")) or s == "heal_launch_count" for s in direct), sorted(direct)
