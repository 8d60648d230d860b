"""Storage of the golden vectors under tests/golden/ (TEST INFRASTRUCTURE ONLY).

A golden is a torch.save'd dict.  To keep every stored file small, `save` drops the inputs that oracle/make_golden.py draws
from fixed, seeded torch generators (they are regenerated bit for bit by `load`) and compresses the rest with xz, as
<name>.pt.xz; `load` accepts the plain <name>.pt too.
"""
import io
import lzma
import os

import torch


def _warp_att_x():
    return torch.randn(3, 128, 24, 40, generator=torch.Generator().manual_seed(11))


def _base_bev_x():
    g = torch.Generator().manual_seed(11)
    torch.randn(3, 128, 24, 40, generator=g)          # the warp_att input comes first from the same generator
    return torch.randn(2, 64, 32, 48, generator=g)


# postprocess.pt: (case, seed, logit mean) of make_golden.postprocess_inputs, and the seed of the iou_preds head
_PP_CASES = {"dense": (3, -3.0), "sparse": (4, -6.0)}
_PP_LATE2 = ((5, -4.0), (6, -4.0))
_PP_IOU = (7, -3.5, 17)


def _pp_heads(params, seed, mean):
    from oracle.make_golden import postprocess_inputs
    cls, reg, dirp, _ = postprocess_inputs(params, seed, mean)
    return {"cls": cls, "reg": reg, "dir": dirp}


def _strip(name, d):
    d = dict(d)
    if name == "warp_att.pt":
        assert torch.equal(d.pop("x"), _warp_att_x())
    elif name == "base_bev_backbone_small.pt":
        assert torch.equal(d.pop("x"), _base_bev_x())
    elif name == "postprocess.pt":
        cases = {k: dict(v) for k, v in d["cases"].items()}
        for k, (seed, mean) in _PP_CASES.items():
            for h, t in _pp_heads(d["params"], seed, mean).items():
                assert torch.equal(cases[k].pop(h), t)
        multi = {k: dict(v, cavs=[dict(c) for c in v["cavs"]]) for k, v in d["multi"].items()}
        for c, (seed, mean) in zip(multi["late2"]["cavs"], _PP_LATE2):
            for h, t in _pp_heads(d["params"], seed, mean).items():
                assert torch.equal(c.pop(h), t)
        c = multi["iou"]["cavs"][0]
        heads = _pp_heads(d["params"], *_PP_IOU[:2])
        for h, t in heads.items():
            assert torch.equal(c.pop(h), t)
        assert torch.equal(c.pop("iou"), torch.randn(heads["cls"].shape, generator=torch.Generator().manual_seed(_PP_IOU[2])))
        d["cases"], d["multi"] = cases, multi
    return d


def _restore(name, d):
    if name == "warp_att.pt":
        d["x"] = _warp_att_x()
    elif name == "base_bev_backbone_small.pt":
        d["x"] = _base_bev_x()
    elif name == "postprocess.pt":
        for k, (seed, mean) in _PP_CASES.items():
            d["cases"][k].update(_pp_heads(d["params"], seed, mean))
        for c, (seed, mean) in zip(d["multi"]["late2"]["cavs"], _PP_LATE2):
            c.update(_pp_heads(d["params"], seed, mean))
        c = d["multi"]["iou"]["cavs"][0]
        c.update(_pp_heads(d["params"], *_PP_IOU[:2]))
        c["iou"] = torch.randn(c["cls"].shape, generator=torch.Generator().manual_seed(_PP_IOU[2]))
    return d


def save(obj, path):
    """Write golden `obj` for tests/golden/<name>.pt as <name>.pt.xz without its seeded inputs."""
    buf = io.BytesIO()
    torch.save(_strip(os.path.basename(path), obj), buf)
    with lzma.open(path + ".xz", "wb", preset=9 | lzma.PRESET_EXTREME) as fh:
        fh.write(buf.getvalue())


def load(path):
    """The golden dict of tests/golden/<name>.pt (stored as <name>.pt or <name>.pt.xz)."""
    if os.path.exists(path):
        return torch.load(path, weights_only=False)
    with lzma.open(path + ".xz", "rb") as fh:
        d = torch.load(io.BytesIO(fh.read()), weights_only=False)
    return _restore(os.path.basename(path), d)
