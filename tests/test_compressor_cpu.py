"""CPU checks of `compressor:`: the mirror keeps the reference's state-dict keys, the packing of heal_conv3x3_narrow_tc
restates the conv (+ folded BN) exactly up to the hi / lo split, training stays refused, and the agent-sharded path refuses a
compressed model."""
import copy

import pytest
import torch
import torch.nn as nn

from oracle import make_golden, make_golden_compressor as mgc


def test_state_dict_keys_are_the_references():
    from heal_b200.models.sub_modules.naive_compress import NaiveCompressor
    keys = set(NaiveCompressor(64, 8).state_dict())
    want = {f"{s}.{k}" for s in ("encoder.0", "decoder.0", "decoder.3") for k in ("weight", "bias")}
    want |= {f"{s}.{k}" for s in ("encoder.1", "decoder.1", "decoder.4")
             for k in ("weight", "bias", "running_mean", "running_var", "num_batches_tracked")}
    assert keys == want


@pytest.mark.parametrize("cin,cout", [(1, 64), (3, 256), (8, 64), (21, 256), (32, 256), (63, 64), (8, 48)])
def test_narrow_packing_restates_the_conv(cin, cout):
    """Unpack [nblk][kb][hi | lo][64][64] back to (Cout, Cin, 3, 3): hi + lo is the folded weight to bf16-pair precision, and
    every pad position (odd Cin's pad channel, k past 9 * cinp, channels past Cout) is zero."""
    from heal_b200 import ops
    torch.manual_seed(cin + cout)
    conv, bn = nn.Conv2d(cin, cout, 3, padding=1), nn.BatchNorm2d(cout, eps=1e-3)
    with torch.no_grad():
        bn.running_mean.normal_()
        bn.running_var.uniform_(0.5, 1.5)
        bn.weight.normal_()
    pc = ops.pack_conv3x3_narrow(conv.eval(), bn.eval(), True)
    nblk, kb = pc.w.shape[:2]
    cinp = cin + (cin & 1)
    assert pc.w.shape == (nblk, kb, 2, 64, 64) and nblk == (cout + 63) // 64 and kb * 64 >= 9 * cinp > kb * 64 - 64
    full = (pc.w[:, :, 0].float() + pc.w[:, :, 1].float())              # (nblk, kb, 64 rows, 64 k)
    mat = full.permute(0, 2, 1, 3).reshape(nblk * 64, kb * 64)
    scale = bn.weight.double() / torch.sqrt(bn.running_var.double() + bn.eps)
    w = (conv.weight.double() * scale[:, None, None, None]).permute(0, 2, 3, 1)   # (Cout, ky, kx, Cin)
    got = mat[:cout, :9 * cinp].reshape(cout, 3, 3, cinp)
    assert torch.allclose(got[..., :cin].double(), w, rtol=2 ** -15, atol=1e-30)
    assert not got[..., cin:].any() and not mat[:cout, 9 * cinp:].any() and not mat[cout:].any()
    b = bn.bias.double() - bn.running_mean.double() * scale + conv.bias.double() * scale
    assert torch.allclose(pc.bias.double(), b, rtol=1e-6, atol=1e-7)


def test_eligibility():
    from heal_b200 import ops
    assert ops.narrow_eligible(nn.Conv2d(8, 256, 3, padding=1))
    assert not ops.narrow_eligible(nn.Conv2d(64, 64, 3, padding=1))
    assert not ops.narrow_eligible(nn.Conv2d(8, 72, 3, padding=1))
    assert not ops.narrow_eligible(nn.Conv2d(8, 64, 3, padding=1, stride=2))


def _collab():
    from heal_b200.models.heter_pyramid_collab import HeterPyramidCollab
    return HeterPyramidCollab(copy.deepcopy(mgc.collab_compress_args()))


def test_training_stays_refused():
    """The reference's model_train_init leaves only the compressor in train mode: the forward refuses it like a model in train
    mode, and so does a model after .train()."""
    from heal_b200.models.heter_model_baseline import HeterModelBaseline
    for m in (_collab(), HeterModelBaseline(copy.deepcopy(mgc.baseline_compress_args()))):
        assert m.compress and m.compressor.training and not m.training
        assert all(p.requires_grad for p in m.compressor.parameters())
        assert not any(p.requires_grad for n, p in m.named_parameters() if not n.startswith("compressor."))
        with pytest.raises(NotImplementedError):
            m.compressor.forward_nhwc(None)
        m.eval()
        m.model_train_init()
        with pytest.raises(NotImplementedError):
            m.compressor.forward_nhwc(None)
        m.train()
        with pytest.raises(NotImplementedError):
            m({})


def test_agent_sharded_paths_refuse_a_compressed_model():
    from heal_b200 import parallel
    m = _collab().eval()
    with pytest.raises(NotImplementedError, match="compressor"):
        parallel.AgentShardedFrame(m, 3, 0, 1, 4096, (1, 5, 5, 4, 4))
    with pytest.raises(NotImplementedError, match="compressor"):
        parallel.forward_agent_sharded(m, make_golden.small_scene(), 0, 1)
