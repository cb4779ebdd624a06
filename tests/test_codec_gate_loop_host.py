"""Host checks of SoundStream(use_gate_loop_layers=True): the oracle restatement against the reference
(tests/golden/gate_loop.pt), the state-dict surface, the weight folding and which configurations the tensor-core plans
take."""

import math

import pytest
import torch

from oracle import golden

PARTS = ("encoder", "decoder", "rq")


@pytest.fixture(scope="module")
def g():
    return golden.load("gate_loop.pt")


def _keys(ss):
    return [(k, tuple(v.shape)) for k, v in ss.state_dict().items() if k.split(".")[0] in PARTS]


def test_linear_scan_matches_sequential_recurrence():
    from oracle.codec_gate_loop import linear_scan

    gen = torch.Generator().manual_seed(3)
    a = torch.rand(2, 3, 301, generator=gen, dtype=torch.float64)
    kv = torch.randn(2, 3, 301, generator=gen, dtype=torch.float64)
    h, ref = torch.zeros(2, 3, dtype=torch.float64), []
    for t in range(301):
        h = a[..., t] * h + kv[..., t]
        ref.append(h)
    assert torch.allclose(linear_scan(a, kv), torch.stack(ref, -1), rtol=1e-12, atol=1e-12)


def test_oracle_matches_reference(g):
    from oracle import codec_gate_loop as ogl
    from oracle.transformer import sub

    s = g["small"]
    st, wave = s["state"], s["wave"]
    enc = ogl.encoder(sub(st, "encoder"), wave[:, None, :])
    assert (enc - s["enc"]).abs().max() < 1e-4 * s["enc"].abs().max()
    quant, idx = ogl.soundstream_tokenize(st, wave)
    assert torch.equal(idx, s["idx"])
    assert (quant - s["quant"]).abs().max() < 1e-5
    recon = ogl.soundstream_decode_indices(st, idx)
    assert (recon - s["recon"]).abs().max() < 1e-4 * s["recon"].abs().max()


def test_state_dict_matches_reference_small(g):
    from audiolm_pytorch_b200 import SoundStream

    s = g["small"]
    ss = SoundStream(**s["kwargs"])
    assert _keys(ss) == s["keys"]
    assert ("encoder.2.fn.fn.norm.gamma", (8,)) in s["keys"]
    assert ("decoder.8.fn.fn.to_qkva.0.weight", (12, 4)) in s["keys"]
    ss.load_state_dict(s["state"], strict=True)


def test_state_dict_matches_reference_c1(g):
    from audiolm_pytorch_b200 import SoundStream

    c1 = g["c1"]
    assert _keys(SoundStream(**c1["kwargs"])) == c1["keys"]


def test_default_soundstream_has_no_gate_loop_modules():
    from audiolm_pytorch_b200 import SoundStream

    keys = SoundStream(codebook_size=64, channels=4, codebook_dim=32, use_local_attn=False).state_dict().keys()
    assert not any(".fn.fn." in k for k in keys)
    assert "encoder.2.0.fn.0.conv.weight" in keys   # blocks keep consecutive indices without gate loops


def test_folded_weight_matches_fp64():
    from audiolm_pytorch_b200 import ops

    gen = torch.Generator().manual_seed(5)
    C = 48
    w = torch.randn(3 * C, C, generator=gen)
    gamma = 1 + 0.3 * torch.randn(C, generator=gen)
    got = ops.gate_loop_fold_weight(w, gamma)
    ref = w.double() * gamma.double()[None, :] * math.sqrt(C)
    assert got.dtype == torch.float32 and got.shape == (3 * C, C)
    assert torch.equal(got, ref.float())


@pytest.mark.parametrize("C", [32, 128])
def test_tc_units_hold_each_slices_q_kv_a_rows(C):
    from audiolm_pytorch_b200 import ops

    w = torch.randn(3 * C, C, generator=torch.Generator().manual_seed(C))
    units = ops.pack_gate_loop_weights(w)
    ns = ops.gate_loop_slice(C)
    assert units.dtype == torch.bfloat16 and units.shape == (C // ns, C // 16, 2, 2, 3 * ns, 8)
    v = units.float().sum(2)                                         # hi + lo: [S, kk, cc, 3 ns, 8]
    back = v.permute(0, 3, 1, 2, 4).reshape(C // ns, 3, ns, C)       # [S, (q, kv, a), i, c]
    ref = w.reshape(3, C // ns, ns, C).permute(1, 0, 2, 3)
    assert (back - ref).abs().max() <= 2.0 ** -16 * w.abs().max()


def test_tc_plans_take_the_c1_gate_loop_model():
    from audiolm_pytorch_b200 import SoundStream

    ss = SoundStream(codebook_size=1024, use_gate_loop_layers=True, use_local_attn=False)
    first, blocks, last = ss._tc_plan()
    assert [gl.norm.gamma.numel() for _, _, gl in blocks] == [64, 128, 256, 512]
    first, blocks, last = ss._tc_plan_dec()
    assert [gl.norm.gamma.numel() for _, _, gl in blocks] == [256, 128, 64, 32]
    plain = SoundStream(codebook_size=1024, use_local_attn=False)
    assert all(gl is None for _, _, gl in plain._tc_plan()[1]) and all(gl is None for _, _, gl in plain._tc_plan_dec()[1])


def test_tc_plans_reject_what_the_kernels_do_not_take():
    from audiolm_pytorch_b200 import SoundStream
    from audiolm_pytorch_b200 import soundstream as ss_mod

    # a 1024-channel gate loop after the last encoder block (and before the first decoder block's output) is outside
    # alm_codec_gate_loop_tc; the same model without gate loops is inside the conv plans
    kw = dict(codebook_size=64, channel_mults=(2, 4, 8, 32), codebook_dim=64, use_local_attn=False)
    assert SoundStream(**kw)._tc_plan() is not None
    assert SoundStream(**kw, use_gate_loop_layers=True)._tc_plan() is None
    # channels 4: the convs are outside the plans, so are the gate loops
    small = SoundStream(codebook_size=64, channels=4, codebook_dim=32, use_local_attn=False, use_gate_loop_layers=True)
    assert small._tc_plan() is None and small._tc_plan_dec() is None
    # a gate loop that does not follow a block
    ss = SoundStream(codebook_size=1024, use_gate_loop_layers=True, use_local_attn=False)
    enc = list(ss.encoder)
    enc[1], enc[2] = enc[2], enc[1]
    ss.encoder = torch.nn.Sequential(*enc)
    assert ss._tc_plan() is None
    old = ss_mod.ENCODER_ON_TENSOR_CORES
    try:
        ss_mod.ENCODER_ON_TENSOR_CORES = False
        assert SoundStream(codebook_size=1024, use_gate_loop_layers=True, use_local_attn=False)._tc_plan() is None
    finally:
        ss_mod.ENCODER_ON_TENSOR_CORES = old
