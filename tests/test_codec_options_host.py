"""Host checks of SoundStream(squeeze_excite=True) and the bottleneck's head widths: constructors, state-dict surface
against the reference (tests/golden/codec_options.pt), the SE oracle against the reference, the weight folding."""

import pytest
import torch

from oracle import golden


@pytest.fixture(scope="module")
def g():
    return golden.load("codec_options.pt")


def test_squeeze_excite_state_dict_matches_reference(g):
    from audiolm_pytorch_b200 import SoundStream

    se = g["squeeze_excite"]
    ours = [(k, tuple(v.shape)) for k, v in SoundStream(**se["kwargs"]).state_dict().items()]
    assert ours == se["keys"]
    assert any(k.endswith("fn.4.net.0.weight") and s == (8, 4, 1) for k, s in ours)      # Ci = max(8, C // 4)
    assert any(k.endswith("fn.4.net.2.weight") and s == (32, 8, 1) for k, s in ours)
    ss = SoundStream(**se["kwargs"])
    ss.load_state_dict(se["state"], strict=True)


def test_default_soundstream_has_no_squeeze_excite_modules():
    from audiolm_pytorch_b200 import SoundStream

    keys = SoundStream(codebook_size=64, channels=4, codebook_dim=32, use_local_attn=False).state_dict().keys()
    assert not any(".fn.4." in k for k in keys)


def test_oracle_squeeze_excite_matches_reference(g):
    from oracle import codec_se as ose
    from oracle.transformer import sub

    se = g["squeeze_excite"]
    st, wave = se["state"], se["wave"]
    enc = ose.encoder(sub(st, "encoder"), wave[:, None, :])
    assert (enc - se["enc"]).abs().max() < 2e-5 * max(1.0, se["enc"].abs().max().item())
    _, idx = ose.soundstream_tokenize(st, wave)
    assert torch.equal(idx, se["idx"])
    recon = ose.soundstream_decode_indices(st, idx)
    assert (recon - se["recon"]).abs().max() < 2e-5 * max(1.0, se["recon"].abs().max().item())


def test_squeeze_excite_mean_is_over_channels():
    """the reference's SqueezeExcite cumsums dim -2 of [B, C, T]: permuting time steps permutes the output the same way"""
    from oracle import codec_se as ose

    gen = torch.Generator().manual_seed(3)
    C, Ci = 16, 8
    st = {"net.0.weight": torch.randn(Ci, C, 1, generator=gen), "net.0.bias": torch.randn(Ci, generator=gen),
          "net.2.weight": torch.randn(C, Ci, 1, generator=gen), "net.2.bias": torch.randn(C, generator=gen)}
    y = torch.randn(2, C, 11, generator=gen)
    perm = torch.randperm(11, generator=gen)
    assert torch.allclose(ose.squeeze_excite(st, y)[..., perm], ose.squeeze_excite(st, y[..., perm]), atol=1e-6)


def test_se_fold_weight_equals_cumulative_mean():
    from audiolm_pytorch_b200 import ops

    gen = torch.Generator().manual_seed(5)
    C, Ci = 64, 16
    w1 = torch.randn(Ci, C, 1, generator=gen)
    y = torch.randn(C, 7, generator=gen, dtype=torch.float64)
    m = y.cumsum(0) / torch.arange(1, C + 1, dtype=torch.float64)[:, None]
    ref = w1[..., 0].double() @ m
    got = ops.se_fold_weight(w1).double() @ y
    assert (got - ref).abs().max() < 1e-5 * ref.abs().max()


@pytest.mark.parametrize("C", [32, 64, 128, 256])
def test_pack_ru_se_weights_layout(C):
    """conv units first (unchanged), then the folded first SE conv and the second, zero-padded to NS inner channels"""
    from audiolm_pytorch_b200 import ops

    gen = torch.Generator().manual_seed(C)
    Ci = max(8, C // 4)
    ns = ops.se_inner_pad(C)
    w7, w1 = torch.randn(C, C, 7, generator=gen), torch.randn(C, C, 1, generator=gen)
    s1, s2 = torch.randn(Ci, C, 1, generator=gen), torch.randn(C, Ci, 1, generator=gen)
    packed = ops.pack_ru_se_weights(w7, w1, s1, s2)
    base = ops.pack_ru_weights(w7, w1).flatten()
    assert packed.dtype == torch.bfloat16
    assert packed.numel() == base.numel() + 2 * 2 * 8 * (C // 16 * ns + ns // 16 * C)
    assert torch.equal(packed[:base.numel()], base)
    n1 = (C // 16) * 2 * 2 * ns * 8
    u1 = packed[base.numel():base.numel() + n1].view(C // 16, 2, 2, ns, 8)       # [k-step][hi, lo][chunk][row][8]
    w1f = (u1[:, 0].float() + u1[:, 1].float()).permute(2, 0, 1, 3).reshape(ns, C)
    assert (w1f[:Ci] - ops.se_fold_weight(s1)).abs().max() < 1e-5 * s1.abs().max()
    assert torch.equal(w1f[Ci:], torch.zeros_like(w1f[Ci:]))
    u2 = packed[base.numel() + n1:].view(ns // 16, 2, 2, C, 8)
    w2 = (u2[:, 0].float() + u2[:, 1].float()).permute(2, 0, 1, 3).reshape(C, ns)
    assert (w2[:, :Ci] - s2[..., 0]).abs().max() < 1e-5 * s2.abs().max()
    assert torch.equal(w2[:, Ci:], torch.zeros_like(w2[:, Ci:]))


@pytest.mark.parametrize("dim_head", [32, 64, 128])
def test_bottleneck_head_widths_construct(dim_head):
    from audiolm_pytorch_b200 import SoundStream

    ss = SoundStream(codebook_size=64, channels=4, codebook_dim=32, attn_dim_head=dim_head, attn_heads=2)
    assert ss.encoder_attn.layers[0][0].q_scale.shape == (dim_head,)
    assert ss.decoder_attn.layers[0][0].to_qkv.weight.shape == (3 * 2 * dim_head, 32)


def test_bottleneck_state_dict_matches_reference(g):
    from audiolm_pytorch_b200 import SoundStream

    for dh, case in g["local_attn"].items():
        ss = SoundStream(**case["kwargs"])
        ss.load_state_dict(case["state"], strict=True)
        assert ss.encoder_attn.layers[0][0].dim_head == dh


def test_unbuilt_options_still_raise():
    from audiolm_pytorch_b200 import SoundStream

    kw = dict(codebook_size=64, channels=4, codebook_dim=32)
    with pytest.raises(NotImplementedError):
        SoundStream(attn_dim_head=48, **kw)
    with pytest.raises(NotImplementedError):
        SoundStream(attn_dynamic_pos_bias=True, **kw)
    SoundStream(squeeze_excite=True, **kw)
