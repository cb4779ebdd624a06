"""H100: SoundStream(squeeze_excite=True) on the tensor-core and CUDA-core codec kernels, and the local-attention
bottleneck at dim_head 32 and 128, against the reference (tests/golden/codec_options.pt) and the oracle restatements."""

import pytest
import torch
import torch.nn.functional as F

from oracle import golden

pytestmark = pytest.mark.gpu
DEV = "cuda"


def err(a, b):
    return (a.float().cpu() - b.float().cpu()).abs().max().item()


def rms_rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).pow(2).mean().sqrt() / b.pow(2).mean().sqrt().clamp(min=1e-12)).item()


def _se_state(C, seed):
    """an RU + SE parameter set at the scale of a trained unit (gates spread over (0, 1))"""
    g = torch.Generator().manual_seed(seed)
    Ci = max(8, C // 4)
    return {"fn.0.conv.weight": torch.randn(C, C, 7, generator=g) * (0.7 / (7 * C) ** 0.5),
            "fn.0.conv.bias": torch.randn(C, generator=g) * 0.1,
            "fn.2.conv.weight": torch.randn(C, C, 1, generator=g) * (0.7 / C ** 0.5),
            "fn.2.conv.bias": torch.randn(C, generator=g) * 0.1,
            "fn.4.net.0.weight": torch.randn(Ci, C, 1, generator=g) * (2.0 / C ** 0.5),
            "fn.4.net.0.bias": torch.randn(Ci, generator=g) * 0.3,
            "fn.4.net.2.weight": torch.randn(C, Ci, 1, generator=g) * (2.0 / Ci ** 0.5),
            "fn.4.net.2.bias": torch.randn(C, generator=g) * 0.3}


@pytest.mark.parametrize("C,T", [(32, 5000), (64, 3000), (128, 1500), (256, 700)])
@pytest.mark.parametrize("d,phases,mode", [(1, 1, "reflect"), (3, 1, "constant"), (9, 4, "reflect"), (9, 5, "reflect")])
def test_residual_unit_se_tc_vs_oracle(C, T, d, phases, mode):
    """alm_codec_ru_se_tc (two more wgmma GEMMs per tile, the second with its A operand in registers) vs the oracle
    restatement of soundstream.py:145-169, 362-369; ragged last tile, reflect / constant halo, phase-split output."""
    from audiolm_pytorch_b200 import ops
    from oracle import codec_se as ose

    st = _se_state(C, 300 + C + d)
    x = torch.randn(2, C, T, generator=torch.Generator().manual_seed(27 + d))
    ref = ose.residual_unit(st, x, d, pad_mode=mode)
    dv = {k: v.to(DEV) for k, v in st.items()}
    wu = ops.pack_ru_se_weights(dv["fn.0.conv.weight"], dv["fn.2.conv.weight"], dv["fn.4.net.0.weight"],
                                dv["fn.4.net.2.weight"])
    y = ops.codec_ru_se_tc(ops.c8s_pack(x.to(DEV)), wu, dv["fn.0.conv.bias"], dv["fn.2.conv.bias"],
                           dv["fn.4.net.0.bias"], dv["fn.4.net.2.bias"], dilation=d, pad_mode=mode, out_phases=phases)
    assert y.shape == (2, 2 * C // 8, phases, T // phases, 8)
    got = ops.c8s_unpack(y)
    scale = max(1.0, ref.abs().max().item())
    e = err(got, ref)
    print(f"RU+SE tc C={C} d={d}: max abs err {e:.2e} (scale {scale:.2f})")
    assert e < 1e-4 * scale
    assert err(got[..., :64], ref[..., :64]) < 1e-4 * scale
    # the SE term matters at this scale: dropping it would fail the bound by orders of magnitude
    from oracle import codec as oc
    assert err(oc.residual_unit(st, x, d, pad_mode=mode), ref) > 100 * 1e-4 * scale


@pytest.mark.parametrize("C,T", [(4, 3000), (8, 1000), (32, 5000), (64, 700), (256, 333)])
def test_se_fp32_vs_oracle(C, T):
    """alm_codec_se_fp32 through ResidualUnit.forward (the path of configurations outside the tensor-core plans)"""
    from audiolm_pytorch_b200 import soundstream as ss_mod
    from oracle import codec_se as ose

    st = _se_state(C, 400 + C)
    x = torch.randn(2, C, T, generator=torch.Generator().manual_seed(C))
    ref = ose.residual_unit(st, x, 3)
    ru = ss_mod.ResidualUnit(C, C, 3, squeeze_excite=True)
    ru.load_state_dict(st, strict=True)
    with torch.no_grad():
        got = ru.to(DEV).eval()(x.to(DEV))
    scale = max(1.0, ref.abs().max().item())
    assert err(got, ref) < 2e-5 * scale, (err(got, ref), scale)


def test_squeeze_excite_golden_end_to_end():
    from audiolm_pytorch_b200 import SoundStream

    g = golden.load("codec_options.pt")["squeeze_excite"]
    ss = SoundStream(**g["kwargs"])
    ss.load_state_dict(g["state"], strict=True)
    ss = ss.to(DEV).eval()
    wave = g["wave"].to(DEV)
    with torch.no_grad():
        enc = ss.encoder(wave[:, None, :])
        quant, idx, _ = ss(wave, return_encoded=True)
        recon = ss(wave, return_recons_only=True)
        recon_idx = ss.decode_from_codebook_indices(idx)
    assert err(enc, g["enc"]) < 1e-4
    assert torch.equal(idx.cpu(), g["idx"]), "RVQ indices must be bit-exact"
    assert err(quant, g["quant"]) < 1e-5
    assert err(recon, g["recon"]) < 1e-4
    assert err(recon_idx, recon) < 1e-5


def _c1_se_model(seed):
    from audiolm_pytorch_b200.soundstream import SoundStream

    torch.manual_seed(seed)
    ss = SoundStream(codebook_size=1024, rq_num_quantizers=8, target_sample_hz=24000, use_local_attn=False,
                     squeeze_excite=True)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for n_, p_ in ss.named_parameters():
            if ".fn.4." in n_:
                p_.add_(torch.randn(p_.shape, generator=g) * 0.2)
    return ss


def test_c1_encoder_se_and_rvq_indices_vs_oracle():
    """C1 encoder (32 channels, strides 2/4/5/8, 48 000 samples -> 150 frames) with SE units, on the tensor-core plan,
    + 8-stage RVQ: indices bit-exact on every margin-safe frame, the rule of test_c1_encoder_and_rvq_indices_vs_oracle"""
    from oracle import codec as oc
    from oracle import codec_se as ose
    from oracle.transformer import sub

    ss = _c1_se_model(22)
    g = torch.Generator().manual_seed(7)
    for layer in ss.rq.rvqs[0].layers:
        layer._codebook.embed.copy_(torch.randn(1, 1024, 512, generator=g) * 0.05)
        layer._codebook.initted.fill_(True)
    st = {k: v.detach().clone() for k, v in ss.state_dict().items()}
    wave = torch.randn(2, 48000, generator=g)
    torch.set_num_threads(min(32, torch.get_num_threads()))
    enc_ref = ose.encoder(sub(st, "encoder"), wave[:, None, :]).transpose(1, 2)
    cbs = oc.codebooks_of(st)
    flat = enc_ref.reshape(-1, 512)
    q_ref, i_ref = oc.rvq_encode(flat, cbs)
    margin = oc.rvq_margin(flat, cbs)
    ss = ss.to(DEV).eval()
    assert ss._tc_plan() is not None
    with torch.no_grad():
        enc = ss.encode_frames(wave.to(DEV)[:, None, :])
        quant, idx, _ = ss(wave.to(DEV), return_encoded=True)
    e = err(enc, enc_ref)
    scale = enc_ref.abs().max().item()
    print(f"C1 SE encoder max abs err {e:.3e} (scale {scale:.2f})")
    assert e < 2e-4 * max(1.0, scale)
    idx = idx.reshape(-1, 8).cpu()
    safe = margin > max(20 * e, 1e-4)
    print(f"margin-safe frames {safe.float().mean().item():.2%}, frames with any differing index "
          f"{(idx != i_ref).any(-1).float().mean().item():.2%}")
    assert safe.float().mean() > 0.5
    assert torch.equal(idx[safe], i_ref[safe]), "RVQ indices must be bit-exact on margin-safe frames"
    same = (idx == i_ref).all(-1)
    assert err(quant.reshape(-1, 512)[same.to(DEV)], q_ref[same]) < 1e-4


def test_c1_decoder_se_vs_oracle():
    from oracle import codec_se as ose
    from oracle.transformer import sub

    ss = _c1_se_model(23)
    st = {k: v.detach().clone() for k, v in ss.state_dict().items()}
    q = torch.randn(2, 150, 512, generator=torch.Generator().manual_seed(5)) * 0.5
    torch.set_num_threads(min(32, torch.get_num_threads()))
    ref = ose.decoder(sub(st, "decoder"), q.transpose(1, 2))
    ss = ss.to(DEV).eval()
    assert ss._tc_plan_dec() is not None
    with torch.no_grad():
        got = ss.decode(q.to(DEV))
    e, scale = err(got, ref), ref.abs().max().item()
    print(f"C1 SE decoder max abs err {e:.3e} (scale {scale:.3f})")
    assert got.shape == ref.shape == (2, 1, 48000) and e < 2e-4 * max(1.0, scale)


@pytest.mark.parametrize("dim_head", [32, 128])
def test_bottleneck_golden(dim_head):
    from audiolm_pytorch_b200 import SoundStream

    g = golden.load("codec_options.pt")["local_attn"][dim_head]
    ss = SoundStream(**g["kwargs"])
    ss.load_state_dict(g["state"], strict=True)
    ss = ss.to(DEV).eval()
    with torch.no_grad():
        out = ss.encoder_attn(g["h"].to(DEV))
        _, idx, _ = ss(g["wave"].to(DEV), return_encoded=True)
        recon = ss(g["wave"].to(DEV), return_recons_only=True)
        recon_idx = ss.decode_from_codebook_indices(idx)
    e = rms_rel(out, g["enc_attn_out"])
    print(f"dim_head {dim_head}: LocalTransformer rms-rel err vs reference {e:.2e}")
    assert e < 1e-2
    agree = (idx.cpu() == g["idx"]).float().mean().item()
    print("code agreement with the fp32 reference", agree)
    assert agree > 0.8
    assert rms_rel(recon, g["recon"]) < 0.15
    assert torch.allclose(recon_idx, recon, atol=1e-4)


@pytest.mark.parametrize("dim_head,heads", [(32, 16), (128, 4)])
def test_bottleneck_c1_size_vs_oracle(dim_head, heads):
    """dim 512, window 128, 150 frames, the checks of test_local_transformer_c1_size_vs_oracle at other head widths"""
    from audiolm_pytorch_b200.local_attn import LocalTransformer
    from oracle import third_party as tp

    torch.manual_seed(5 + dim_head)
    lt = LocalTransformer(dim=512, depth=1, heads=heads, window_size=128, dim_head=dim_head, prenorm=True, causal=True)
    with torch.no_grad():
        for p_ in lt.parameters():
            if p_.ndim == 1:
                p_.add_(torch.randn_like(p_) * 0.1)
    attn, ff = lt.layers[0]
    o_attn = tp.LocalMHA(dim=512, heads=heads, qk_rmsnorm=True, window_size=128, use_rotary_pos_emb=True,
                         gate_values_per_head=True, use_xpos=True, dim_head=dim_head, prenorm=True, causal=True).eval()
    o_ff = tp.LocalFeedForward(512).eval()
    o_attn.load_state_dict(attn.state_dict(), strict=True)
    o_ff.load_state_dict(ff.state_dict(), strict=True)
    x = torch.randn(3, 150, 512)
    with torch.no_grad():
        ref = o_attn(x) + x
        ref = o_ff(ref) + ref
        got = lt.to(DEV)(x.to(DEV))
    e = rms_rel(got - x.to(DEV), ref - x)
    print(f"dim_head {dim_head}: C1-size LocalTransformer delta rms-rel err {e:.2e}")
    assert e < 2e-2
    x2 = x.clone()
    x2[:, 140:] += 1.0
    x3 = x.clone()
    x3[:, 0] += 1.0
    with torch.no_grad():
        got2, got3 = lt(x2.to(DEV)), lt(x3.to(DEV))
    assert torch.equal(got2[:, :140], got[:, :140])
    assert torch.equal(got3[:, 129:], got[:, 129:]) and not torch.equal(got3[:, :129], got[:, :129])
