"""H100: SoundStream(use_gate_loop_layers=True) on the gate-loop kernels (csrc/codec_gate_loop.cu) against an fp64
restatement (oracle/codec_gate_loop.py) and the reference's golden (tests/golden/gate_loop.pt)."""

import math

import pytest
import torch

from oracle import golden

pytestmark = pytest.mark.gpu
DEV = "cuda"
f64 = torch.float64

# Error model of one layer, propagated through the scan by error_bound():
# - split-bf16 projection (alm_codec_conv_tc): x and W' are carried as hi + lo bf16 pairs (16 significant bits each,
#   2^-17 relative) and the lo * lo product is dropped (2^-16): 2^-15 of sum |W'| |u| covers the three; its fp32
#   accumulation over C terms adds C * 2^-24 of the same sum;
# - the kernel's MUFU rsqrt / reciprocal and fp32 rounding: 2^-21 relative per quantity (<= 2 ulp, 4x margin);
# - sigmoid(a) = 1 / (1 + __expf(-a)): __expf is good to 2 + floor(1.16 |a|) ulp, so sigmoid carries up to
#   (3 + 1.16 |a|) 2^-23 relative (exp, reciprocal and the sum, 2x margin), which grows with |a|;
# - the C8S output: hi + lo carries y to 2^-16 relative.
# The expected value folds sqrt(C) * gamma into W here in fp64, independently of ops.gate_loop_fold_weight.
EPS_SPLIT = 2.0 ** -15
EPS_F32 = 2.0 ** -21
EPS_OUT = 2.0 ** -16


def _layer_state(C, seed, gate_scale=2.0):
    g = torch.Generator().manual_seed(seed)
    w = torch.randn(3 * C, C, generator=g) / math.sqrt(C)
    w[2 * C:] *= gate_scale
    return {"norm.gamma": 1 + 0.3 * torch.randn(C, generator=g), "to_qkva.0.weight": w}


def error_bound(u, st, tc):
    """per-element bound on |y - y_exact| for x = u [B, C, T] (fp64 on the device), from the model above"""
    from oracle.codec_gate_loop import linear_scan

    C = u.shape[1]
    wf = st["to_qkva.0.weight"].to(f64) * st["norm.gamma"].to(f64)[None, :] * math.sqrt(C)
    r = 1 / u.norm(dim=1, keepdim=True).clamp_min(1e-12)
    P = torch.einsum("oc,bct->bot", wf, u) * r
    Pabs = torch.einsum("oc,bct->bot", wf.abs(), u.abs()) * r
    e = ((EPS_SPLIT if tc else 0.0) + C * 2.0 ** -24) * Pabs + EPS_F32 * P.abs()
    q, kv, a = P.split(C, dim=1)
    eq, ekv, ea = e.split(C, dim=1)
    gate = torch.sigmoid(a)
    eg = gate * (1 - gate) * ea + (3 + 1.16 * a.abs()) * 2.0 ** -23 * gate
    h = linear_scan(gate, kv)
    h_prev = torch.cat((torch.zeros_like(h[..., :1]), h[..., :-1]), dim=-1)
    eh = linear_scan(gate, eg * h_prev.abs() + ekv + EPS_F32 * ((gate * h_prev).abs() + kv.abs()))
    y = 2 * u + q * h
    return y, q.abs() * eh + h.abs() * eq + EPS_F32 * (q * h).abs() + (EPS_OUT if tc else EPS_F32) * y.abs()


def _run_tc(x, st):
    from audiolm_pytorch_b200 import ops

    dv = {k: v.to(DEV) for k, v in st.items()}
    units = ops.pack_gate_loop_weights(ops.gate_loop_fold_weight(dv["to_qkva.0.weight"], dv["norm.gamma"]))
    xp = ops.c8s_pack(x)
    return ops.c8s_unpack(ops.codec_gate_loop_tc(xp, units)), ops.c8s_unpack(xp)


def _check(got, u, st, tc, label):
    y, bound = error_bound(u.to(f64), {k: v.to(DEV) for k, v in st.items()}, tc)
    e = (got.to(f64) - y).abs()
    ratio = (e / bound).max().item()
    print(f"{label}: max abs err {e.max().item():.2e}, max err / bound {ratio:.3f}")
    assert ratio <= 1.0, f"{label}: error exceeds the split-bf16 error model ({ratio:.2f}x)"


TC_SHAPES = ([(C, T, 1) for C in (32, 64, 128, 256, 512) for T in (1, 127, 128, 129, 5000, 48000)]
             + [(C, T, 3) for C in (32, 64, 128, 256, 512) for T in (1, 127, 129, 5000)]
             + [(32, 48000, 64), (64, 5000, 64), (256, 129, 64), (512, 127, 64), (128, 1, 64)])


@pytest.mark.parametrize("C,T,B", TC_SHAPES)
def test_gate_loop_tc_vs_fp64(C, T, B):
    st = _layer_state(C, 100 + C)
    x = torch.randn(B, C, T, generator=torch.Generator().manual_seed(T + B), device="cpu").to(DEV)
    got, u = _run_tc(x, st)
    _check(got, u, st, True, f"tc C={C} T={T} B={B}")


@pytest.mark.parametrize("C", [4, 8, 24, 64])
@pytest.mark.parametrize("T", [1, 129, 5000])
def test_gate_loop_fp32_vs_fp64(C, T):
    from audiolm_pytorch_b200 import ops

    st = _layer_state(C, 200 + C)
    x = torch.randn(2, C, T, generator=torch.Generator().manual_seed(C + T)).to(DEV)
    wf = ops.gate_loop_fold_weight(st["to_qkva.0.weight"].to(DEV), st["norm.gamma"].to(DEV))
    got = ops.codec_gate_loop_fp32(x, wf)
    _check(got, x, st, False, f"fp32 C={C} T={T}")


@pytest.mark.parametrize("C,T", [(32, 48000), (64, 24000), (512, 3000)])
def test_gate_loop_long_memory(C, T):
    """a constant channel drives every gate to sigmoid(a) >= 0.99 for the whole sequence, so h carries thousands of
    steps across many time tiles: a wrong or missing carry between tiles moves y far outside the bound"""
    from audiolm_pytorch_b200 import ops
    from oracle.codec_gate_loop import linear_scan

    gen = torch.Generator().manual_seed(C)
    st = _layer_state(C, 300 + C, gate_scale=0.0)
    st["norm.gamma"] = torch.ones(C)
    st["to_qkva.0.weight"][2 * C:, 0] = 5.5 / math.sqrt(C)   # a_c = 5.5 x_0 / ||x|| ~ 5.4: sigmoid(a) ~ 0.995
    x = 0.1 * torch.randn(2, C, T, generator=gen)
    x[:, 0] = 3.0 * math.sqrt(C) / 6
    x = x.to(DEV)
    got, u = _run_tc(x, st)
    wf = ops.gate_loop_fold_weight(st["to_qkva.0.weight"], st["norm.gamma"]).to(DEV, f64)
    a = torch.einsum("oc,bct->bot", wf[2 * C:], u.to(f64)) / u.to(f64).norm(dim=1, keepdim=True)
    assert torch.sigmoid(a).min() >= 0.99
    _check(got, u, st, True, f"long memory C={C} T={T}")
    # the same layer with the state reset at every 128-step boundary is far off: the carry is what the test sees
    y, bound = error_bound(u.to(f64), {k: v.to(DEV) for k, v in st.items()}, True)
    q, kv, a = (torch.einsum("oc,bct->bot", wf, u.to(f64)) / u.to(f64).norm(dim=1, keepdim=True)).split(C, dim=1)
    Tc = T // 128 * 128
    h_cut = linear_scan(torch.sigmoid(a[..., :Tc]).reshape(2, C, -1, 128), kv[..., :Tc].reshape(2, C, -1, 128))
    y_cut = 2 * u.to(f64)[..., :Tc] + q[..., :Tc] * h_cut.reshape(2, C, Tc)
    assert ((y_cut - y[..., :Tc]).abs() > 100 * bound[..., :Tc]).float().mean() > 0.25


def test_gate_loop_deterministic():
    from audiolm_pytorch_b200 import ops

    st = _layer_state(64, 7)
    x1 = torch.randn(3, 64, 24000, generator=torch.Generator().manual_seed(1)).to(DEV)
    x2 = torch.randn(5, 64, 3001, generator=torch.Generator().manual_seed(2)).to(DEV)
    a1, _ = _run_tc(x1, st)
    a2, _ = _run_tc(x2, st)
    b1, _ = _run_tc(x1, st)
    b2, _ = _run_tc(x2, st)
    assert torch.equal(a1, b1) and torch.equal(a2, b2)
    wf = ops.gate_loop_fold_weight(st["to_qkva.0.weight"], st["norm.gamma"]).to(DEV)
    f1, f2 = ops.codec_gate_loop_fp32(x1, wf), ops.codec_gate_loop_fp32(x2, wf)
    assert torch.equal(f1, ops.codec_gate_loop_fp32(x1, wf)) and torch.equal(f2, ops.codec_gate_loop_fp32(x2, wf))


def test_gate_loop_golden_end_to_end():
    from audiolm_pytorch_b200 import SoundStream

    g = golden.load("gate_loop.pt")["small"]
    ss = SoundStream(**g["kwargs"])
    ss.load_state_dict(g["state"], strict=True)
    ss = ss.to(DEV).eval()
    wave = g["wave"].to(DEV)
    with torch.no_grad():
        enc = ss.encoder(wave[:, None, :])
        quant, idx, _ = ss(wave, return_encoded=True)
        codes = ss.tokenize(wave)
        recon = ss(wave, return_recons_only=True)
        recon_idx = ss.decode_from_codebook_indices(idx)
    scale = g["enc"].abs().max().item()
    assert (enc.cpu() - g["enc"]).abs().max() < 1e-4 * scale
    assert torch.equal(idx.cpu(), g["idx"]), "RVQ indices must be bit-exact"
    assert torch.equal(codes[0].cpu(), g["idx"])
    assert (quant.cpu() - g["quant"]).abs().max() < 1e-5
    rscale = g["recon"].abs().max().item()
    assert (recon.cpu() - g["recon"]).abs().max() < 1e-4 * rscale
    assert (recon_idx.cpu() - g["recon_idx"]).abs().max() < 1e-4 * rscale


def _c1_model(seed):
    from audiolm_pytorch_b200.soundstream import SoundStream

    torch.manual_seed(seed)
    ss = SoundStream(codebook_size=1024, rq_num_quantizers=8, target_sample_hz=24000, use_local_attn=False,
                     use_gate_loop_layers=True)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for n_, p_ in ss.named_parameters():
            if n_.endswith("fn.fn.norm.gamma"):
                p_.copy_(1 + 0.3 * torch.randn(p_.shape, generator=g))
            elif n_.endswith("fn.fn.to_qkva.0.weight"):
                C = p_.shape[1]
                p_.copy_(torch.randn(p_.shape, generator=g) / math.sqrt(C))
                p_[2 * C:] *= 2.0
    return ss


# the whole C1 stack (29 layers on each side) against the fp32 CPU oracle: the per-layer split-bf16 error (~1e-5
# relative, test_residual_unit_tc_vs_oracle) compounded over the layers, with the gate loops' doubling skip
C1_REL = 1e-3


def test_c1_encoder_and_rvq_indices_vs_oracle():
    """C1 encoder with gate loops (32 channels, strides 2/4/5/8, 48 000 samples -> 150 frames) on the tensor-core plan +
    8-stage RVQ: indices bit-exact on every margin-safe frame, the rule of test_c1_encoder_and_rvq_indices_vs_oracle"""
    from audiolm_pytorch_b200 import soundstream as ss_mod
    from oracle import codec as oc
    from oracle import codec_gate_loop as ogl
    from oracle.transformer import sub

    ss = _c1_model(32)
    g = torch.Generator().manual_seed(7)
    wave = torch.randn(2, 48000, generator=g)
    torch.set_num_threads(min(32, torch.get_num_threads()))
    enc_ref = ogl.encoder(sub({k: v.detach() for k, v in ss.state_dict().items()}, "encoder"),
                          wave[:, None, :]).transpose(1, 2)
    # codes at the scale of the encoder output (the gate loops' doubling skips make it larger than without them), so
    # the nearest-code decisions have margins the fp32-level encoder error cannot cross
    std = enc_ref.std().item()
    for layer in ss.rq.rvqs[0].layers:
        layer._codebook.embed.copy_(torch.randn(1, 1024, 512, generator=g) * std)
        layer._codebook.initted.fill_(True)
    st = {k: v.detach().clone() for k, v in ss.state_dict().items()}
    cbs = oc.codebooks_of(st)
    flat = enc_ref.reshape(-1, 512)
    q_ref, i_ref = oc.rvq_encode(flat, cbs)
    margin = oc.rvq_margin(flat, cbs)
    ss = ss.to(DEV).eval()
    assert ss._tc_plan() is not None
    with torch.no_grad():
        enc = ss.encode_frames(wave.to(DEV)[:, None, :])
        quant, idx, _ = ss(wave.to(DEV), return_encoded=True)
    e = (enc.cpu() - enc_ref).abs().max().item()
    scale = enc_ref.abs().max().item()
    print(f"C1 gate-loop encoder max abs err {e:.3e} (scale {scale:.2f})")
    assert e < C1_REL * max(1.0, scale)
    idx = idx.reshape(-1, 8).cpu()
    safe = margin > max(20 * e, 1e-4)
    print(f"margin-safe frames {safe.float().mean().item():.2%}, frames with any differing index "
          f"{(idx != i_ref).any(-1).float().mean().item():.2%}")
    assert safe.float().mean() > 0.5
    assert torch.equal(idx[safe], i_ref[safe]), "RVQ indices must be bit-exact on margin-safe frames"
    # the CUDA-core path of the same model agrees with the tensor-core one
    old = ss_mod.ENCODER_ON_TENSOR_CORES
    try:
        ss_mod.ENCODER_ON_TENSOR_CORES = False
        assert ss._tc_plan() is None
        with torch.no_grad():
            enc_fp32 = ss.encode_frames(wave.to(DEV)[:, None, :])
    finally:
        ss_mod.ENCODER_ON_TENSOR_CORES = old
    e2 = (enc_fp32 - enc).abs().max().item()
    print(f"C1 gate-loop encoder, tensor cores vs CUDA cores: max abs diff {e2:.3e}")
    assert e2 < C1_REL * max(1.0, scale)


def test_c1_decoder_vs_oracle():
    from audiolm_pytorch_b200 import soundstream as ss_mod
    from oracle import codec_gate_loop as ogl
    from oracle.transformer import sub

    ss = _c1_model(33)
    st = {k: v.detach().clone() for k, v in ss.state_dict().items()}
    q = torch.randn(2, 150, 512, generator=torch.Generator().manual_seed(5)) * 0.5
    torch.set_num_threads(min(32, torch.get_num_threads()))
    ref = ogl.decoder(sub(st, "decoder"), q.transpose(1, 2))
    ss = ss.to(DEV).eval()
    assert ss._tc_plan_dec() is not None
    with torch.no_grad():
        got = ss.decode(q.to(DEV))
    e, scale = (got.cpu() - ref).abs().max().item(), ref.abs().max().item()
    print(f"C1 gate-loop decoder max abs err {e:.3e} (scale {scale:.3f})")
    assert got.shape == ref.shape == (2, 1, 48000) and e < C1_REL * max(1.0, scale)
    old = ss_mod.ENCODER_ON_TENSOR_CORES
    try:
        ss_mod.ENCODER_ON_TENSOR_CORES = False
        with torch.no_grad():
            got_fp32 = ss.decode(q.to(DEV))
    finally:
        ss_mod.ENCODER_ON_TENSOR_CORES = old
    assert (got_fp32 - got).abs().max().item() < C1_REL * max(1.0, scale)
