"""H100: SoundStream's LocalTransformer bottleneck (soundstream.py:397-440) on the attention / GEMM kernels vs the
reference run over the restated `local-attention` package (tests/golden/local_attn.pt; PARITY UNPINNED upstream) and vs
the oracle restatement at the C1 size (dim 512, window 128, 150 frames)."""

import pytest
import torch

from oracle import golden

pytestmark = pytest.mark.gpu
DEV = "cuda"


def rms_rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).pow(2).mean().sqrt() / b.pow(2).mean().sqrt().clamp(min=1e-12)).item()


def test_local_transformer_golden_and_default_soundstream():
    from audiolm_pytorch_b200 import SoundStream

    g = golden.load("local_attn.pt")
    ss = SoundStream(**g["kwargs"])                       # default use_local_attn=True constructs
    ss.load_state_dict(g["state"], strict=True)
    ss = ss.to(DEV).eval()
    with torch.no_grad():
        out = ss.encoder_attn(g["h"].to(DEV))
        quant, idx, _ = ss(g["wave"].to(DEV), return_encoded=True)
        recon = ss(g["wave"].to(DEV), return_recons_only=True)
        recon_idx = ss.decode_from_codebook_indices(idx)
    e = rms_rel(out, g["enc_attn_out"])
    print("LocalTransformer rms-rel err vs reference", e)
    assert e < 1e-2                                        # bf16 attention / GEMMs vs the fp32 reference
    # codes downstream of a bf16 block: not bit-exact by construction; most frames must agree
    agree = (idx.cpu() == g["idx"]).float().mean().item()
    print("code agreement with the fp32 reference", agree)
    assert agree > 0.8
    assert rms_rel(recon, g["recon"]) < 0.15
    assert torch.allclose(recon_idx, recon, atol=1e-4)     # README round trip (decoder_attn on both paths)


def test_local_transformer_c1_size_vs_oracle():
    from audiolm_pytorch_b200.local_attn import LocalTransformer
    from oracle import third_party as tp

    torch.manual_seed(5)
    lt = LocalTransformer(dim=512, depth=1, heads=8, window_size=128, dim_head=64, prenorm=True, causal=True)
    with torch.no_grad():
        for p_ in lt.parameters():
            if p_.ndim == 1:
                p_.add_(torch.randn_like(p_) * 0.1)
    attn, ff = lt.layers[0]
    o_attn = tp.LocalMHA(dim=512, heads=8, qk_rmsnorm=True, window_size=128, use_rotary_pos_emb=True,
                         gate_values_per_head=True, use_xpos=True, dim_head=64, prenorm=True, causal=True).eval()
    o_ff = tp.LocalFeedForward(512).eval()
    o_attn.load_state_dict(attn.state_dict(), strict=True)
    o_ff.load_state_dict({k: v for k, v in ff.state_dict().items()}, strict=True)
    x = torch.randn(3, 150, 512)
    with torch.no_grad():
        ref = o_attn(x) + x
        ref = o_ff(ref) + ref
        got = lt.to(DEV)(x.to(DEV))
    e = rms_rel(got - x.to(DEV), ref - x)                  # error of what the block adds to the residual stream
    print("C1-size LocalTransformer delta rms-rel err", e)
    assert e < 2e-2
    # causality + locality: frames >= 140 changed -> outputs before 140 unchanged; frame 0 cannot influence frame 129+
    x2 = x.clone()
    x2[:, 140:] += 1.0
    x3 = x.clone()
    x3[:, 0] += 1.0
    with torch.no_grad():
        got2, got3 = lt(x2.to(DEV)), lt(x3.to(DEV))
    assert torch.equal(got2[:, :140], got[:, :140])
    assert torch.equal(got3[:, 129:], got[:, 129:]) and not torch.equal(got3[:, :129], got[:, :129])
