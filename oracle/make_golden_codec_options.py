"""Generate tests/golden/codec_options.pt from the REAL reference (oracle/ref_import.py) - build container only.

    python -m oracle.make_golden_codec_options

Two SoundStream constructor options the other fixtures do not cover (oracle/make_golden.py is not touched):
- `squeeze_excite=True` (soundstream.py:145-169, 362-369) on a small seeded model (channels 4, no local attention):
  the state_dict, the reference's encoder / decoder / rq key list with shapes, a wave, the encoder output, quantized
  frames, code indices and the reconstruction.  The run asserts that oracle/codec_se.py reproduces the reference to fp32
  round-off and the code indices exactly.
- the local-attention bottleneck at `attn_dim_head` 32 and 128 (window 8, 30 frames -> 4 buckets, the last ragged; two
  heads; narrow conv stacks, channel_mults (1, 2, 2, 4), to keep the file small): the state_dict, a bottleneck input and the reference's output, and the codes and reconstruction of a wave.
"""
from __future__ import annotations

import random
import sys
import warnings

import torch

from . import codec_se as ose
from . import golden, ref_import
from . import third_party as tp
from .make_golden import check, clone_state
from .transformer import sub

NAME = "codec_options.pt"
ATTN_WIDTHS = (32, 128)
PARTS = ("encoder", "decoder", "rq")


def squeeze_excite_model(ref):
    torch.manual_seed(71)
    kw = dict(codebook_size=64, rq_num_quantizers=4, channels=4, use_local_attn=False, codebook_dim=32,
              target_sample_hz=24000, squeeze_excite=True)
    ss = ref.ss.SoundStream(**kw).eval()
    tp.seed_codebooks(ss.rq, seed=7, std=0.5)
    g = torch.Generator().manual_seed(72)
    with torch.no_grad():   # move the SE convs off their init so the gates spread around 0.5
        for n_, p_ in ss.named_parameters():
            if ".fn.4." in n_:
                p_.add_(torch.randn(p_.shape, generator=g) * 0.2)
    wave = torch.randn(2, 3200)
    with torch.no_grad():
        enc = ss.encoder(wave[:, None, :])
        quant, idx, _ = ss(wave, return_encoded=True)
        recon = ss(wave, return_recons_only=True)
        recon_idx = ss.decode_from_codebook_indices(idx)
    st = {k: v for k, v in clone_state(ss).items() if k.split(".")[0] in PARTS}
    keys = [(k, tuple(v.shape)) for k, v in ss.state_dict().items() if k.split(".")[0] in PARTS]
    assert any(".fn.4.net.0.weight" in k for k, _ in keys) and any(k.startswith("decoder.") and ".fn.4." in k
                                                                   for k, _ in keys)
    print("squeeze_excite:")
    check("encoder", ose.encoder(sub(st, "encoder"), wave[:, None, :]), enc)
    oq, oi = ose.soundstream_tokenize(st, wave)
    assert torch.equal(oi, idx), "rvq indices differ"
    print("  [ok] rvq indices bit-exact")
    check("quantized", oq, quant)
    check("decode from indices", ose.soundstream_decode_indices(st, idx), recon_idx)
    check("round trip (README.md:100-113)", recon_idx, recon, tol=1e-5)
    return dict(kwargs=kw, state=st, keys=keys, wave=wave, enc=enc, quant=quant, idx=idx, recon=recon)


def local_attn_model(ref, dim_head):
    torch.manual_seed(81 + dim_head)
    kw = dict(codebook_size=64, rq_num_quantizers=4, channels=4, channel_mults=(1, 2, 2, 4), codebook_dim=32,
              attn_window_size=8, attn_dim_head=dim_head, attn_heads=2, target_sample_hz=24000)
    ss = ref.ss.SoundStream(**kw).eval()
    tp.seed_codebooks(ss.rq, seed=7, std=0.5)
    g = torch.Generator().manual_seed(82 + dim_head)
    with torch.no_grad():
        for n_, p_ in ss.named_parameters():   # move the attention block off its init (gates, scales, norms)
            if "_attn." in n_ and p_.ndim == 1:
                p_.add_(torch.randn(p_.shape, generator=g) * 0.1)
    wave = torch.randn(2, 9600)
    h = torch.randn(2, 30, 32)
    with torch.no_grad():
        enc_attn_out = ss.encoder_attn(h)
        quant, idx, _ = ss(wave, return_encoded=True)
        recon = ss(wave, return_recons_only=True)
        recon_idx = ss.decode_from_codebook_indices(idx)
    st = {k: v for k, v in clone_state(ss).items() if k.split(".")[0] in (*PARTS, "encoder_attn", "decoder_attn")}
    assert st["encoder_attn.layers.0.0.q_scale"].shape == (dim_head,)
    print(f"local attention bottleneck, dim_head {dim_head}:")
    check("round trip with decoder_attn (README.md:100-113)", recon_idx, recon, tol=1e-5)
    return dict(kwargs=kw, state=st, wave=wave, h=h, enc_attn_out=enc_attn_out, quant=quant, idx=idx, recon=recon)


def main():
    ref = ref_import.load()
    random.seed(20240607)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        out = dict(squeeze_excite=squeeze_excite_model(ref),
                   local_attn={dh: local_attn_model(ref, dh) for dh in ATTN_WIDTHS})
    golden.save(out, NAME)
    size = sum(p.stat().st_size for p in golden.GOLDEN.glob(NAME + "*"))
    print(f"wrote {NAME}: {size / 1e6:.2f} MB")


if __name__ == "__main__":
    sys.exit(main())
