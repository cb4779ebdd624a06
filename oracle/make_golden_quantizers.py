"""Generate tests/golden/quantizers.pt from the REAL reference (oracle/ref_import.py) - build container only.

    python -m oracle.make_golden_quantizers

SoundStream's codebook-free quantizers (soundstream.py:555-609, 839-845, 691-699), with the reference's soundstream.py
running on the restatements in oracle/scalar_quant.py.  Four small seeded models (channels 4, no local attention,
codebook_dim 32 unless stated): residual FSQ with levels [8, 5, 5, 5] (projection 32 -> 4), FSQ with codebook_dim 8 in
two groups and levels [5, 5, 4, 4] (identity projections), LFQ with codebook_size 1024 (projection 32 -> 10) and LFQ
with two groups and codebook_size 2^16 (identity projections).  The
projections are moved off their init so the codes spread.  Per model: the encoder / decoder / rq state_dict and key
list with shapes, a wave, the encoder output, quantized frames, indices (with their dtype), the reconstruction, and
decode_from_codebook_indices on the full and on coarse-only ids.  The run asserts that the functional codec oracle
with the quantizer restatement reproduces the reference, the indices exactly.
"""
from __future__ import annotations

import random
import sys
import warnings

import torch

from . import golden, ref_import
from . import scalar_quant as osq
from .make_golden import check, clone_state

NAME = "quantizers.pt"
PARTS = ("encoder", "decoder", "rq")
BASE = dict(channels=4, use_local_attn=False, codebook_dim=32, target_sample_hz=24000, rq_num_quantizers=4)
MODELS = {
    "fsq": dict(use_finite_scalar_quantizer=True, finite_scalar_quantizer_levels=[8, 5, 5, 5]),
    "fsq_groups": dict(use_finite_scalar_quantizer=True, finite_scalar_quantizer_levels=[5, 5, 4, 4], codebook_dim=8,
                       rq_groups=2),
    "lfq": dict(use_lookup_free_quantizer=True, codebook_size=1024),
    "lfq_groups": dict(use_lookup_free_quantizer=True, codebook_size=2 ** 16, rq_groups=2),
}
COARSE = 2   # stages per group kept in the coarse-only decode


def model(ref, name, seed):
    torch.manual_seed(seed)
    kw = {**BASE, **MODELS[name]}
    ss = ref.ss.SoundStream(**kw).eval()
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():   # spread the projections so the first stages use most of the levels
        for n_, p_ in ss.named_parameters():
            if n_.startswith("rq.") and n_.endswith("project_in.weight"):
                p_.mul_(4.0).add_(torch.randn(p_.shape, generator=g) * 0.5)
    wave = torch.randn(2, 3200)
    with torch.no_grad():
        enc = ss.encoder(wave[:, None, :]).transpose(1, 2)
        idx_raw = ss(wave, return_codes_only=True)
        quant, idx, _ = ss(wave, return_encoded=True)
        recon = ss(wave, return_recons_only=True)
        recon_idx = ss.decode_from_codebook_indices(idx)
        coarse = idx_raw[..., :COARSE]
        recon_coarse = ss.decode_from_codebook_indices(coarse)
    st = {k: v for k, v in clone_state(ss).items() if k.split(".")[0] in PARTS}
    keys = [(k, tuple(v.shape)) for k, v in ss.state_dict().items() if k.split(".")[0] in PARTS]
    assert any(".project_in." in k for k, _ in keys) == (name in ("fsq", "lfq"))
    print(f"{name}: codebook_size {ss.codebook_size}, indices {tuple(idx_raw.shape)} {idx_raw.dtype}, "
          f"{idx_raw.unique().numel()} distinct")
    assert idx_raw.dtype == (torch.int32 if name.startswith("fsq") else torch.int64)
    oenc, oq, oi = osq.soundstream_tokenize(kw, st, wave)
    check("encoder", oenc, enc)
    assert torch.equal(oi, idx_raw), "indices differ"
    print("  [ok] indices bit-exact")
    check("quantized", oq, quant)
    check("decode from indices", osq.soundstream_decode_indices(kw, st, idx_raw), recon_idx)
    check("decode from coarse ids", osq.soundstream_decode_indices(kw, st, coarse), recon_coarse)
    check("round trip", recon_idx, recon, tol=1e-5)
    return dict(kwargs=kw, state=st, keys=keys, wave=wave, enc=enc, quant=quant, idx=idx_raw, idx_dtype=str(idx_raw.dtype),
                recon=recon, recon_idx=recon_idx, coarse_q=COARSE, recon_coarse=recon_coarse,
                codebook_size=ss.codebook_size)


def main():
    ref = ref_import.load()
    osq.register(ref)
    random.seed(20240611)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        out = {name: model(ref, name, 91 + 10 * i) for i, name in enumerate(MODELS)}
    golden.save(out, NAME)
    size = sum(p.stat().st_size for p in golden.GOLDEN.glob(NAME + "*"))
    print(f"wrote {NAME}: {size / 1e6:.2f} MB")


if __name__ == "__main__":
    sys.exit(main())
