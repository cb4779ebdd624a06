"""Generate tests/golden/encodec.pt - build container only.

    python -m oracle.make_golden_encodec

1. Pins oracle/encodec.py against transformers' EncodecModel (its default config is the 24 kHz model) in fp64 with the
   keys mapped: encoder output, codes at 6 kbps and decoder output at several lengths, including T not a multiple of
   320 and T < 320.
2. Runs the REAL reference encodec.py (oracle/ref_import.py) with `encodec.EncodecModel.encodec_model_24khz()` bound to
   the seeded oracle model and encodec.utils._linear_overlap_add restated, at 1.5 and 6 kbps.
3. Writes: the seed and a checksum of the seeded state (the full-size weights, ~60 MB, are regenerated from the seed
   by tests), waves, the reference's codes and embeddings at both bandwidths, and its batch-1 decoded audio.
"""
from __future__ import annotations

import re
import sys

import torch
from torch import nn

from . import encodec as oe
from . import golden, ref_import

NAME = "encodec.pt"
SEED = 1234
PIN_LENGTHS = (1, 319, 321, 3200, 4817)
WAVE_LENGTHS = (6400, 4817)


def to_transformers(st):
    out = {}
    for k, v in st.items():
        k = k.replace("encoder.model.", "encoder.layers.").replace("decoder.model.", "decoder.layers.")
        k = k.replace("conv.conv.", "conv.").replace("convtr.convtr.", "conv.")
        k = k.replace("weight_g", "parametrizations.weight.original0").replace("weight_v",
                                                                               "parametrizations.weight.original1")
        k = re.sub(r"quantizer\.vq\.layers\.(\d+)\._codebook\.", r"quantizer.layers.\1.codebook.", k)
        out[k] = v.double()
    return out


def pin(st):
    from transformers import EncodecConfig, EncodecModel

    m = EncodecModel(EncodecConfig()).double().eval()
    m.load_state_dict(to_transformers(st), strict=True)
    gen = torch.Generator().manual_seed(7)
    worst = 0.0
    for T in PIN_LENGTHS:
        x = torch.randn(2, 1, T, generator=gen, dtype=torch.float64)
        with torch.no_grad():
            e_hf, e = m.encoder(x), oe.encoder(st, x)
            codes_hf = m.encode(x, bandwidth=6.0).audio_codes
            d_hf, d = m.decoder(e_hf), oe.decoder(st, e)
        codes, _, _ = oe.rvq_encode(e.permute(0, 2, 1).reshape(-1, oe.DIM), oe.codebooks(st, 8))
        assert e.shape == (2, oe.DIM, oe.n_frames(T)) and d.shape == (2, 1, oe.HOP * oe.n_frames(T))
        err = max(((e_hf - e).abs().max() / e.abs().max()).item(), ((d_hf - d).abs().max() / d.abs().max()).item())
        assert err < 1e-12, (T, err)
        assert torch.equal(codes_hf.reshape(-1, 2, 8, e.shape[-1])[0].permute(0, 2, 1).reshape(-1, 8), codes), T
        worst = max(worst, err)
    print(f"[golden] oracle vs transformers.EncodecModel (fp64): max relative error {worst:.1e}, codes equal")


class _OracleEncodec(nn.Module):
    """encodec.EncodecModel as the reference wrapper uses it, computed by oracle/encodec.py in fp64"""

    channels, sample_rate, segment_stride = 1, 24000, None

    def __init__(self, st):
        super().__init__()
        self.st, self.normalize, self.n_q = st, True, oe.N_CODEBOOKS
        outer = self

        class _Quantizer(nn.Module):
            def __init__(self):
                super().__init__()
                self.vq = nn.Module()
                self.vq.layers = nn.ModuleList()
                for q in range(oe.N_CODEBOOKS):
                    layer = nn.Module()
                    layer._codebook = nn.Module()
                    layer._codebook.register_buffer("embed", st[f"quantizer.vq.layers.{q}._codebook.embed"].clone())
                    self.vq.layers.append(layer)

            def decode(self, codes):  # [q, b, t] -> [b, 128, t]
                q, b, t = codes.shape
                emb = oe.rvq_decode(codes.permute(1, 2, 0).reshape(-1, q), oe.codebooks(outer.st, q))
                return emb.reshape(b, t, oe.DIM).permute(0, 2, 1)

        self.quantizer = _Quantizer()
        self.eval()

    @classmethod
    def encodec_model_24khz(cls):
        return cls(oe.random_state(SEED))

    def set_target_bandwidth(self, bandwidth):
        self.n_q = oe.BANDWIDTHS[bandwidth]

    def encode(self, wav):
        assert not self.normalize
        e = oe.encoder(self.st, wav)
        codes, _, _ = oe.rvq_encode(e.permute(0, 2, 1).reshape(-1, oe.DIM), oe.codebooks(self.st, self.n_q))
        return [(codes.reshape(wav.shape[0], -1, self.n_q).permute(0, 2, 1), None)]

    def decoder(self, emb):
        return oe.decoder(self.st, emb)


def linear_overlap_add(frames, stride):
    """encodec.utils._linear_overlap_add restated: iterates over `frames` (the reference passes a [B, 1, T] tensor, so
    over the batch) and blends them with a triangular window at offsets of `stride`"""
    dtype, shape = frames[0].dtype, frames[0].shape[:-1]
    total = stride * (len(frames) - 1) + frames[-1].shape[-1]
    flen = frames[0].shape[-1]
    t = torch.linspace(0, 1, flen + 2, dtype=dtype)[1:-1]
    weight = 0.5 - (t - 0.5).abs()
    out = torch.zeros(*shape, total, dtype=dtype)
    wsum = torch.zeros(total, dtype=dtype)
    offset = 0
    for frame in frames:
        n = frame.shape[-1]
        out[..., offset:offset + n] += weight[:n] * frame
        wsum[offset:offset + n] += weight[:n]
        offset += stride
    return out / wsum


def main():
    st = oe.random_state(SEED)
    if "--no-pin" not in sys.argv:
        pin(st)
    ref_import.load()
    import audiolm_pytorch.encodec as ref_encodec  # noqa: E402  (bound to the stubs when ref_import loaded it)

    ref_encodec.EncodecModel = _OracleEncodec
    ref_encodec._linear_overlap_add = linear_overlap_add
    gen = torch.Generator().manual_seed(11)
    waves = [0.3 * torch.randn(2, T, generator=gen) for T in WAVE_LENGTHS]
    out = dict(seed=SEED, checksum=oe.checksum(st), waves=waves, codes={}, emb={}, n_q={})
    for bw in (1.5, 6.0):
        wrapper = ref_encodec.EncodecWrapper(bandwidth=bw)
        out["n_q"][bw] = wrapper.num_quantizers
        out["codes"][bw], out["emb"][bw] = [], []
        for w in waves:
            emb, codes, _ = wrapper(w, return_encoded=True)
            out["codes"][bw].append(codes)
            out["emb"][bw].append(emb.float())
        if bw == 6.0:
            out["decoded_b1"] = wrapper.decode_from_codebook_indices(out["codes"][bw][0][:1]).float()
            both = wrapper.decode_from_codebook_indices(out["codes"][bw][0])
            out["decoded_batch_ref"] = both.float()  # the reference's blended batch decode, [1, 1, T + B - 1]
    golden.save(out, NAME)
    print(f"[golden] wrote {NAME}: codes {[tuple(c.shape) for c in out['codes'][6.0]]}, "
          f"decoded {tuple(out['decoded_b1'].shape)}, batch decode {tuple(out['decoded_batch_ref'].shape)}")


if __name__ == "__main__":
    main()
