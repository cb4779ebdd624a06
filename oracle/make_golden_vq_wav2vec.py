"""Generate tests/golden/vq_wav2vec.pt - build container only.

    python -m oracle.make_golden_vq_wav2vec

1. Runs the REAL reference vq_wav2vec.py (oracle/ref_import.py) with fairseq's
   `checkpoint_utils.load_model_ensemble_and_task` bound to oracle/vq_wav2vec.py, on two small seeded models (width
   64, the published kernels and strides, num_vars 320, G = 2):
     A: gelu, no skip, no log compression, affine norms, combine_groups=True;
     B: relu, skip with residual_scale 0.5, log compression, non-affine norms, combine_groups=False.
2. Records, per model: the fairseq-layout state dict and cfg; waves of one frame (465 samples), odd lengths, a length
   where r_tsz // tsz differs from the stride at some layer, and 1 s at 24 kHz; the fp64 oracle's features and ze;
   the reference's ids with flatten=False and flatten=True; and the reference with input_sample_hz=16000 and
   seq_len_multiple_of=320 on one wave.
"""
from __future__ import annotations

import sys
import tempfile
from pathlib import Path
from types import SimpleNamespace

import torch

from . import golden, ref_import
from . import vq_wav2vec as ov

NAME = "vq_wav2vec.pt"
SMALL_LAYERS = ("[(64, 10, 5), (64, 8, 4), (64, 4, 2), (64, 4, 2), (64, 4, 2), (64, 1, 1), (64, 1, 1), "
                "(64, 1, 1)]")
MODELS = {
    "A": dict(ov.PUBLISHED, conv_feature_layers=SMALL_LAYERS, activation="gelu", skip_connections_feat=False,
              log_compression=False, non_affine_group_norm=False, combine_groups=True),
    "B": dict(ov.PUBLISHED, conv_feature_layers=SMALL_LAYERS, activation="relu", skip_connections_feat=True,
              residual_scale=0.5, log_compression=True, non_affine_group_norm=True, combine_groups=False),
}
# 465: one frame, where conv 4 sees r_tsz 4 and tsz 1 (step 4, stride 2); 545: conv 4 sees r_tsz 5, tsz 1 (step 5);
# 1000 and 3203: odd lengths; 24000: 1 s at 24 kHz
LENGTHS = (465, 545, 1000, 3203, 24000)
RESAMPLED_LENGTH = 16000 + 37


def strided_steps(arch, n):
    """(layer, r_tsz // tsz, stride) of every strided layer of the extractor on a clip of n samples"""
    out = []
    for i, (_, k, s) in enumerate(ov.conv_layers(arch)):
        m = (n - k) // s + 1
        out.append((i, n // m, s))
        n = m
    return out


class _OracleVectorQuantizer:
    """fairseq's KmeansVectorQuantizer (time_first=False) at inference, on the oracle's tensors"""

    def __init__(self, st):
        self.st = st
        self.embedding = st[ov.EMBEDDING]
        w = st[ov.PROJ + "0.weight"]
        self.groups = w.shape[0] // w.shape[1]

    def forward_idx(self, x):
        ze = ov.project(self.st, x.transpose(1, 2))  # x [B, C, T]
        bsz, tsz, G, vd = ze.shape
        e = ov.codewords(self.st, G)
        num_vars = e.shape[0]
        d = (ze.unsqueeze(0) - e.unsqueeze(1).unsqueeze(1)).view(num_vars, bsz, tsz, G, -1).norm(dim=-1, p=2)
        idx = d.argmin(dim=0)
        return ze, idx


class _OracleVQWav2Vec(torch.nn.Module):
    def __init__(self, st, arch):
        super().__init__()
        st = {k: v.double() for k, v in st.items()}
        self.feature_extractor = lambda wav: ov.features(st, arch, wav.double()).transpose(1, 2)
        self.vector_quantizer = _OracleVectorQuantizer(st)


def load_model_ensemble_and_task(inputs):
    (ckpt,) = inputs.values()
    return [_OracleVQWav2Vec(ckpt["model"], ckpt["cfg"]["model"])], ckpt["cfg"], None


def main():
    ref_import.load()
    sys.modules["fairseq"].checkpoint_utils = SimpleNamespace(load_model_ensemble_and_task=load_model_ensemble_and_task)
    import audiolm_pytorch.vq_wav2vec as rv  # noqa: E402  (the reference module, through ref_import's package)

    out = {}
    gen = torch.Generator().manual_seed(31)
    for seed, (name, arch) in enumerate(MODELS.items()):
        st = ov.random_state(arch, seed=40 + seed, groups=arch["vq_groups"], num_vars=arch["vq_vars"],
                             combine_groups=arch["combine_groups"], affine=not arch["non_affine_group_norm"])
        waves = [torch.randn(1 if n in (465, 545) else 2, n, generator=gen) for n in LENGTHS]
        st64 = {k: v.double() for k, v in st.items()}
        # codewords: ze vectors of the clips themselves, perturbed, so the search has realistic margins
        pool = torch.cat([ov.project(st64, ov.features(st64, arch, w.double())).flatten(0, 2) for w in waves])
        pick = pool[torch.randperm(pool.shape[0], generator=gen)[:arch["vq_vars"] * st[ov.EMBEDDING].shape[1]]]
        st[ov.EMBEDDING] = (pick.float() + 0.3 * torch.randn(pick.shape, generator=gen)).view(st[ov.EMBEDDING].shape)
        st64 = {k: v.double() for k, v in st.items()}
        feats = [ov.features(st64, arch, w.double()) for w in waves]
        zes = [ov.project(st64, f) for f in feats]
        with tempfile.TemporaryDirectory() as d:
            ck = Path(d) / "vq.pt"
            torch.save({"model": st, "cfg": {"model": dict(arch)}}, ck)
            ref = rv.FairseqVQWav2Vec(str(ck))
            assert (ref.groups, ref.codebook_size, ref.downsample_factor) == (2, 320, 80)
            ids = [ref(w, flatten=False) for w in waves]
            ids_flat = [ref(w) for w in waves]
            wave16 = torch.randn(2, RESAMPLED_LENGTH, generator=gen)
            ref.seq_len_multiple_of = 320
            ids_resampled = ref(wave16, flatten=False, input_sample_hz=16000)
        for w, ze, i, fl in zip(waves, zes, ids, ids_flat):
            e = ov.codewords(st64, 2)
            assert torch.equal(i, ov.ids(ze, e)), "reference ids differ from the fp64 oracle's"
            assert torch.equal(fl, i.reshape(i.shape[0], -1))
            print(f"  {name} wave {tuple(w.shape)}: ids {tuple(i.shape)}, smallest codeword gap "
                  f"{ov.margins(ze, e).min():.2e}")
        steps = [s for n in LENGTHS for s in strided_steps(arch, n) if s[1] != s[2]]
        assert steps, "no length where r_tsz // tsz differs from the stride"
        print(f"  {name}: layers where r_tsz // tsz != stride (layer, step, stride): {sorted(set(steps))}")
        out[name] = dict(arch=arch, state=st, waves=waves, features=[f.float() for f in feats],
                         ze=[z.float() for z in zes], ids=ids, ids_flat=ids_flat, wave16=wave16,
                         ids_resampled=ids_resampled, resample_kw=dict(input_sample_hz=16000, seq_len_multiple_of=320))
    print("  [ok] reference ids equal the fp64 oracle's")
    golden.save(out, NAME)
    size = sum(p.stat().st_size for p in golden.GOLDEN.glob(NAME + "*"))
    print(f"wrote {NAME}: {size / 1e6:.2f} MB")


if __name__ == "__main__":
    sys.exit(main())
