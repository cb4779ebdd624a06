"""ops.resample on the GPU (csrc/resample.cu).

* against the fp64 oracle (oracle/resample.py) across the envelope: the rate pairs the callers meet, large ratios and
  coprime rates whose table does not fit in shared memory, lengths 1, o - 1, o, o + 1 and 1 s + 17, 1 / 3 / 64 rows,
  windows from the left and from the right, on a 1e-3 sine plus unit noise;
* against torchaudio.functional.resample on the same CUDA tensor;
* bitwise determinism and batch invariance, strided and batched inputs;
* every consumer with input_sample_hz equal to the same consumer fed ops.resample's output, and AudioLM with a 44.1 kHz
  prime wave, all with torchaudio unimportable.

Error model (fp32, u = 2^-24): output j of phase p sums T_p products of a fp32-rounded tap and a fp32 sample with fp32
FMAs, so |y - y64| <= (T_p + 1) u sum_m |K[p, m] x[m]| plus the tap rounding u sum |K x|.  The bound checked is
2 (T_p + 2) u sum |K x| per element.
"""
import sys

import pytest
import torch

from audiolm_pytorch_b200 import ops
from oracle import golden
from oracle import resample as orr

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24

PAIRS = [(44100, 16000), (44100, 24000), (22050, 16000), (48000, 16000), (48000, 24000), (24000, 16000),
         (16000, 24000)]
ENVELOPE = PAIRS + [(96000, 8000), (8000, 96000), (44100, 16001)]


def _lengths(orig, new):
    o, n = ops.resample_rates(orig, new)
    return sorted({L for L in (1, o - 1, o, o + 1, orig + 17) if L >= 1})


def _signal(rows, L, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    t = torch.arange(L, device=DEV, dtype=torch.float64)
    return (1e-3 * torch.sin(0.05 * t) + torch.randn(rows, L, device=DEV, generator=g, dtype=torch.float64)).float()


def _check(y, x, orig, new, start, count):
    o, n = ops.resample_rates(orig, new)
    ref, mag = orr.resample(x, orig, new, with_magnitude=True)
    ref, mag = ref[..., start:start + count], mag[..., start:start + count]
    counts = ops.resample_table(o, n)[2].to(DEV)
    T_p = counts[(torch.arange(start, start + count, device=DEV) % n)].double()
    bound = 2 * (T_p + 2) * U * mag
    err = (y.double() - ref).abs()
    assert y.dtype == torch.float32 and y.shape == ref.shape
    assert bool((err <= bound).all()), f"worst err / bound {(err / bound.clamp_min(1e-300)).max().item():.3g}"


@pytest.mark.parametrize("rows", [1, 3, 64])
@pytest.mark.parametrize("orig, new", ENVELOPE)
def test_against_fp64(orig, new, rows):
    for i, L in enumerate(_lengths(orig, new)):
        x = _signal(rows, L, seed=orig + new + rows + i)
        total = ops.resample_length(L, orig, new)
        y = ops.resample(x, orig, new)
        assert y.shape == (rows, total)
        _check(y, x, orig, new, 0, total)
        for start, count in ((0, total // 2), (total - total // 3, total // 3), (total // 5, total // 2)):
            w = ops.resample(x, orig, new, start=start, count=count)
            _check(w, x, orig, new, start, count)
            assert torch.equal(w, y[:, start:start + count])


@pytest.mark.parametrize("orig, new", PAIRS)
def test_against_torchaudio(orig, new):
    """within 1e-5 max|x| of torchaudio, beyond torchaudio's own distance from the exact result: on fp32 input
    torchaudio forms the filter positions base (m - width) / o in fp32, an absolute error up to base 2^-24 in t, which
    moves its taps by up to 1.6e-5 max|x| at 22050 -> 16000 (measured on the CPU against the fp64 oracle).  TF32 is
    off for its convolution so that it computes in fp32."""
    from torchaudio.functional import resample

    for i, L in enumerate(_lengths(orig, new) + [10 * orig + 3]):
        x = _signal(3, L, seed=7 * i + orig)
        with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
            ref = resample(x, orig, new)
        y = ops.resample(x, orig, new)
        assert y.shape == ref.shape
        own = (ref.double() - orr.resample(x, orig, new)).abs()
        assert bool(((y - ref).abs() <= 1e-5 * x.abs().max() + own).all())


def test_deterministic_and_batch_invariant():
    x = _signal(5, 44100 * 3 + 11, seed=1)
    a, b = ops.resample(x, 44100, 16000), ops.resample(x, 44100, 16000)
    assert torch.equal(a, b)
    assert torch.equal(ops.resample(x[2:3].clone(), 44100, 16000)[0], a[2])
    # strided rows, a non-unit sample stride, extra leading dims and other dtypes
    wide = _signal(5, 44100 * 3 + 40, seed=1)
    wide[:, :44100 * 3 + 11] = x
    assert torch.equal(ops.resample(wide[:, :44100 * 3 + 11], 44100, 16000), a)
    inter = torch.stack((x, -x), dim=-1)[..., 0]
    assert inter.stride(-1) == 2 and torch.equal(ops.resample(inter, 44100, 16000), a)
    assert torch.equal(ops.resample(x.view(5, 1, -1).expand(5, 2, -1), 44100, 16000)[:, 1], a)
    assert torch.equal(ops.resample(x.double(), 44100, 16000), a)
    h = x.half()
    assert torch.equal(ops.resample(h, 44100, 16000), ops.resample(h.float(), 44100, 16000))


def test_empty():
    x = torch.zeros(3, 0, device=DEV)
    assert ops.resample(x, 44100, 16000).shape == (3, 0)
    assert ops.resample(torch.zeros(0, 100, device=DEV), 44100, 16000).shape == (0, 37)


# ---- consumers ---------------------------------------------------------------------------------------------------------
@pytest.fixture
def no_torchaudio(monkeypatch):
    monkeypatch.setitem(sys.modules, "torchaudio", None)
    monkeypatch.setitem(sys.modules, "torchaudio.functional", None)


def _soundstream(num_quantizers=4):
    from audiolm_pytorch_b200 import SoundStream

    torch.manual_seed(3)
    codec = SoundStream(codebook_size=64, rq_num_quantizers=num_quantizers, channels=32, codebook_dim=64,
                        use_local_attn=False)
    gen = torch.Generator().manual_seed(4)
    for layer in codec.rq.rvqs[0].layers:
        layer._codebook.embed.copy_(torch.randn(layer._codebook.embed.shape, generator=gen) * 0.05)
        layer._codebook.initted.fill_(True)
    return codec.to(DEV).eval()


def test_soundstream(no_torchaudio):
    ss = _soundstream()
    wave = _signal(2, 44100 + 1234, seed=5)
    w16 = ops.resample(wave, 44100, 16000)
    with torch.no_grad():
        assert torch.equal(ss(wave, input_sample_hz=44100, return_codes_only=True), ss(w16, return_codes_only=True))
        for left in (False, True):
            got = ss(wave, input_sample_hz=44100, return_recons_only=True, curtail_from_left=left)
            assert torch.equal(got, ss(w16, return_recons_only=True, curtail_from_left=left))
        lead = ss(wave.view(1, 2, -1), input_sample_hz=44100, return_recons_only=True)
        assert torch.equal(lead[0], ss(w16, return_recons_only=True))


def test_encodec(no_torchaudio, tmp_path):
    from audiolm_pytorch_b200 import EncodecWrapper
    from oracle import encodec as oe

    torch.save(oe.random_state(5, noise_clips=1, noise_samples=24000), tmp_path / "encodec_24khz.th")
    w = EncodecWrapper(bandwidth=6.0, checkpoint_path=tmp_path / "encodec_24khz.th").to(DEV)
    wave = _signal(2, 44100 // 2 + 321, seed=6)
    emb, codes, _ = w(wave, input_sample_hz=44100, return_encoded=True)
    emb2, codes2, _ = w(ops.resample(wave, 44100, 24000), return_encoded=True)
    assert torch.equal(codes, codes2) and torch.equal(emb, emb2)


@pytest.fixture(scope="module")
def hubert(tmp_path_factory):
    from audiolm_pytorch_b200.hubert import HubertWithKmeans
    from oracle import hubert as oh

    d = tmp_path_factory.mktemp("hubert")
    gd = golden.load("hubert.pt")
    oh.write_checkpoint(d / "ck.pt", gd["state"], gd["arch"])
    oh.write_kmeans(d / "km.bin", gd["centers"])
    return HubertWithKmeans(d / "ck.pt", d / "km.bin", output_layer=gd["output_layer"]).to(DEV)


def test_hubert(no_torchaudio, hubert):
    wave = _signal(2, 44100 + 999, seed=7)
    for mult in (None, 320):
        hubert.seq_len_multiple_of = mult
        try:
            ids = hubert(wave, input_sample_hz=44100, flatten=False)
            assert torch.equal(ids, hubert(ops.resample(wave, 44100, 16000), flatten=False))
        finally:
            hubert.seq_len_multiple_of = None
    assert torch.equal(hubert(wave, input_sample_hz=16000), hubert(wave))


def test_vq_wav2vec(no_torchaudio, tmp_path):
    from audiolm_pytorch_b200.vq_wav2vec import FairseqVQWav2Vec
    from oracle import vq_wav2vec as ov

    m = golden.load("vq_wav2vec.pt")["A"]
    ov.write_checkpoint(tmp_path / "vq.pt", m["state"], m["arch"])
    q = FairseqVQWav2Vec(tmp_path / "vq.pt", seq_len_multiple_of=320).to(DEV)
    wave = _signal(2, 44100 + 555, seed=8)
    ids = q(wave, input_sample_hz=44100, flatten=False)
    assert torch.equal(ids, q(ops.resample(wave, 44100, 24000), flatten=False))


def test_audiolm_prime_wave_44k(no_torchaudio, hubert, monkeypatch):
    """AudioLM and the three wrappers' generate with a 44.1 kHz prime wave handed over on the CPU"""
    from audiolm_pytorch_b200 import AudioLM, CoarseTransformer, FineTransformer, SemanticTransformer

    kw = dict(dim=64, depth=2, heads=2, flash_attn=True)
    codec = _soundstream(4)
    torch.manual_seed(5)
    n = hubert.codebook_size
    sem = SemanticTransformer(num_semantic_tokens=n, **kw).to(DEV)
    coarse = CoarseTransformer(num_semantic_tokens=n, codebook_size=64, num_coarse_quantizers=2, **kw).to(DEV)
    fine = FineTransformer(num_coarse_quantizers=2, num_fine_quantizers=2, codebook_size=64, **kw).to(DEV)
    lm = AudioLM(wav2vec=hubert, codec=codec, semantic_transformer=sem, coarse_transformer=coarse,
                 fine_transformer=fine)
    real = lm.coarse.generate
    monkeypatch.setattr(lm.coarse, "generate", lambda **k: real(**{**k, "max_time_steps": 8}))
    prime = _signal(1, 44100, seed=9).cpu()
    n_sem = hubert(ops.resample(prime.to(DEV), 44100, 16000)).shape[1]
    wav = lm(prime_wave=prime, prime_wave_input_sample_hz=44100, max_length=n_sem + 4)
    wavs = [wav] if torch.is_tensor(wav) and wav.dim() == 1 else list(wav)
    assert len(wavs) == 1 and all(w_ is None or torch.isfinite(w_).all() for w_ in wavs)
    # the wrappers on their own, prime wave on the CPU
    sem_ids = lm.semantic.generate(prime_wave=prime, prime_wave_input_sample_hz=44100, max_length=n_sem + 2)
    coarse_ids = real(semantic_token_ids=sem_ids, prime_wave=prime, prime_wave_input_sample_hz=44100,
                      max_time_steps=8)
    out = lm.fine.generate(coarse_token_ids=coarse_ids, prime_wave=prime, prime_wave_input_sample_hz=44100)
    assert out.shape[0] == 1
