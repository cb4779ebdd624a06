"""FairseqVQWav2Vec on the GPU (csrc/vq_wav2vec.cu + conv 0 of csrc/hubert.cu + the split-bf16 GEMM + the RVQ
codeword search).

* alm_w2v_group_stats and alm_w2v_norm_act against an fp64 restatement: G in {1, 2, 4}, C in {64, 512}, one frame to
  30 s of frames, B in {1, 3, 16}, every flag combination (activation, affine, skip, log compression), skip steps of
  1, the stride and one that is not the stride; each element held to a bound of the error model below;
* the published shape (eight 512-wide convs, G = 2, 320 codewords) with seeded weights, both flag settings, against
  the fp64 oracle (oracle/vq_wav2vec.py): features and ze within FEAT_TOL, and ids equal to the fp64 ids on every frame
  and group whose codeword margin exceeds 2 |d ze|;
* both golden models (the reference's own ids) end to end with both flatten layouts, and with input_sample_hz and
  seq_len_multiple_of; bitwise determinism and batch invariance;
* SemanticTransformerWrapper / CoarseTransformerWrapper losses with raw_wave= equal to those with the golden ids;
  AudioLM construction; CPU input.

Error model (fp32 arithmetic, unit roundoff u = 2^-24):
  group statistics: fp64 sums of (y - y_0) over fixed chunks, rounded once to fp32:
    |mean - mean64| <= STAT_U u (|mean| + std),  |rstd - rstd64| <= STAT_U u rstd            with STAT_U = 4
  norm / activation / skip / log output: NORM_U u (|gamma| (rstd (|y| + |mean|) + 1) + |beta| + |residual| + |out|),
    scaled by sqrt(residual_scale) after a skip, with NORM_U = 64 (the statistics' error, the affine, erf, the skip
    add and log1p, each a few ulps and each term at most 1-Lipschitz)
  split-bf16 GEMM products: 2^-15 |x| |w| per product, plus K u sum |x| |w| for fp32 accumulation; through eight
  normalised layers this gives the model-level FEAT_TOL below (about 1e-5 measured, see DESIGN).
"""
import itertools
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import golden
from oracle import vq_wav2vec as ov

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24
STAT_U = 4
NORM_U = 64
F64 = torch.float64


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _stats64(y, G):
    B, T, C = y.shape
    v = y.double().view(B, T, G, C // G).permute(0, 2, 1, 3).reshape(B, G, -1)
    mean = v.mean(-1)
    var = v.var(-1, unbiased=False)
    return mean, (var + 1e-5).rsqrt(), var.sqrt()


def _check_split(s, ref):
    C = ref.shape[-1]
    hi, lo, hi2 = s[..., :C].double(), s[..., C:2 * C].double(), s[..., 2 * C:].double()
    assert torch.equal(hi, hi2)
    assert torch.equal(hi, ref.to(torch.bfloat16).double())
    assert ((hi + lo - ref).abs() <= 2.0 ** -16 * ref.abs() + 1e-38).all()


# ---- kernels -----------------------------------------------------------------------------------------------------------
SHAPES = [(1, 1, 64, 1), (3, 97, 64, 2), (16, 3, 512, 4), (1, 1499, 512, 2), (3, 4799, 512, 1), (16, 149, 64, 4)]
LONG = [(1, 143999, 512, 1), (1, 1500 * 3, 512, 2)]  # layer 0 and the quantizer of a 30 s clip at 24 kHz


@pytest.mark.parametrize("B, T, C, G", SHAPES + LONG)
def test_group_stats(B, T, C, G):
    from audiolm_pytorch_b200 import ops

    g = _gen(B * T + C + G)
    y = torch.randn(B, T, C, device=DEV, generator=g) * 3 + 100 * torch.randn(C, device=DEV, generator=g).abs()
    stats = ops.w2v_group_stats(y, G)
    mean, rstd, std = _stats64(y, G)
    assert stats.shape == (B, G, 2)
    assert ((stats[..., 0].double() - mean).abs() <= STAT_U * U * (mean.abs() + std)).all()
    assert ((stats[..., 1].double() - rstd).abs() <= STAT_U * U * rstd).all()


FLAGS = list(itertools.product([None, "relu", "gelu"], [True, False], ["none", "1", "stride", "other"], [False, True]))


def _norm_act_case(B, T, C, G, act, affine, skip, log, seed):
    from audiolm_pytorch_b200 import ops

    g = _gen(seed)
    y = torch.randn(B, T, C, device=DEV, generator=g) * 2 + torch.randn(C, device=DEV, generator=g)
    gamma = 1 + 0.2 * torch.randn(C, device=DEV, generator=g) if affine else None
    beta = 0.2 * torch.randn(C, device=DEV, generator=g) if affine else None
    step = {"none": 1, "1": 1, "stride": 2, "other": 5}[skip]
    res = None
    if skip != "none":
        Tr = (T - 1) * step + 1 + (step - 1 if skip == "other" else 0)
        res = torch.randn(B, Tr, C, device=DEV, generator=g)
    scale = math.sqrt(0.5) if res is not None else 1.0
    stats = ops.w2v_group_stats(y, G)
    out, s = ops.w2v_norm_act(y, stats, gamma=gamma, beta=beta, act=act, residual=res, step=step,
                              residual_scale=scale, log_compress=log, want_out=True, want_split=True)
    mean, rstd, _ = _stats64(y, G)
    Cg = C // G
    m = mean.repeat_interleave(Cg, dim=1)[:, None, :]
    r = rstd.repeat_interleave(Cg, dim=1)[:, None, :]
    ga = gamma.double() if affine else torch.ones(C, device=DEV, dtype=F64)
    be = beta.double() if affine else torch.zeros(C, device=DEV, dtype=F64)
    ref = (y.double() - m) * r * ga + be
    ref = {None: lambda v: v, "relu": F.relu, "gelu": F.gelu}[act](ref)
    scale_in = ga.abs() * (r * (y.double().abs() + m.abs()) + 1) + be.abs()
    if res is not None:
        rs = res.double()[:, ::step][:, :T]
        ref = (ref + rs) * math.sqrt(0.5)
        scale_in = (scale_in + rs.abs()) * math.sqrt(0.5)
    if log:
        ref = torch.log1p(ref.abs())
    bound = NORM_U * U * (scale_in + ref.abs())
    err = (out.double() - ref).abs()
    assert (err <= bound).all(), f"max err/bound {(err / bound).max().item():.3g}"
    _check_split(s, out.double())


@pytest.mark.parametrize("B, T, C, G", SHAPES)
@pytest.mark.parametrize("act, affine, skip, log", FLAGS)
def test_norm_act(B, T, C, G, act, affine, skip, log):
    _norm_act_case(B, T, C, G, act, affine, skip, log, seed=B * T + C + G)


@pytest.mark.parametrize("B, T, C, G", LONG)
@pytest.mark.parametrize("act, affine, skip, log", [("relu", True, "stride", True), ("gelu", False, "other", False),
                                                    (None, True, "none", False)])
def test_norm_act_30_seconds(B, T, C, G, act, affine, skip, log):
    _norm_act_case(B, T, C, G, act, affine, skip, log, seed=T)


# ---- model level ------------------------------------------------------------------------------------------------------
FEAT_TOL = 1e-3  # max |f - f64| / max |f64| for features and ze


def _model(tmp_path, arch, seed, form="cfg"):
    from audiolm_pytorch_b200.vq_wav2vec import FairseqVQWav2Vec

    st = ov.random_state(arch, seed=seed, groups=arch["vq_groups"], num_vars=arch["vq_vars"],
                         combine_groups=arch["combine_groups"], affine=not arch["non_affine_group_norm"])
    ov.write_checkpoint(tmp_path / "vq.pt", st, arch, form)
    return FairseqVQWav2Vec(tmp_path / "vq.pt").to(DEV), st


def _compare(q, st, arch, wave):
    std = {k: v.to(DEV, F64) for k, v in st.items()}
    f64 = ov.features(std, arch, wave.double())
    ze64 = ov.project(std, f64)
    f = q.extract_features(wave)
    ze = q.quantizer_input(wave)
    ids = q(wave, flatten=False)
    e = ov.codewords(std, ze.shape[2])
    ids64 = ov.ids(ze64, e)
    rel_f = ((f.double() - f64).abs().max() / f64.abs().max()).item()
    dze = ze.double() - ze64
    rel_ze = (dze.abs().max() / ze64.abs().max()).item()
    safe = ov.margins(ze64, e) > 2 * dze.norm(dim=-1)
    assert rel_f < FEAT_TOL and rel_ze < FEAT_TOL, f"feature error {rel_f:.3g}, ze error {rel_ze:.3g}"
    assert ids.dtype == torch.int64 and ids.shape == ids64.shape
    assert torch.equal(ids[safe], ids64[safe]), "ids differ on a margin-safe frame"
    print(f"\n  features {rel_f:.2e}, ze {rel_ze:.2e} max rel err; ids equal on "
          f"{100 * (ids == ids64).double().mean().item():.2f} % of {ids.numel()} ({int(safe.sum())} margin-safe)")
    return ids


PUBLISHED_VARIANT = dict(ov.PUBLISHED, activation="gelu", skip_connections_feat=False, log_compression=False,
                         combine_groups=True, non_affine_group_norm=True)


@pytest.mark.parametrize("variant", ["published", "variant"])
def test_published_shape_against_fp64(tmp_path, variant):
    arch = ov.PUBLISHED if variant == "published" else PUBLISHED_VARIANT
    q, st = _model(tmp_path, arch, seed=3 if variant == "published" else 4)
    g = torch.Generator().manual_seed(5)
    for B, T in ((2, 24000 + 17), (1, 465), (3, 1234)):
        _compare(q, st, arch, torch.randn(B, T, generator=g).to(DEV))


def test_published_shape_30_seconds(tmp_path):
    q, st = _model(tmp_path, ov.PUBLISHED, seed=6)
    _compare(q, st, ov.PUBLISHED, torch.randn(1, 30 * 24000, generator=torch.Generator().manual_seed(7)).to(DEV))


@pytest.fixture(scope="module")
def gd():
    return golden.load("vq_wav2vec.pt")


def _golden_model(tmp_path, m):
    from audiolm_pytorch_b200.vq_wav2vec import FairseqVQWav2Vec

    ov.write_checkpoint(tmp_path / "vq.pt", m["state"], m["arch"])
    return FairseqVQWav2Vec(tmp_path / "vq.pt").to(DEV)


@pytest.mark.parametrize("name", ["A", "B"])
def test_golden_end_to_end(tmp_path, gd, name):
    from torchaudio.functional import resample

    m = gd[name]
    q = _golden_model(tmp_path, m)
    e = ov.codewords({k: v.double() for k, v in m["state"].items()}, 2)
    for wave, feats, ze_g, ids, flat in zip(m["waves"], m["features"], m["ze"], m["ids"], m["ids_flat"]):
        w = wave.to(DEV)
        f = q.extract_features(w).cpu()
        ze = q.quantizer_input(w).cpu()
        assert (f - feats).abs().max() <= FEAT_TOL * feats.abs().max()
        assert (ze - ze_g).abs().max() <= FEAT_TOL * ze_g.abs().max()
        safe = ov.margins(ze_g.double(), e) > 2 * (ze.double() - ze_g.double()).norm(dim=-1) + 1e-6
        got, got_flat = q(w, flatten=False).cpu(), q(w).cpu()
        assert got.shape == ids.shape and got_flat.shape == flat.shape
        assert torch.equal(got[safe], ids[safe]) and torch.equal(got_flat, got.reshape(got.shape[0], -1))
        assert safe.double().mean() > 0.95
    # input_sample_hz resamples (torchaudio) and seq_len_multiple_of curtails, as in the reference
    q.seq_len_multiple_of = m["resample_kw"]["seq_len_multiple_of"]
    got = q(m["wave16"].to(DEV), flatten=False, input_sample_hz=m["resample_kw"]["input_sample_hz"]).cpu()
    w24 = resample(m["wave16"].double(), 16000, 24000)
    w24 = w24[:, :w24.shape[-1] // 320 * 320]
    st64 = {k: v.double() for k, v in m["state"].items()}
    ze64 = ov.project(st64, ov.features(st64, m["arch"], w24))
    ze = q.quantizer_input(w24.float().to(DEV)).cpu().double()
    safe = ov.margins(ze64, e) > 2 * (ze - ze64).norm(dim=-1) + 1e-4
    assert got.shape == m["ids_resampled"].shape
    assert torch.equal(got[safe], m["ids_resampled"][safe]) and safe.double().mean() > 0.9


def test_determinism_and_batch_invariance(tmp_path):
    q, _ = _model(tmp_path, ov.PUBLISHED, seed=8)
    batch = torch.randn(5, 2 * 24000 + 3, generator=torch.Generator().manual_seed(9)).to(DEV)
    f1, f2 = q.extract_features(batch), q.extract_features(batch)
    z1, z2 = q.quantizer_input(batch), q.quantizer_input(batch)
    assert torch.equal(f1, f2) and torch.equal(z1, z2) and torch.equal(q(batch), q(batch))
    alone = batch[3:4].clone()
    assert torch.equal(q.extract_features(alone)[0], f1[3]) and torch.equal(q.quantizer_input(alone)[0], z1[3])
    assert torch.equal(q(alone)[0], q(batch)[3])


def test_cpu_input_raises(tmp_path, gd):
    from audiolm_pytorch_b200._lib import AlmError

    q = _golden_model(tmp_path, gd["B"])
    with pytest.raises(AlmError):
        q(gd["B"]["waves"][0])


# ---- wrappers and AudioLM ----------------------------------------------------------------------------------------------
SMALL_KW = dict(dim=64, depth=2, heads=2, flash_attn=True)


@pytest.fixture(scope="module")
def golden_vq(tmp_path_factory, gd):
    return _golden_model(tmp_path_factory.mktemp("vq"), gd["A"]), gd["A"]


def test_semantic_wrapper_raw_wave(golden_vq):
    from audiolm_pytorch_b200 import SemanticTransformer, SemanticTransformerWrapper

    q, m = golden_vq
    torch.manual_seed(1)
    w = SemanticTransformerWrapper(transformer=SemanticTransformer(num_semantic_tokens=q.codebook_size,
                                                                   **SMALL_KW).to(DEV),
                                   wav2vec=q, mask_prob=0.0).eval()
    wave, ids = m["waves"][-1].to(DEV), m["ids"][-1].to(DEV)
    with torch.no_grad():
        l_wave = w(raw_wave=wave, return_loss=True)
        l_ids = w(semantic_token_ids=ids.clone(), return_loss=True)
    assert torch.isfinite(l_wave) and l_wave.item() == l_ids.item()


def _codec(num_quantizers):
    """a small SoundStream with seeded codebooks (the RVQ's k-means init is not built)"""
    from audiolm_pytorch_b200 import SoundStream

    torch.manual_seed(3)
    codec = SoundStream(codebook_size=64, rq_num_quantizers=num_quantizers, channels=32, codebook_dim=64,
                        use_local_attn=False)
    gen = torch.Generator().manual_seed(4)
    for layer in codec.rq.rvqs[0].layers:
        layer._codebook.embed.copy_(torch.randn(layer._codebook.embed.shape, generator=gen) * 0.05)
        layer._codebook.initted.fill_(True)
    return codec.to(DEV).eval()


def test_coarse_wrapper_raw_wave(golden_vq):
    from audiolm_pytorch_b200 import CoarseTransformer, CoarseTransformerWrapper

    q, m = golden_vq
    codec = _codec(2)
    torch.manual_seed(2)
    coarse = CoarseTransformer(num_semantic_tokens=q.codebook_size, codebook_size=64, num_coarse_quantizers=2,
                               **SMALL_KW).to(DEV)
    w = CoarseTransformerWrapper(transformer=coarse, codec=codec, wav2vec=q, mask_prob=0.0).eval()
    wave, ids = m["waves"][-1].to(DEV), m["ids"][-1].to(DEV)
    with torch.no_grad():
        l_wave = w(raw_wave=wave, raw_wave_for_codec=wave, return_loss=True)
        l_ids = w(semantic_token_ids=ids.clone(), raw_wave_for_codec=wave, return_loss=True)
    assert torch.isfinite(l_wave) and l_wave.item() == l_ids.item()


def test_audiolm_constructs(golden_vq):
    from audiolm_pytorch_b200 import AudioLM, CoarseTransformer, FineTransformer, SemanticTransformer

    q, _ = golden_vq
    codec = _codec(4)
    n = q.codebook_size
    sem = SemanticTransformer(num_semantic_tokens=n, **SMALL_KW).to(DEV)
    coarse = CoarseTransformer(num_semantic_tokens=n, codebook_size=64, num_coarse_quantizers=2, **SMALL_KW).to(DEV)
    fine = FineTransformer(num_coarse_quantizers=2, num_fine_quantizers=2, codebook_size=64, **SMALL_KW).to(DEV)
    lm = AudioLM(wav2vec=q, codec=codec, semantic_transformer=sem, coarse_transformer=coarse, fine_transformer=fine)
    assert lm.semantic.wav2vec is q and lm.coarse.wav2vec is q
