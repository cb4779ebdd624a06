"""HubertWithKmeans on the GPU (csrc/hubert.cu + the split-bf16 GEMM + the bf16 attention kernel).

* every new kernel against an fp64 restatement, C / D in {128, ..., 1024}, one frame to 30 s of frames, B in {1, 3, 16},
  both norm modes, each element held to a bound of the error model below;
* HuBERT-base and HuBERT-large shapes with seeded random weights at output_layer 1, 9 and the last, against the fp64
  oracle (oracle/hubert.py): the feature error within a stated tolerance, and ids equal to the fp64 ids on every frame
  whose gap to the runner-up centroid exceeds 2 |df|;
* the golden (the reference's own ids) end to end; bitwise determinism and batch invariance;
* SemanticTransformerWrapper / CoarseTransformerWrapper / AudioLM driven by HubertWithKmeans.

Error model (fp32 arithmetic, unit roundoff u = 2^-24):
  split-bf16 products: |x w - (x_hi w_hi + x_lo w_hi + x_hi w_lo)| <= 2^-15 |x| |w|   (SPLIT)
  fp32 accumulation of K products: K u sum |x| |w|                                     (ACC)
  a fp32 norm / activation output: NORM_U * u (|y| + |gamma|) with NORM_U = 64, room for the two-pass statistics and erf
The attention stage rounds q, k, v and its output to bf16 (2^-8 relative each): its bound is ATTN_REL * max |v|.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import golden
from oracle import hubert as oh

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24
SPLIT = 2.0 ** -15
NORM_U = 64
ATTN_REL = 2.0 ** -6
F64 = torch.float64


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _unsplit(s, C):
    """split layout [.., 3C] -> (hi, lo) fp64; checks the layout's third block repeats hi"""
    hi, lo, hi2 = s[..., :C].double(), s[..., C:2 * C].double(), s[..., 2 * C:].double()
    assert torch.equal(hi, hi2)
    return hi, lo


def _check_split(s, ref):
    hi, lo = _unsplit(s, ref.shape[-1])
    assert torch.equal(hi, ref.to(torch.bfloat16).double())
    assert ((hi + lo - ref).abs() <= 2.0 ** -16 * ref.abs() + 1e-38).all()


# ---- kernels -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B, T, C", [(1, 2, 128), (3, 97, 256), (16, 3, 512), (1, 95999, 512), (3, 500, 768),
                                     (1, 1499, 1024)])
@pytest.mark.parametrize("mode", ["group", "layer", "none"])
def test_norm_act_kernel(B, T, C, mode):
    from audiolm_pytorch_b200 import ops

    g = _gen(B * T + C)
    y = torch.randn(B, T, C, device=DEV, generator=g) * 3 + torch.randn(C, device=DEV, generator=g)
    gamma = 1 + 0.2 * torch.randn(C, device=DEV, generator=g)
    beta = 0.2 * torch.randn(C, device=DEV, generator=g)
    bias = torch.randn(C, device=DEV, generator=g) if mode != "group" else None
    yd = y.double() + (bias.double() if bias is not None else 0)
    if mode == "group":
        out, s = ops.hubert_norm_act(y, stats=ops.hubert_chan_stats(y), gamma=gamma, beta=beta, gelu=True,
                                     want_out=True)
        ref = F.group_norm(yd.transpose(1, 2), C, gamma.double(), beta.double(), 1e-5).transpose(1, 2)
    elif mode == "layer":
        out, s = ops.hubert_norm_act(y, bias=bias, ln=True, gamma=gamma, beta=beta, gelu=True, want_out=True)
        ref = F.layer_norm(yd, (C,), gamma.double(), beta.double(), 1e-5)
    else:
        out, s = ops.hubert_norm_act(y, bias=bias, gelu=True, want_out=True)
        ref = yd
    norm_scale = gamma.double().abs() + (ref.abs() if mode == "none" else 1)
    ref = F.gelu(ref)
    err = (out.double() - ref).abs()
    bound = NORM_U * U * (ref.abs() + norm_scale) * (1 + (math.log2(T) if mode == "group" else 0))
    assert (err <= bound).all(), f"max err/bound {(err / bound).max().item():.3g}"
    _check_split(s, out.double())


@pytest.mark.parametrize("B, T, D", [(1, 1, 128), (3, 50, 768), (16, 7, 1024), (1, 1500, 256)])
@pytest.mark.parametrize("case", ["post_ln", "pre_ln", "pos_conv", "plain"])
def test_add_ln_kernel(B, T, D, case):
    from audiolm_pytorch_b200 import ops

    g = _gen(B + T + D)
    r = torch.randn(B, T, D, device=DEV, generator=g)
    gamma = 1 + 0.2 * torch.randn(D, device=DEV, generator=g)
    beta = 0.2 * torch.randn(D, device=DEV, generator=g)
    groups = 16 if case == "pos_conv" else 1
    y = torch.randn(B, groups, T, D // groups, device=DEV, generator=g) if groups > 1 else \
        torch.randn(B, T, D, device=DEV, generator=g)
    y_bias = torch.randn(D, device=DEV, generator=g) if case == "pos_conv" else None
    yd = y.double().permute(0, 2, 1, 3).reshape(B, T, D) if groups > 1 else y.double()
    if y_bias is not None:
        yd = F.gelu(yd + y_bias.double())
    r_new = r.double() + yd
    x = r.clone()
    kw = dict(gamma=gamma, beta=beta) if case != "plain" else {}
    s = ops.hubert_add_ln(x, y, T=T, groups=groups, y_bias=y_bias, y_gelu=y_bias is not None,
                          keep_ln=case in ("post_ln", "pos_conv"), **kw)
    ln = F.layer_norm(r_new, (D,), gamma.double(), beta.double(), 1e-5)
    ref = ln if case in ("post_ln", "pos_conv") else r_new
    bound = NORM_U * U * (ref.abs() + gamma.double().abs() + r_new.abs())
    assert ((x.double() - ref).abs() <= bound).all()
    if case != "plain":
        hi, lo = _unsplit(s, D)
        assert ((hi + lo - ln).abs() <= bound + 2.0 ** -16 * ln.abs()).all()
    else:
        assert s is None


def _conv_bound(x, w, stride, groups=1, padding=0):
    """SPLIT + ACC bound of a conv computed from split operands, elementwise"""
    k = w.shape[1] * w.shape[2]
    absconv = F.conv1d(x.abs(), w.abs(), stride=stride, groups=groups, padding=padding)
    return (SPLIT + k * U) * absconv + 1e-30


@pytest.mark.parametrize("B, T, C, Cout, k, s", [(1, 3, 128, 128, 3, 2), (3, 401, 512, 512, 3, 2),
                                                 (16, 64, 256, 768, 2, 2), (1, 47999, 512, 512, 3, 2),
                                                 (3, 21, 1024, 1024, 2, 2), (1, 2, 512, 512, 2, 2)])
def test_conv_gemm(B, T, C, Cout, k, s):
    from audiolm_pytorch_b200 import ops

    g = _gen(T + C)
    x = torch.randn(B, T, C, device=DEV, generator=g)
    w = torch.randn(Cout, C, k, device=DEV, generator=g) / math.sqrt(C * k)
    bias = torch.randn(Cout, device=DEV, generator=g)
    _, xs = ops.hubert_norm_act(x)
    y = ops.hubert_conv_gemm(xs, ops.pack_split_conv_weight(w), bias, kernel_size=k, stride=s)
    ref = F.conv1d(x.double().transpose(1, 2), w.double(), bias.double(), stride=s).transpose(1, 2)
    bound = _conv_bound(x.double().transpose(1, 2), w.double(), s).transpose(1, 2) + U * ref.abs()
    assert y.shape == ref.shape and ((y.double() - ref).abs() <= bound).all()


@pytest.mark.parametrize("B, T, D, groups", [(1, 1, 768, 16), (3, 50, 768, 16), (16, 9, 1024, 16),
                                             (1, 1500, 1024, 16), (3, 31, 256, 16), (1, 64, 128, 4)])
def test_pos_conv(B, T, D, groups):
    from audiolm_pytorch_b200 import ops

    g = _gen(T + D)
    k = 128
    x = torch.randn(B, T, D, device=DEV, generator=g)
    w = torch.randn(D, D // groups, k, device=DEV, generator=g) / math.sqrt(k * D // groups)
    wp = ops.pack_split_conv_weight(w).view(groups, D // groups, -1)
    y = ops.hubert_pos_conv(x, wp, kernel_size=k)
    y = y.permute(0, 2, 1, 3).reshape(B, T, D).double()
    xd = x.double().transpose(1, 2)
    ref = F.conv1d(xd, w.double(), padding=k // 2, groups=groups)[..., :T].transpose(1, 2)
    bound = _conv_bound(xd, w.double(), 1, groups, k // 2)[..., :T].transpose(1, 2)
    assert ((y - ref).abs() <= bound).all()


@pytest.mark.parametrize("B, T, D, heads", [(1, 1, 768, 12), (3, 50, 1024, 16), (16, 13, 256, 4), (1, 1500, 768, 12)])
def test_attention_stage(B, T, D, heads):
    from audiolm_pytorch_b200 import ops

    g = _gen(T + D)
    qkv = torch.randn(B, T, 3 * D, device=DEV, generator=g)
    s = ops.hubert_attention(qkv, heads=heads)
    o, lo = _unsplit(s, D)
    assert (lo == 0).all()
    dh = D // heads
    q, k, v = (t.double().view(B, T, heads, dh).transpose(1, 2) for t in qkv.split(D, dim=-1))
    ref = (torch.softmax(q @ k.transpose(-1, -2) * dh ** -0.5, -1) @ v).transpose(1, 2).reshape(B, T, D)
    assert ((o - ref).abs() <= ATTN_REL * v.abs().amax()).all()


def test_conv0_kernel():
    from audiolm_pytorch_b200 import ops

    for B, T in ((1, 400), (3, 16001), (16, 4003)):
        g = _gen(T)
        wave = torch.randn(B, T, device=DEV, generator=g)
        w = torch.randn(512, 1, 10, device=DEV, generator=g)
        bias = torch.randn(512, device=DEV, generator=g)
        y = ops.hubert_conv0(wave, w, bias, stride=5)
        ref = F.conv1d(wave.double()[:, None], w.double(), bias.double(), stride=5).transpose(1, 2)
        bound = 11 * U * (F.conv1d(wave.double().abs()[:, None], w.double().abs(), stride=5).transpose(1, 2)
                          + bias.double().abs())
        assert ((y.double() - ref).abs() <= bound).all()


# ---- model level ------------------------------------------------------------------------------------------------------
FEAT_TOL = 1e-2  # max |f - f64| / max |f64|: the bf16 attention dominates (3.6e-3 at most measured)


def _model(tmp_path, arch, output_layer, seed, n_clusters=500, wn="weight_g"):
    from audiolm_pytorch_b200.hubert import HubertWithKmeans

    st = oh.random_state(arch, seed=seed)
    if wn != "weight_g":
        st = oh.parametrized_weight_norm(st)
    centers = torch.randn(n_clusters, arch["encoder_embed_dim"], generator=torch.Generator().manual_seed(seed + 1))
    oh.write_checkpoint(tmp_path / "ck.pt", st, arch)
    oh.write_kmeans(tmp_path / "km.bin", centers)
    return HubertWithKmeans(tmp_path / "ck.pt", tmp_path / "km.bin", output_layer=output_layer).to(DEV), st, centers


def _compare(h, st, arch, centers, wave, output_layer):
    f = h.extract_features(wave)
    ids = h(wave)
    std = {k: v.to(DEV, F64) for k, v in st.items()}
    f64 = oh.extract_features(std, arch, wave.double(), output_layer)
    c64 = centers.to(DEV, F64)
    ids64 = oh.assign(f64, c64)
    df = (f.double() - f64)
    rel = (df.abs().max() / f64.abs().max()).item()
    safe = oh.margins(f64, c64) > 2 * df.norm(dim=-1)
    agree = (ids == ids64).double().mean().item()
    assert rel < FEAT_TOL, f"feature error {rel:.3g}"
    assert torch.equal(ids[safe], ids64[safe]), "ids differ on a margin-safe frame"
    print(f"\n  feature max rel err {rel:.2e}, ids equal on {100 * agree:.1f} % of {ids.numel()} frames "
          f"({int(safe.sum())} margin-safe)")
    return ids, f


@pytest.mark.parametrize("family, output_layer", [("base", 1), ("base", 9), ("base", 12), ("large", 1), ("large", 9),
                                                  ("large", 24)])
def test_published_shapes_against_fp64(tmp_path, family, output_layer):
    arch = oh.BASE if family == "base" else oh.LARGE
    h, st, centers = _model(tmp_path, arch, output_layer, seed=output_layer,
                            wn="weight_g" if family == "base" else "parametrizations")
    g = torch.Generator().manual_seed(3)
    for B, T in ((3, 16000 + 17), (1, 400)):
        _compare(h, st, arch, centers, torch.randn(B, T, generator=g).to(DEV), output_layer)


def test_base_30_seconds(tmp_path):
    h, st, centers = _model(tmp_path, oh.BASE, 2, seed=30)
    wave = torch.randn(1, 30 * 16000, generator=torch.Generator().manual_seed(4)).to(DEV)
    _compare(h, st, oh.BASE, centers, wave, 2)


def test_golden_end_to_end(tmp_path):
    from audiolm_pytorch_b200.hubert import HubertWithKmeans

    gd = golden.load("hubert.pt")
    oh.write_checkpoint(tmp_path / "ck.pt", gd["state"], gd["arch"])
    oh.write_kmeans(tmp_path / "km.bin", gd["centers"])
    h = HubertWithKmeans(tmp_path / "ck.pt", tmp_path / "km.bin", output_layer=gd["output_layer"]).to(DEV)
    for wave, feats, ids in zip(gd["waves"], gd["features"], gd["ids"]):
        f = h.extract_features(wave.to(DEV)).cpu()
        assert (f - feats).abs().max() <= FEAT_TOL * feats.abs().max()
        assert torch.equal(h(wave.to(DEV)).cpu(), ids)


def test_determinism_and_batch_invariance(tmp_path):
    h, _, _ = _model(tmp_path, oh.BASE, 9, seed=5)
    g = torch.Generator().manual_seed(6)
    batch = torch.randn(8, 2 * 16000 + 3, generator=g).to(DEV)
    f1, f2 = h.extract_features(batch), h.extract_features(batch)
    assert torch.equal(f1, f2) and torch.equal(h(batch), h(batch))
    alone = h.extract_features(batch[5:6].clone())
    assert torch.equal(alone[0], f1[5])
    assert torch.equal(h(batch[5:6].clone())[0], h(batch)[5])


def test_forward_options(tmp_path):
    """input_sample_hz resamples with torchaudio, seq_len_multiple_of curtails, flatten=False gives [B, n]"""
    from torchaudio.functional import resample

    h, _, _ = _model(tmp_path, oh.BASE, 1, seed=7)
    h.seq_len_multiple_of = 320
    wave = torch.randn(2, 24000 + 77, generator=torch.Generator().manual_seed(8)).to(DEV)
    ids = h(wave, input_sample_hz=24000, flatten=False)
    w16 = resample(wave, 24000, 16000)
    assert ids.dtype == torch.int64 and ids.shape == (2, (w16.shape[-1] // 320 * 320 - 400) // 320 + 1)
    assert torch.equal(ids, h(w16[:, :w16.shape[-1] // 320 * 320]))


# ---- wrappers and AudioLM ----------------------------------------------------------------------------------------------
SMALL_KW = dict(dim=64, depth=2, heads=2, flash_attn=True)


@pytest.fixture(scope="module")
def golden_hubert(tmp_path_factory):
    from audiolm_pytorch_b200.hubert import HubertWithKmeans

    d = tmp_path_factory.mktemp("hubert")
    gd = golden.load("hubert.pt")
    oh.write_checkpoint(d / "ck.pt", gd["state"], gd["arch"])
    oh.write_kmeans(d / "km.bin", gd["centers"])
    return HubertWithKmeans(d / "ck.pt", d / "km.bin", output_layer=gd["output_layer"]).to(DEV)


def test_semantic_wrapper_raw_wave(golden_hubert):
    from audiolm_pytorch_b200 import SemanticTransformer, SemanticTransformerWrapper

    torch.manual_seed(1)
    n = golden_hubert.codebook_size
    w = SemanticTransformerWrapper(transformer=SemanticTransformer(num_semantic_tokens=n, **SMALL_KW).to(DEV),
                                   wav2vec=golden_hubert, mask_prob=0.0).eval()
    wave = torch.randn(2, 16000, generator=torch.Generator().manual_seed(2)).to(DEV)
    ids = golden_hubert(wave, flatten=False)
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


def test_coarse_wrapper_raw_wave(golden_hubert):
    from audiolm_pytorch_b200 import CoarseTransformer, CoarseTransformerWrapper

    codec = _codec(2)
    coarse = CoarseTransformer(num_semantic_tokens=golden_hubert.codebook_size, codebook_size=64,
                               num_coarse_quantizers=2, **SMALL_KW).to(DEV)
    w = CoarseTransformerWrapper(transformer=coarse, codec=codec, wav2vec=golden_hubert, mask_prob=0.0).eval()
    wave = torch.randn(2, 16000, generator=torch.Generator().manual_seed(4)).to(DEV)
    with torch.no_grad():
        loss = w(raw_wave=wave, raw_wave_for_codec=wave, return_loss=True)
    assert torch.isfinite(loss)


def test_audiolm_prime_wave(golden_hubert, monkeypatch):
    from audiolm_pytorch_b200 import AudioLM, CoarseTransformer, FineTransformer, SemanticTransformer

    codec = _codec(4)
    torch.manual_seed(5)
    n = golden_hubert.codebook_size
    sem = SemanticTransformer(num_semantic_tokens=n, **SMALL_KW).to(DEV)
    coarse = CoarseTransformer(num_semantic_tokens=n, codebook_size=64, num_coarse_quantizers=2, **SMALL_KW).to(DEV)
    fine = FineTransformer(num_coarse_quantizers=2, num_fine_quantizers=2, codebook_size=64, **SMALL_KW).to(DEV)
    lm = AudioLM(wav2vec=golden_hubert, codec=codec, semantic_transformer=sem, coarse_transformer=coarse,
                 fine_transformer=fine)
    real = lm.coarse.generate
    monkeypatch.setattr(lm.coarse, "generate", lambda **k: real(**{**k, "max_time_steps": 8}))
    prime = torch.randn(1, 16000, generator=torch.Generator().manual_seed(6)).to(DEV)
    wav = lm(prime_wave=prime, prime_wave_input_sample_hz=16000, max_length=golden_hubert(prime).shape[1] + 4)
    wavs = [wav] if torch.is_tensor(wav) and wav.dim() == 1 else list(wav)
    assert len(wavs) == 1 and all(w_ is None or torch.isfinite(w_).all() for w_ in wavs)
