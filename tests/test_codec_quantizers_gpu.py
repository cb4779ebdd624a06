"""H100: residual FSQ / LFQ (csrc/scalar_quant.cu) against the fp64 restatement in oracle/scalar_quant.py across the
kernels' envelope, the reference models of tests/golden/quantizers.pt end to end, C1-size FSQ / LFQ codecs on the
tensor-core encoder and decoder, and the AudioLM wrappers on top of them."""

import pytest
import torch

from oracle import golden
from oracle import scalar_quant as osq
from oracle.transformer import sub

pytestmark = pytest.mark.gpu
DEV = "cuda"
EPS = 2.0 ** -23

LEVELS = {1: [2], 3: [3, 4, 7], 4: [8, 5, 5, 5], 10: [5, 4, 3, 2, 6, 7, 3, 4, 2, 5], 16: [2, 3] * 8}
FLIPS = {}


def _cases():
    """every dc with every Dg, each mode; Q, groups and N rotate so each value meets each of the others"""
    out = []
    for mode in ("fsq", "lfq"):
        for i, dc in enumerate(LEVELS):
            for k, dg in enumerate((dc, 32, 512, 1024)):
                out.append((mode, dc, dg, (1, 4, 32)[(i + k) % 3], (1, 2, 4)[(i + 2 * k) % 3],
                            (1, 7, 9600)[(i + k + (mode == "lfq")) % 3]))
    return out


def _setup(mode, dc, dg, Q, groups, N, seed):
    from audiolm_pytorch_b200 import ops

    gen = torch.Generator().manual_seed(seed)
    D = groups * dg
    # strided rows: x is a window of a wider buffer
    buf = torch.randn(N, D + 12, generator=gen) * 1.5
    x = buf[:, 5:5 + D]
    weights = None
    if dg != dc:
        weights = (torch.randn(groups, dc, dg, generator=gen) * (2.0 / dg ** 0.5), torch.randn(groups, dc, generator=gen),
                   torch.randn(groups, dg, dc, generator=gen) / dc ** 0.5, torch.randn(groups, dg, generator=gen))
    consts, ints = ops.fsq_constants(LEVELS[dc], Q) if mode == "fsq" else ops.lfq_constants(dc, Q)
    kw = dict(mode=mode, levels=LEVELS[dc], codebook_dim=dc, num_quantizers=Q)
    return buf, x, weights, consts, ints, kw


def _dev_weights(weights):
    if weights is None:
        return None
    w_in, b_in, w_out, b_out = weights
    return tuple(t.to(DEV).contiguous() for t in (w_in, b_in, w_out.transpose(1, 2), b_out))


def _proj_error(x, weights, groups):
    """a bound on the fp32 project_in error of any row (lane-strided fmas + a 5-level butterfly + the bias)"""
    if weights is None:
        return 0.0
    dg = x.shape[1] // groups
    mag = max((x[:, g * dg:(g + 1) * dg].abs().double() @ weights[0][g].abs().double().t()).max().item()
              + weights[1][g].abs().max().item() for g in range(groups))
    return (dg // 32 + 8) * EPS * mag


@pytest.mark.parametrize("mode,dc,dg,Q,groups,N", _cases())
def test_sq_kernels_vs_fp64(mode, dc, dg, Q, groups, N):
    from audiolm_pytorch_b200 import ops

    buf, x, weights, consts, ints, kw = _setup(mode, dc, dg, Q, groups, N, seed=dc * 1000 + dg + Q + groups + N)
    q64, i64, margin = osq.residual_sq_fp64(x, groups=groups, weights=weights,
                                            fp32_projection_error=_proj_error(x, weights, groups), **kw)
    dw = _dev_weights(weights)
    xd = buf.to(DEV)[:, 5:5 + x.shape[1]]
    assert xd.stride(0) == x.shape[1] + 12
    dt = torch.int32 if mode == "fsq" else torch.int64
    quant, idx = ops.sq_encode(xd, mode=mode, groups=groups, weights=dw, consts=consts.to(DEV), ints=ints.to(DEV),
                               index_dtype=dt)
    torch.cuda.synchronize()
    assert idx.dtype == dt and idx.shape == (groups, N, Q) and quant.shape == x.shape
    idx_c, quant_c = idx.cpu().long(), quant.cpu().double()
    safe_q = margin > 1                                                      # [g, N, Q]: stages 0..q decided with margin
    safe = safe_q[..., -1]
    flips = (idx_c != i64).any(-1)
    FLIPS[(mode, dc, dg, Q, groups, N)] = (safe.float().mean().item(), flips[~safe].float().mean().item()
                                           if (~safe).any() else 0.0)
    print(f"{mode} dc={dc} Dg={dg} Q={Q} g={groups} N={N}: margin-safe rows {safe.float().mean().item():.1%}, "
          f"stages {safe_q.float().mean().item():.1%}; rows with a differing index outside the margin "
          f"{FLIPS[(mode, dc, dg, Q, groups, N)][1]:.2%}")
    assert torch.equal(idx_c[safe_q], i64[safe_q]), "indices must be bit-exact on margin-safe stages"
    if mode == "lfq" and weights is None:
        # identity LFQ has no inexact step: every row matches the fp32 quantizer bit for bit
        rq = osq.GroupedResidualLFQ(dim=x.shape[1], groups=groups, codebook_size=2 ** dc, num_quantizers=Q).eval()
        q32, i32, _ = rq(x.contiguous()[None])
        assert torch.equal(idx_c, i32[:, 0]) and torch.equal(quant.cpu(), q32[0])
    # quantized on rows whose every group has the fp64 indices: within the fp32 projections' error
    rows = (idx_c == i64).all(-1).all(0)
    if rows.any():
        if weights is None:
            tol = 4 * EPS * q64.abs().max().item() * Q
        else:
            tol = 1e-5 * max(1.0, q64.abs().max().item())
        assert (quant_c[rows] - q64[rows]).abs().max().item() <= tol
    # decoding the encoder's own indices is bit-exact, from int32 and from int64
    w = dict(mode=mode, Dg=dg, weights=dw, consts=consts.to(DEV), ints=ints.to(DEV))
    assert torch.equal(ops.sq_decode(idx, **w), quant)
    assert torch.equal(ops.sq_decode(idx.to(torch.int64 if dt == torch.int32 else torch.int32), **w), quant)
    # leading stages only, and dropped (-1) entries, against the fp64 restatement of the same indices
    part = idx[..., :max(1, Q // 2)].clone()
    part[:, ::3, 0] = -1
    got = ops.sq_decode(part, **w).cpu().double()
    ref = osq.decode_fp64(part.cpu(), weights=weights, **kw)
    assert (got - ref).abs().max().item() <= 1e-5 * max(1.0, ref.abs().max().item())


def test_sq_unsupported_refused():
    from audiolm_pytorch_b200 import _lib, ops

    consts, ints = (t.to(DEV) for t in ops.lfq_constants(4, 2))
    x = torch.randn(3, 12, device=DEV)
    with pytest.raises(_lib.AlmError, match="-4"):   # groups 3
        ops.sq_encode(x, mode="lfq", groups=3, weights=None, consts=consts, ints=ints, index_dtype=torch.int64)
    idx = torch.zeros(1, 3, 3, dtype=torch.int64, device=DEV)
    with pytest.raises(_lib.AlmError, match="-4"):   # more stages than the quantizer has
        ops.sq_decode(idx, mode="lfq", Dg=4, weights=None, consts=consts, ints=ints)


def test_flip_rates_reported():
    """summary of the rows outside the margin (printed; the bit-exact rule covers the rest)"""
    if not FLIPS:
        pytest.skip("run with the envelope test")
    worst = max(v[1] for v in FLIPS.values())
    print(f"{len(FLIPS)} cases; worst differing-row rate outside the margin {worst:.2%}; "
          f"mean margin-safe share {sum(v[0] for v in FLIPS.values()) / len(FLIPS):.1%}")


@pytest.mark.parametrize("name", ["fsq", "fsq_groups", "lfq", "lfq_groups"])
def test_golden_end_to_end(name):
    from audiolm_pytorch_b200 import SoundStream

    g = golden.load("quantizers.pt")[name]
    ss = SoundStream(**g["kwargs"])
    ss.load_state_dict(g["state"], strict=True)
    ss = ss.to(DEV).eval()
    wave = g["wave"].to(DEV)
    # the quantizer on the reference's encoder output: exact on margin-safe frames
    groups = g["kwargs"].get("rq_groups", 1)
    rq = osq.build_rq(g["kwargs"], sub(g["state"], "rq"))
    weights = None
    if isinstance(rq.rvqs[0].project_in, torch.nn.Linear):
        weights = tuple(torch.stack([getattr(getattr(r, m), a) for r in rq.rvqs]).detach()
                        for m, a in (("project_in", "weight"), ("project_in", "bias"), ("project_out", "weight"),
                                     ("project_out", "bias")))
    kw = dict(mode=name[:3], levels=g["kwargs"].get("finite_scalar_quantizer_levels"),
              codebook_dim=(g["codebook_size"].bit_length() - 1), num_quantizers=g["kwargs"]["rq_num_quantizers"])
    enc = g["enc"]
    flat = enc.reshape(-1, enc.shape[-1])
    _, i64, margin = osq.residual_sq_fp64(flat, groups=groups, weights=weights,
                                          fp32_projection_error=_proj_error(flat, weights, groups), **kw)
    with torch.no_grad():
        out = ss.rq(enc.to(DEV))
    idx = out[1].cpu()
    assert idx.dtype == g["idx"].dtype
    safe = (margin > 1).reshape(groups, *enc.shape[:2], -1)
    assert torch.equal(idx[safe], g["idx"][safe])
    if name == "lfq_groups":   # identity projections: exact everywhere
        assert torch.equal(idx, g["idx"])
    assert (out[0].cpu() - g["quant"]).abs().max() < 1e-4
    with torch.no_grad():
        tok = ss.tokenize(wave)
        recon = ss(wave, return_recons_only=True)
        recon_idx = ss.decode_from_codebook_indices(g["idx"].to(DEV))
        recon_c = ss.decode_from_codebook_indices(g["idx"][..., :g["coarse_q"]].to(DEV))
        quant, ids, loss = ss(wave, return_encoded=True)
    print(f"{name}: tokenize agrees with the reference on {(tok.cpu() == g['idx']).float().mean().item():.2%} of ids")
    assert tok.dtype == g["idx"].dtype and tok.shape == g["idx"].shape
    assert (tok.cpu() == g["idx"]).float().mean() > 0.9
    assert ids.shape == (2, 10, groups * kw["num_quantizers"]) and float(loss.sum()) == 0.0
    scale = max(1.0, g["recon_idx"].abs().max().item())
    assert (recon_idx.cpu() - g["recon_idx"]).abs().max() < 1e-4 * scale
    assert (recon_c.cpu() - g["recon_coarse"]).abs().max() < 1e-4 * scale
    if torch.equal(tok.cpu(), g["idx"]):
        assert (recon.cpu() - g["recon"]).abs().max() < 1e-4 * scale


def _c1_codec(kind, seed):
    from audiolm_pytorch_b200 import SoundStream

    torch.manual_seed(seed)
    kw = dict(target_sample_hz=24000, use_local_attn=False)
    if kind == "fsq":
        return SoundStream(finite_scalar_quantizer_levels=[8, 5, 5, 5], use_finite_scalar_quantizer=True, **kw)
    return SoundStream(codebook_size=1024, use_lookup_free_quantizer=True, **kw)


@pytest.mark.parametrize("kind", ["fsq", "lfq"])
def test_c1_codec_vs_oracle(kind):
    """C1 codec (32 channels, codebook_dim 512, 8 stages) on the tensor-core encoder and decoder, batch 64 x 48 000:
    the quantizer on the encoder output against the fp64 restatement, the decoder against the codec oracle"""
    from oracle import codec as oc

    ss = _c1_codec(kind, 31)
    st = {k: v.detach().clone() for k, v in ss.state_dict().items()}
    ss = ss.to(DEV).eval()
    assert ss._tc_plan() is not None and ss._tc_plan_dec() is not None
    wave = torch.randn(64, 48000, generator=torch.Generator().manual_seed(9))
    with torch.no_grad():
        enc = ss.encode_frames(wave.to(DEV)[:, None, :])
        quant, idx, _ = ss(wave.to(DEV), return_encoded=True)
        ids = ss.tokenize(wave.to(DEV))
        recon = ss.decode_from_codebook_indices(idx[:2])
    assert ids.dtype == (torch.int32 if kind == "fsq" else torch.int64) and ids.shape == (1, 64, 150, 8)
    rq = ss.rq.rvqs[0]
    weights = tuple(t.detach().cpu()[None] for t in (rq.project_in.weight, rq.project_in.bias, rq.project_out.weight,
                                                      rq.project_out.bias))
    flat = enc.reshape(-1, 512).cpu()
    kw = dict(mode=kind, levels=[8, 5, 5, 5], codebook_dim=10, num_quantizers=8)
    q64, i64, margin = osq.residual_sq_fp64(flat, groups=1, weights=weights,
                                            fp32_projection_error=_proj_error(flat, weights, 1), **kw)
    got = idx.reshape(-1, 8).cpu().long()
    safe_q = margin[0] > 1
    safe = safe_q[:, -1]
    print(f"C1 {kind}: margin-safe frames {safe.float().mean().item():.1%}, stages {safe_q.float().mean().item():.1%}; "
          f"differing frames outside the margin "
          f"{(got != i64[0]).any(-1)[~safe].float().mean().item() if (~safe).any() else 0.0:.2%}")
    assert safe_q[:, 0].float().mean() > 0.9
    assert torch.equal(got[safe_q], i64[0][safe_q])
    same = (got == i64[0]).all(-1)
    assert same.float().mean() > 0.9
    assert (quant.reshape(-1, 512).cpu().double()[same] - q64[same]).abs().max() < 1e-4
    torch.set_num_threads(min(32, torch.get_num_threads()))
    x = osq.decode_fp64(ids[:, :2].reshape(1, -1, 8).cpu(), weights=weights, **kw).float().reshape(2, 150, 512)
    ref = oc.decoder(sub(st, "decoder"), x.transpose(1, 2))
    e, scale = (recon.cpu() - ref).abs().max().item(), ref.abs().max().item()
    print(f"C1 {kind} decoder max abs err {e:.3e} (scale {scale:.3f})")
    assert recon.shape == ref.shape == (2, 1, 48000) and e < 2e-4 * max(1.0, scale)


@pytest.fixture
def no_eos(monkeypatch):
    """random weights would sample EOS now and then, leaving clips shorter than the codec's reflect halo (the reference
    cannot decode those either): keep the last class out of the sampler, as test_wrappers_gpu does"""
    from audiolm_pytorch_b200 import ops

    sample = ops.topk_gumbel_sample

    def sampler(logits, noise, *, k, temperature=1.0):
        logits = logits.clone()
        logits[:, -1] = float("-inf")
        return sample(logits, noise, k=k, temperature=temperature)

    monkeypatch.setattr(ops, "topk_gumbel_sample", sampler)


def _tiny_audiolm(kind):
    from audiolm_pytorch_b200 import AudioLM, CoarseTransformer, FineTransformer, SemanticTransformer, SoundStream

    torch.manual_seed(5)
    if kind == "fsq":
        codec = SoundStream(finite_scalar_quantizer_levels=[5, 4, 4], use_finite_scalar_quantizer=True,
                            rq_num_quantizers=4, channels=32, codebook_dim=64, use_local_attn=False)
    else:
        codec = SoundStream(codebook_size=64, use_lookup_free_quantizer=True, rq_num_quantizers=4, channels=32,
                            codebook_dim=64, use_local_attn=False)
    cs = codec.codebook_size
    kw = dict(dim=64, depth=2, heads=2, flash_attn=True)
    sem = SemanticTransformer(num_semantic_tokens=50, **kw).to(DEV)
    coarse = CoarseTransformer(num_semantic_tokens=50, codebook_size=cs, num_coarse_quantizers=2, **kw).to(DEV)
    fine = FineTransformer(num_coarse_quantizers=2, num_fine_quantizers=2, codebook_size=cs, **kw).to(DEV)
    codec = codec.to(DEV).eval()
    return AudioLM(wav2vec=None, codec=codec, semantic_transformer=sem, coarse_transformer=coarse,
                   fine_transformer=fine), codec, coarse, fine


def test_coarse_wrapper_raw_wave_on_fsq_codec():
    """raw_wave tokenisation through an FSQ codec (int32 ids) gives the loss of the codec's own ids"""
    from audiolm_pytorch_b200 import CoarseTransformerWrapper

    _, codec, coarse, _ = _tiny_audiolm("fsq")
    w = CoarseTransformerWrapper(transformer=coarse, codec=codec, mask_prob=0.0).eval()
    wave = torch.randn(2, 320 * 20, generator=torch.Generator().manual_seed(4)).to(DEV)
    sem = torch.randint(0, 50, (2, 16), generator=torch.Generator().manual_seed(5)).to(DEV)
    ids = codec.tokenize(wave)
    assert ids.dtype == torch.int32
    with torch.no_grad():
        l_wave = w(semantic_token_ids=sem, raw_wave=wave, return_loss=True)
        l_ids = w(semantic_token_ids=sem, coarse_token_ids=ids[0][..., :2], return_loss=True)
    assert torch.isfinite(l_wave) and l_wave.item() == l_ids.item()


@pytest.mark.parametrize("kind", ["fsq", "lfq"])
def test_wrappers_generate_reconstruct_wave(kind, no_eos):
    from audiolm_pytorch_b200 import CoarseTransformerWrapper, FineTransformerWrapper

    lm, codec, coarse, fine = _tiny_audiolm(kind)
    cw = CoarseTransformerWrapper(transformer=coarse, codec=codec, mask_prob=0.0)
    fw = FineTransformerWrapper(transformer=fine, codec=codec, mask_prob=0.0)
    torch.manual_seed(2)
    sem = torch.randint(0, 50, (2, 12), device=DEV)
    coarse_ids = cw.generate(semantic_token_ids=sem, max_time_steps=12)
    wav_c = cw.generate(semantic_token_ids=sem, max_time_steps=12, reconstruct_wave=True)
    for w_ in (wav_c if isinstance(wav_c, list) else list(wav_c)):
        assert w_ is None or torch.isfinite(w_).all()
    prime = torch.randint(0, codec.codebook_size, (2, 10, 2), device=DEV)
    wav_f = fw.generate(coarse_token_ids=prime, reconstruct_wave=True)
    wav_f = wav_f if torch.is_tensor(wav_f) else torch.stack(wav_f)
    assert wav_f.shape == (2, 10 * codec.seq_len_multiple_of) and torch.isfinite(wav_f).all()
    # the fine wrapper's raw-wave path tokenises through the codec too
    wave = torch.randn(2, 20 * codec.seq_len_multiple_of, device=DEV)
    with torch.no_grad():
        assert torch.isfinite(fw(raw_wave=wave, return_loss=True))
    assert coarse_ids.dtype == torch.int64


@pytest.mark.parametrize("kind", ["fsq", "lfq"])
def test_audiolm_end_to_end(kind, no_eos, monkeypatch):
    """AudioLM (semantic -> coarse -> fine -> codec decode) on an FSQ / LFQ codec"""
    lm, codec, _, _ = _tiny_audiolm(kind)
    real = lm.coarse.generate
    monkeypatch.setattr(lm.coarse, "generate", lambda **k: real(**{**k, "max_time_steps": 8}))
    torch.manual_seed(11)
    wav = lm(batch_size=2, max_length=12)
    wavs = list(wav) if not torch.is_tensor(wav) else [w for w in wav]
    assert len(wavs) == 2
    for w in wavs:
        assert w is not None and torch.isfinite(w).all() and 0 < w.shape[-1] <= 8 * codec.seq_len_multiple_of
