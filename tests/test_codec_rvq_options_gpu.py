"""H100: the residual VQ's cosine-similarity search and codebook_dim projections (csrc/rvq_tc.cu, split-bf16 GEMM).

* The cosine search (ops.rvq_encode_tc(metric="cosine")) against fp64 across its envelope (oracle/rvq_options.py):
  the chosen code lies within the fp32 band of the fp64 maximum on every (row, stage), the fp64 argmax is chosen
  wherever the band isolates it, zero residuals take code 0, quantized equals the fp32 replay of the ids bit for bit,
  and rvq_decode of the ids equals quantized bit for bit.  Codebooks are the generators' own (not unit norm), unit
  norm, and rows rescaled over two decades.
* The split-bf16 score error on normalised rows, measured against fp64, leaves 4x headroom under CAND_TOL_COS.
* project_in / project_out (ops.split_linear) within 1e-5 of fp64, relative to |x| |w_j| + |b_j|.
* SoundStream on tests/golden/rvq_options.pt (fp32 and tensor-core codecs), reproducibility, and the wrappers.
"""

import pytest
import torch

from oracle import golden
from oracle import nearest_code as nc
from oracle import rvq_options as ro

pytestmark = pytest.mark.gpu
DEV = "cuda"
CAND_TOL_COS = 1e-4   # rvq_tc.cu


def _bits(t):
    return t.contiguous().view(torch.int32)


def _cosine(x, cb):
    from audiolm_pytorch_b200 import ops

    return ops.rvq_encode_tc(x, ops.rvq_pack_codebooks(cb), metric="cosine")


def _renorm(cb, norm, g):
    if norm == "unit":
        return cb / cb.norm(dim=-1, keepdim=True)
    if norm == "scaled":   # row norms spread over two decades
        return cb * 10 ** (torch.rand(*cb.shape[:2], 1, generator=g) * 2 - 1)
    return cb


def _cases():
    """every D with every C; Q, generator and codebook norm rotate so each value meets each of the others"""
    out = []
    gens, norms = list(nc.GENERATORS), ["as_generated", "unit", "scaled"]
    for i, D in enumerate((8, 24, 64, 256, 512, 1024)):
        for k, C in enumerate((2, 64, 1024, 4096)):
            Q = (1, 8, 32)[(i + k) % 3]
            if C * D * Q > 2 ** 25:   # keep the fp64 replay of the widest cases affordable
                Q = 8 if Q == 32 else 1
            out.append((D, C, Q, gens[(i + 2 * k) % 4], norms[(i + k) % 3]))
    return out


GEN_KW = {"gaussian": dict(x_scale=3.0), "clustered": dict(spread=1e-2), "offset": dict(level=30.0),
          "shrinking": dict(ratio=0.7)}


@pytest.mark.parametrize("D, C, Q, gen, norm", _cases())
def test_cosine_search_vs_fp64(D, C, Q, gen, norm):
    from audiolm_pytorch_b200 import ops

    N = 700
    g = torch.Generator().manual_seed(D * 7 + C + Q)
    x, cb = nc.GENERATORS[gen](N, C, D, Q, g=g, **GEN_KW[gen])
    cb = _renorm(cb, norm, g)
    x[0] = 0                               # F.normalize(0) = 0: every score 0, code 0
    x, cb = x.to(DEV), cb.to(DEV)
    quant, ids = _cosine(x, cb)
    assert ids.shape == (N, Q) and quant.shape == (N, D)
    assert ids[0, 0].item() == 0
    share = ro.check_cosine_fp64(x, cb, ids, quant=quant, label=f"D={D} C={C} Q={Q} {gen} {norm}")
    _, i64 = ro.cosine_search_fp64(x, cb)
    same = (ids == i64).all(1).float().mean().item()
    print(f"D={D} C={C} Q={Q} {gen} {norm}: {share:.3%} of (row, stage) pairs in the fp32 band; "
          f"rows equal to the fp64 search throughout {same:.2%}")
    assert torch.equal(_bits(ops.rvq_decode(ids, cb)), _bits(quant))


def test_cosine_zero_rows_and_padding():
    """zero rows take code 0 at the first stage and follow the fp64 rule after it; a width that is not a multiple of 8
    runs padded; a strided x (a column slice) reads only its columns"""
    g = torch.Generator().manual_seed(3)
    cb = torch.randn(3, 50, 20, generator=g).to(DEV)
    x = torch.randn(40, 20, generator=g).to(DEV)
    x[:7] = 0
    wide = torch.full((40, 36), float("nan"), device=DEV)
    wide[:, 8:28] = x
    quant, ids = _cosine(wide[:, 8:28], cb)
    assert not ids[:7, 0].any()
    ro.check_cosine_fp64(x, cb, ids, quant=quant, label="zero rows")
    _, i64 = ro.cosine_search_fp64(x, cb)
    assert torch.equal(ids[:7], i64[:7])


@pytest.mark.parametrize("D", [8, 24, 64, 128, 256, 512, 768, 1024])
def test_cosine_score_window_headroom(D):
    """the split-bf16 scores S ~ r^.e with R' built as the cosine prepare builds it (split of the normalised row):
    max |S - r^.e| / (|r^|^2 + |e|^2) must stay under CAND_TOL_COS / 4 for every generator and codebook norm"""
    from audiolm_pytorch_b200 import ops

    N, C = 2048, 1024
    g = torch.Generator().manual_seed(D)
    worst = {}
    for name in nc.GENERATORS:
        for norm in ("as_generated", "unit", "scaled"):
            x, cb = nc.GENERATORS[name](N, C, D, 1, g=g, **GEN_KW[name])
            cb = _renorm(cb, norm, g).to(DEV)
            x = x.to(DEV)
            x[0] = 0
            cbp, packed, e2 = ops.rvq_pack_codebooks(cb)
            r = torch.empty(N, D, device=DEV)
            rp = torch.empty(N, 3 * D, device=DEV, dtype=torch.bfloat16)
            from audiolm_pytorch_b200 import _lib

            _lib.call("alm_rvq_prepare_cos", x, D, r, torch.empty(N, D, device=DEV), D, rp, N, D, D)
            S = ops.gemm(rp, packed[0], out=torch.empty(N, C, device=DEV)).double()
            xh = torch.nn.functional.normalize(x.double(), dim=1)
            e64 = cb[0].double()
            den = (xh * xh).sum(1, keepdim=True) + (e64 * e64).sum(1)[None]
            worst[f"{name}/{norm}"] = ((S - xh @ e64.T).abs() / den).max().item()
    top = max(worst.values())
    print(f"cosine score error / (|r^|^2 + |e|^2) at D = {D} on {torch.cuda.get_device_name()}: max {top:.2e} "
          f"({max(worst, key=worst.get)}); CAND_TOL_COS / max = {CAND_TOL_COS / top:.0f}x")
    assert top <= CAND_TOL_COS / 4


@pytest.mark.parametrize("K, M", [(512, 64), (512, 128), (64, 512), (32, 8), (8, 32), (1024, 8), (16, 16)])
def test_split_linear_vs_fp64(K, M):
    from audiolm_pytorch_b200 import ops

    g = torch.Generator().manual_seed(K + M)
    x = (torch.randn(3000, K, generator=g) * 3).to(DEV)
    w = (torch.randn(M, K, generator=g) / K ** 0.5).to(DEV)
    b = torch.randn(M, generator=g).to(DEV)
    y = ops.split_linear(x, ops.pack_split_weight(w), b)
    y64 = ro.linear_fp64(x, w, b)
    scale = x.double().norm(dim=1, keepdim=True) * w.double().norm(dim=1)[None] + b.double().abs()[None]
    rel = ((y.double() - y64).abs() / scale).max().item()
    print(f"split_linear {K} -> {M}: max error / (|x| |w_j| + |b_j|) {rel:.2e}")
    assert y.shape == (3000, M) and rel <= 1e-5


# ---- SoundStream ----------------------------------------------------------------------------------------------------
G = golden.load("rvq_options.pt")


def _golden_model(name):
    from audiolm_pytorch_b200 import SoundStream

    g = G[name]
    st = {**ro.seeded_state(g["keys"], g["seed"]), **{f"rq.{k}": v for k, v in g["rq_state"].items()}}
    ss = SoundStream(**g["kwargs"])
    ss.load_state_dict({k: v for k, v in st.items() if k.split(".")[0] in ("encoder", "decoder", "rq")}, strict=True)
    return g, ss.to(DEV).eval()


@pytest.mark.parametrize("name", sorted(G))
def test_golden_end_to_end(name):
    g, ss = _golden_model(name)
    tc = name.startswith("tc/")
    assert (ss._tc_plan() is not None) == tc and (ss._tc_plan_dec() is not None) == tc
    wave = g["wave"].to(DEV)
    with torch.no_grad():
        quant_rq, ids_rq, _ = ss.rq(g["enc"].to(DEV))
        quant, ids, loss = ss(wave, return_encoded=True)
        tok = ss.tokenize(wave)
        recon_idx = ss.decode_from_codebook_indices(g["ids"].to(DEV))
    b, n = g["ids"].shape[:2]
    # the quantizer on the reference's encoder output
    ids_flat = ids_rq.permute(1, 2, 0, 3).reshape(b, n, -1).cpu()
    assert torch.equal(ids_flat, g["ids"]), f"{name}: {(ids_flat != g['ids']).sum().item()} ids differ"
    assert (quant_rq.cpu() - g["quant"]).abs().max() < 1e-4 * max(1.0, g["quant"].abs().max().item())
    # through this build's encoder
    agree = (ids.cpu() == g["ids"]).float().mean().item()
    print(f"{name}: tokenize agrees with the reference on {agree:.2%} of ids")
    assert tok.shape == (ss.rq_groups, b, n, g["ids"].shape[-1] // ss.rq_groups) and tok.dtype == torch.int64
    assert torch.equal(tok.permute(1, 2, 0, 3).reshape(b, n, -1), ids) and agree > 0.9
    assert float(loss.sum()) == 0.0
    if torch.equal(ids.cpu(), g["ids"]):
        assert (quant.cpu() - g["quant"]).abs().max() < 1e-4 * max(1.0, g["quant"].abs().max().item())
    scale = max(1.0, g["recon_idx"].abs().max().item())
    assert (recon_idx.cpu() - g["recon_idx"]).abs().max() < 1e-4 * scale


def test_reproducible_and_batch_invariant():
    """a clip's ids and quantized are bitwise the same across runs and alone or inside a batch of 5"""
    _, ss = _golden_model("tc/cosine_proj8_g2")
    wave = torch.randn(5, 320 * 24, generator=torch.Generator().manual_seed(8)).to(DEV)
    with torch.no_grad():
        q1, i1, _ = ss(wave, return_encoded=True)
        q2, i2, _ = ss(wave, return_encoded=True)
        q3, i3, _ = ss(wave[2:3], return_encoded=True)
        h = ss.encode_frames(wave[:, None])
        qa, ia, _ = ss.rq(h)
        qb, ib, _ = ss.rq(h[3:4])
    assert torch.equal(i1, i2) and torch.equal(_bits(q1), _bits(q2))
    assert torch.equal(i3, i1[2:3]) and torch.equal(_bits(q3), _bits(q1[2:3]))
    assert torch.equal(ib, ia[:, 3:4]) and torch.equal(_bits(qb), _bits(qa[3:4]))


# ---- wrappers -------------------------------------------------------------------------------------------------------
@pytest.fixture
def no_eos(monkeypatch):
    """keep EOS out of the sampler so generated clips are long enough for the codec (as test_wrappers_gpu does)"""
    from audiolm_pytorch_b200 import ops

    sample = ops.topk_gumbel_sample

    def sampler(logits, noise, *, k, temperature=1.0):
        logits = logits.clone()
        logits[:, -1] = float("-inf")
        return sample(logits, noise, k=k, temperature=temperature)

    monkeypatch.setattr(ops, "topk_gumbel_sample", sampler)


def _tiny_audiolm():
    from audiolm_pytorch_b200 import AudioLM, CoarseTransformer, FineTransformer, SemanticTransformer, SoundStream

    torch.manual_seed(5)
    codec = SoundStream(codebook_size=64, rq_num_quantizers=4, channels=32, codebook_dim=64, use_local_attn=False,
                        rq_kwargs=dict(use_cosine_sim=True, codebook_dim=16))
    with torch.no_grad():
        for layer in codec.rq.rvqs[0].layers:
            layer._codebook.embed.normal_()
            layer._codebook.initted.fill_(1)
    kw = dict(dim=64, depth=2, heads=2, flash_attn=True)
    sem = SemanticTransformer(num_semantic_tokens=50, **kw).to(DEV)
    coarse = CoarseTransformer(num_semantic_tokens=50, codebook_size=64, num_coarse_quantizers=2, **kw).to(DEV)
    fine = FineTransformer(num_coarse_quantizers=2, num_fine_quantizers=2, codebook_size=64, **kw).to(DEV)
    codec = codec.to(DEV).eval()
    return AudioLM(wav2vec=None, codec=codec, semantic_transformer=sem, coarse_transformer=coarse,
                   fine_transformer=fine), codec, coarse, fine


def test_wrappers_on_cosine_projected_codec(no_eos):
    from audiolm_pytorch_b200 import CoarseTransformerWrapper, FineTransformerWrapper

    _, codec, coarse, fine = _tiny_audiolm()
    cw = CoarseTransformerWrapper(transformer=coarse, codec=codec, mask_prob=0.0)
    fw = FineTransformerWrapper(transformer=fine, codec=codec, mask_prob=0.0)
    wave = torch.randn(2, 320 * 20, generator=torch.Generator().manual_seed(4)).to(DEV)
    sem = torch.randint(0, 50, (2, 16), generator=torch.Generator().manual_seed(5)).to(DEV)
    ids = codec.tokenize(wave)
    with torch.no_grad():
        l_wave = cw(semantic_token_ids=sem, raw_wave=wave, return_loss=True)
        l_ids = cw(semantic_token_ids=sem, coarse_token_ids=ids[0][..., :2], return_loss=True)
    assert torch.isfinite(l_wave) and l_wave.item() == l_ids.item()
    torch.manual_seed(2)
    sem = torch.randint(0, 50, (2, 12), device=DEV)
    coarse_ids = cw.generate(semantic_token_ids=sem, max_time_steps=12)
    assert coarse_ids.dtype == torch.int64
    wav_c = cw.generate(semantic_token_ids=sem, max_time_steps=12, reconstruct_wave=True)
    for w_ in (wav_c if isinstance(wav_c, list) else list(wav_c)):
        assert w_ is None or torch.isfinite(w_).all()
    prime = torch.randint(0, 64, (2, 10, 2), device=DEV)
    wav_f = fw.generate(coarse_token_ids=prime, reconstruct_wave=True)
    wav_f = wav_f if torch.is_tensor(wav_f) else torch.stack(wav_f)
    assert wav_f.shape == (2, 10 * codec.seq_len_multiple_of) and torch.isfinite(wav_f).all()
    with torch.no_grad():
        assert torch.isfinite(fw(raw_wave=wave, return_loss=True))


def test_audiolm_on_cosine_projected_codec(no_eos, monkeypatch):
    lm, codec, _, _ = _tiny_audiolm()
    real = lm.coarse.generate
    monkeypatch.setattr(lm.coarse, "generate", lambda **k: real(**{**k, "max_time_steps": 8}))
    torch.manual_seed(11)
    wav = lm(batch_size=2, max_length=12)
    wavs = list(wav) if not torch.is_tensor(wav) else [w for w in wav]
    assert len(wavs) == 2
    for w in wavs:
        assert w is not None and torch.isfinite(w).all() and 0 < w.shape[-1] <= 8 * codec.seq_len_multiple_of
