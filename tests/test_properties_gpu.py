"""H100, BASELINE.json full sizes: size-independent properties of the CUDA path (no oracle needed)."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"

C3 = dict(num_semantic_tokens=500, codebook_size=1024, num_coarse_quantizers=3, dim=1024, depth=6, heads=8,
          flash_attn=True)


@pytest.fixture(scope="module")
def coarse_model():
    from audiolm_pytorch_b200.audiolm import CoarseTransformer

    torch.manual_seed(11)
    m = CoarseTransformer(**C3)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if "dynamic_alpha_fn" in n or "dynamic_beta_fn" in n:
                p.normal_(0, 0.02)
            if "logit_weights" in n:
                p.mul_(0.05)
    return m.to(DEV).eval()


def test_c3_causality_and_batch_independence(coarse_model):
    """seq 2048: logits at positions < t do not change when tokens >= t change; rows of a batch are independent."""
    torch.manual_seed(0)
    sem = torch.randint(0, 500, (2, 372), device=DEV)
    coarse = torch.randint(0, 1024, (2, 1674), device=DEV)
    with torch.no_grad():
        sl, cl = coarse_model(semantic_token_ids=sem, coarse_token_ids=coarse)
        c2 = coarse.clone()
        c2[:, 1000:] = torch.randint(0, 1024, (2, 674), device=DEV)
        sl2, cl2 = coarse_model(semantic_token_ids=sem, coarse_token_ids=c2)
        sl3, cl3 = coarse_model(semantic_token_ids=sem[1:], coarse_token_ids=coarse[1:])
    assert cl.shape == (2, 1675, 1025) and sl.shape == (2, 372, 501)
    assert torch.equal(sl, sl2)                      # semantic positions precede every changed token
    assert torch.equal(cl[:, :1001], cl2[:, :1001])  # coarse logit p depends on coarse ids < p only
    assert not torch.equal(cl[:, 1001:], cl2[:, 1001:])
    assert torch.equal(cl[1:], cl3) and torch.equal(sl[1:], sl3)
    assert torch.isfinite(cl).all()


def test_c3_kv_cache_equals_full_forward(coarse_model):
    """incremental decode with kv_cache/embed_cache reproduces the full forward at seq 2048 (reference
    self-consistency property, SURVEY.md §4 (i))."""
    torch.manual_seed(1)
    sem = torch.randint(0, 500, (1, 372), device=DEV)
    coarse = torch.randint(0, 1024, (1, 1674), device=DEV)
    with torch.no_grad():
        (_, full), _ = coarse_model(semantic_token_ids=sem, coarse_token_ids=coarse, return_cache=True,
                                    return_only_coarse_logits=True)
        (_, _), (kv, emb) = coarse_model(semantic_token_ids=sem, coarse_token_ids=coarse[:, :1500], return_cache=True,
                                         return_only_coarse_logits=True)
        (_, inc), _ = coarse_model(semantic_token_ids=sem, coarse_token_ids=coarse, return_cache=True, kv_cache=kv,
                                   embed_cache=emb, return_only_coarse_logits=True)
    err = (inc - full).abs().max().item() / full.abs().max().item()
    assert err < 2e-2, err


def test_c3_gradient_linearity(coarse_model):
    """d(2*loss) == 2*d(loss) through the whole hand-written backward (bit-level up to bf16 rounding of dout)."""
    from audiolm_pytorch_b200.heads import cross_entropy

    coarse_model.train()
    torch.manual_seed(2)
    sem = torch.randint(0, 500, (2, 372), device=DEV)
    coarse = torch.randint(0, 1024, (2, 1674), device=DEV)
    labels = torch.cat((coarse, torch.full((2, 1), 1024, device=DEV)), 1)
    grads = []
    for scale in (1.0, 2.0):
        for p in coarse_model.parameters():
            p.grad = None
        _, cl = coarse_model(semantic_token_ids=sem, coarse_token_ids=coarse)
        (cross_entropy(cl, labels) * scale).backward()
        grads.append(coarse_model.transformer.layers[3][2].branch.get_submodule("1").weight.grad.clone())
    coarse_model.eval()
    rel = (grads[1] - 2 * grads[0]).abs().max().item() / grads[1].abs().max().item()
    assert rel < 2e-2, rel


def test_gemm_linearity_full_ffn_shape():
    from audiolm_pytorch_b200 import ops

    torch.manual_seed(3)
    a1 = torch.randn(4096, 1024, device=DEV).to(torch.bfloat16)
    a2 = torch.randn(4096, 1024, device=DEV).to(torch.bfloat16)
    w = (torch.randn(5472, 1024, device=DEV) * 0.03).to(torch.bfloat16)
    y1 = ops.gemm(a1, w, out_dtype=torch.float32)
    y2 = ops.gemm(a2, w, out_dtype=torch.float32)
    y12 = ops.gemm((a1.float() + a2.float()).to(torch.bfloat16), w, out_dtype=torch.float32)
    # (a1 + a2) is re-rounded to bf16, hence the tolerance
    assert (y12 - (y1 + y2)).abs().max().item() < 2e-2 * y12.abs().max().item()
    # transposed-operand forms agree with the plain form: (a w^T)^T == w a^T
    yt = ops.gemm(w, a1, out_dtype=torch.float32)
    assert torch.equal(yt.t().contiguous(), y1) or (yt.t() - y1).abs().max().item() < 1e-3 * y1.abs().max().item()


def test_c1_codec_properties():
    """2 s @ 24 kHz clips: 150 frames, indices in range, decode of the
    emitted indices reproduces `quantized`, encoder causality past the reflect halo."""
    from audiolm_pytorch_b200 import ops
    from audiolm_pytorch_b200.soundstream import SoundStream

    torch.manual_seed(4)
    ss = SoundStream(codebook_size=1024, rq_num_quantizers=8, target_sample_hz=24000, use_local_attn=False)
    for layer in ss.rq.rvqs[0].layers:
        layer._codebook.embed.normal_(0, 0.3)
        layer._codebook.initted.fill_(True)
    ss = ss.to(DEV).eval()
    wave = torch.randn(4, 48000, device=DEV)
    with torch.no_grad():
        quant, idx, _ = ss(wave, return_encoded=True)
        enc = ss.encoder(wave[:, None]).transpose(1, 2).contiguous()
        cb = ss.rq.rvqs[0].codebooks()
        assert idx.shape == (4, 150, 8) and idx.min() >= 0 and idx.max() < 1024
        dec = ops.rvq_decode(idx.reshape(-1, 8), cb).view(4, 150, 512)
        assert (dec - quant).abs().max().item() < 1e-4
        # optimality of every emitted index: no other code of the stage is closer to that stage's residual
        flat = enc.reshape(-1, 512)
        ids = idx.reshape(-1, 8)
        for q in range(8):
            resid = flat - (ops.rvq_decode(ids[:, :q].contiguous(), cb[:q]) if q else 0)
            d_all = torch.cdist(resid, cb[q])                       # [600, 1024]
            d_sel = d_all.gather(1, ids[:, q:q + 1])[:, 0]
            assert (d_sel <= d_all.min(dim=1).values + 1e-3).all()
        w2 = wave.clone()
        w2[:, 24000:] += 1.0
        enc2 = ss.encoder(w2[:, None]).transpose(1, 2)
        assert torch.equal(enc2[:, :74], enc[:, :74])  # frames fully before sample 24000 (75 * 320) are unchanged
        recon = ss(wave, return_recons_only=True)
        assert recon.shape == (4, 1, 48000)
        assert torch.allclose(ss.decode_from_codebook_indices(idx), recon, atol=1e-5)


@pytest.mark.parametrize("which", ["C2", "C3", "C4"])
def test_full_size_logits_vs_cpu_oracle(which):
    """BASELINE.json configs at full model size and sequence length (batch 1): CUDA logits vs the CPU oracle.
    bf16 activations / fp32 accumulation vs fp32: RMS-relative error < 1e-2 (north_star tolerance)."""
    from audiolm_pytorch_b200 import audiolm
    from oracle import transformer as ot

    torch.manual_seed({"C2": 2, "C3": 3, "C4": 4}[which])
    kw = dict(dim=1024, depth=6, heads=8, flash_attn=True)
    if which == "C2":
        m = audiolm.SemanticTransformer(num_semantic_tokens=500, **kw)
    elif which == "C3":
        m = audiolm.CoarseTransformer(num_semantic_tokens=500, codebook_size=1024, num_coarse_quantizers=3, **kw)
    else:
        m = audiolm.FineTransformer(num_coarse_quantizers=3, num_fine_quantizers=5, codebook_size=1024, **kw)
    with torch.no_grad():
        for n_, p in m.named_parameters():
            if "dynamic_alpha_fn" in n_ or "dynamic_beta_fn" in n_:
                p.normal_(0, 0.02)
            if "logit_weights" in n_:
                p.mul_(0.05)
    st = {k: v.detach().clone() for k, v in m.state_dict().items()}
    hk = dict(heads=8, depth=6)
    torch.set_num_threads(min(32, torch.get_num_threads()))
    with torch.no_grad():
        if which == "C2":
            ids = torch.randint(0, 500, (1, 1023))
            ref = [ot.semantic_forward(st, ids, **hk)[0]]
            got = [m.to(DEV).eval()(ids=ids.to(DEV))]
        elif which == "C3":
            sem, co = torch.randint(0, 500, (1, 372)), torch.randint(0, 1024, (1, 1674))
            ref = list(ot.coarse_forward(st, sem, co, codebook_size=1024, num_coarse_quantizers=3, **hk)[0])
            got = list(m.to(DEV).eval()(semantic_token_ids=sem.to(DEV), coarse_token_ids=co.to(DEV)))
        else:
            # full model size; half of C4's length keeps the fp32 CPU oracle affordable on slow hosts (C3 above covers
            # 2048 positions) while still exercising the ragged coarse / fine remainder heads
            co, fi = torch.randint(0, 1024, (1, 384)), torch.randint(0, 1024, (1, 638))
            ref = list(ot.fine_forward(st, co, fi, codebook_size=1024, num_coarse_quantizers=3, num_fine_quantizers=5,
                                       **hk)[0])
            got = list(m.to(DEV).eval()(coarse_token_ids=co.to(DEV), fine_token_ids=fi.to(DEV)))
    for r, g_ in zip(ref, got):
        assert r.shape == g_.shape
        e = ((g_.float().cpu() - r).pow(2).mean().sqrt() / r.pow(2).mean().sqrt()).item()
        assert e < 1e-2, (which, e)


def test_c3_full_size_gradients_vs_oracle_autograd():
    """C3 at full model size and sequence length (d1024 L6 h8, 2048 positions, batch 1) through the wrapper's own loss
    WITH its key mask (CoarseTransformerWrapper.forward always passes one, audiolm_pytorch.py:1801-1812) and an FCM
    mask: every parameter gradient of the hand-written backward vs torch autograd of the fp32 CPU oracle.
    Tolerances as in test_models_gpu (bf16 activations vs fp32): 7 % RMS for tensors, 30 % of the largest same-kind
    gradient for the <= 20-element hyper-connection tensors."""
    from audiolm_pytorch_b200 import audiolm
    from audiolm_pytorch_b200.heads import cross_entropy
    from oracle import transformer as ot

    torch.manual_seed(23)
    m = audiolm.CoarseTransformer(**C3)
    with torch.no_grad():
        for n_, p in m.named_parameters():
            if "dynamic_alpha_fn" in n_ or "dynamic_beta_fn" in n_:
                p.normal_(0, 0.02)
            if "logit_weights" in n_:
                p.mul_(0.05)
    sem = torch.randint(0, 500, (1, 372))
    coarse = torch.randint(0, 1024, (1, 1674))
    sem_l = sem
    co_l = torch.cat((coarse, torch.full((1, 1), 1024)), 1)
    mask = ot.fcm_mask((1, 2048), 0.15, torch.Generator().manual_seed(3))
    st = {k: v.detach().clone().requires_grad_(v.is_floating_point()) for k, v in m.state_dict().items()}
    torch.set_num_threads(min(32, torch.get_num_threads()))
    (osl, ocl), _ = ot.coarse_forward(st, sem, coarse, self_attn_mask=mask, heads=8, depth=6, codebook_size=1024,
                                      num_coarse_quantizers=3)
    oloss = ot.coarse_wrapper_loss(osl, ocl, sem_l, co_l)
    oloss.backward()
    m = m.to(DEV).train()
    sl, cl = m(semantic_token_ids=sem.to(DEV), coarse_token_ids=coarse.to(DEV), self_attn_mask=mask.to(DEV))
    n_s, n_c = sl.shape[1], cl.shape[1]
    loss = (cross_entropy(sl, sem_l.to(DEV)) * n_s + cross_entropy(cl, co_l.to(DEV)) * n_c) / (n_s + n_c)
    loss.backward()
    assert abs(loss.item() - oloss.item()) < 1e-2 * abs(oloss.item())
    shrunk = ("semantic_start_token", "coarse_start_token", "semantic_embedding.weight", "coarse_embedding.weight",
              "coarse_quantize_embedding.weight")  # grad_shrink (audiolm_pytorch.py:93-94): x0.1 into the embeddings
    golden = {}
    for k, p in m.named_parameters():
        if p.grad is None:
            continue
        g = st[k].grad
        golden[k] = (g * 0.1 if k in shrunk else g)
    kind_scale = {}
    for k, gr in golden.items():
        if gr.numel() <= 20:
            kind = k.split(".")[-1]
            kind_scale[kind] = max(kind_scale.get(kind, 0.0), gr.pow(2).mean().sqrt().item())
    errs = {}
    for k, gr in golden.items():
        got = dict(m.named_parameters())[k].grad.float().cpu()
        if gr.numel() <= 20:
            errs[k] = ((got - gr).pow(2).mean().sqrt().item() / kind_scale[k.split(".")[-1]], 0.30)
        else:
            errs[k] = (((got - gr).pow(2).mean().sqrt() / gr.pow(2).mean().sqrt().clamp(min=1e-20)).item(), 7e-2)
    for k, (e, tol) in sorted(errs.items(), key=lambda kv: -kv[1][0] / kv[1][1])[:8]:
        print(f"  C3 full-size grad err {e:.4f} (tol {tol}) {k}")
    bad = {k: v for k, v in errs.items() if v[0] >= v[1]}
    assert not bad, bad
