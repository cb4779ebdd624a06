"""H100: dropout on the sm_90a kernels (attention probabilities, attention-branch output, feed-forward) against fp32
restatements that apply the same masks, materialised with alm_dropout_bf16 on tensors of ones."""
import sys
from pathlib import Path

import numpy as np
import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, str(Path(__file__).resolve().parent))
import dropout_ref  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
bf16 = torch.bfloat16


def rel_err(a, b):
    a, b = a.float(), b.float()
    return ((a - b).abs().max() / b.abs().max().clamp(min=1e-6)).item()


def rms_rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).pow(2).mean().sqrt() / b.pow(2).mean().sqrt().clamp(min=1e-12)).item()


def mask_factors(M, C, p, seed, site):
    """[M, C] fp32 dropout factors (0 or 1/(1-p)) of keep(seed, site, row, col), from the kernel run on ones"""
    from audiolm_pytorch_b200 import ops

    Cp = (C + 15) // 16 * 16
    ones = torch.ones(M, Cp, device=DEV, dtype=bf16)
    ops.dropout_(ones, p, seed, site)
    return (ones[:, :C] != 0).float() / (1 - p)


def attn_mask_factors(b, h, n_q, n_k, p, seed, site):
    """[b, h, n_q, n_k] factors: counter row (b*h + head) * n_q_pad + i, column = key"""
    n_q_pad = (n_q + 127) // 128 * 128
    return mask_factors(b * h * n_q_pad, n_k, p, seed, site).view(b, h, n_q_pad, n_k)[:, :, :n_q]


# ---- 1. the mask itself ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("p", [0.1, 0.5])
def test_mask_statistics(p):
    from audiolm_pytorch_b200 import ops

    N = 4096
    x = torch.ones(N, N, device=DEV, dtype=bf16)
    ops.dropout_(x, p, 0x1234_5678_9ABC_DEF0, 3)
    kept = x != 0
    assert torch.equal(x[kept], torch.full_like(x[kept], 1 / (1 - p)))  # 1/(1-p) rounded to bf16
    k = kept.double()
    sd = lambda n: 5 * np.sqrt(p * (1 - p) / n)  # noqa: E731
    assert abs(k.mean().item() - (1 - p)) < sd(N * N)
    assert (k.mean(1) - (1 - p)).abs().max().item() < sd(N)
    assert (k.mean(0) - (1 - p)).abs().max().item() < sd(N)

    def corr(a, b):
        a, b = a.double().flatten(), b.double().flatten()
        return torch.corrcoef(torch.stack((a, b)))[0, 1].item()

    y = torch.ones(N, N, device=DEV, dtype=bf16)
    ops.dropout_(y, p, 0x1234_5678_9ABC_DEF1, 3)   # another seed
    z = torch.ones(N, N, device=DEV, dtype=bf16)
    ops.dropout_(z, p, 0x1234_5678_9ABC_DEF0, 4)   # another site
    assert abs(corr(kept, y != 0)) < 5 / N and abs(corr(kept, z != 0)) < 5 / N
    # bit-exact against the numpy restatement of keep() on a block away from the origin
    rows, cols = np.arange(1000, 1064), np.arange(2000, 2512)
    ref = dropout_ref.keep(0x1234_5678_9ABC_DEF0, 3, rows, cols, p)
    assert np.array_equal(kept[1000:1064, 2000:2512].cpu().numpy(), ref)


def test_dropout_is_its_own_backward_and_handles_tails():
    """same (seed, site) on a strided [M, C] view with ragged M and C: the same elements are kept"""
    from audiolm_pytorch_b200 import ops

    torch.manual_seed(0)
    buf = torch.randn(77, 264, device=DEV).to(bf16)
    x = buf[:, :200]
    ref = x.float() * mask_factors(77, 200, 0.3, 99, 5)
    ops.dropout_(x, 0.3, 99, 5)
    assert rel_err(x, ref) < 1e-2
    assert torch.equal(x == 0, ref == 0)


# ---- 2. attention ------------------------------------------------------------------------------------------------
def attend_drop_ref(q, k, v, mask, causal, Z, bias=None):
    scale = q.shape[-1] ** -0.5
    sim = torch.einsum("bhid,bjd->bhij", q, k) * scale
    if bias is not None:
        sim = sim + bias
    neg = -torch.finfo(sim.dtype).max
    if mask is not None:
        sim = sim.masked_fill(~mask[:, None, None, :], neg)
    if causal:
        i, j = sim.shape[-2:]
        sim = sim.masked_fill(torch.ones(i, j, dtype=torch.bool, device=q.device).triu(j - i + 1), neg)
    return torch.einsum("bhij,bjd->bhid", sim.softmax(-1) * Z, v)


ATTN_CASES = [
    # b, h, n_q, n_k, masked, causal, bias  (the CASES of test_attn_gpu.py, plus a score-bias case)
    (1, 1, 128, 128, False, True, False),
    (2, 8, 256, 256, False, True, False),
    (2, 8, 300, 300, True, True, False),
    (1, 8, 2048, 2048, True, True, False),
    (2, 4, 128, 384, False, True, False),
    (2, 2, 200, 200, True, False, False),
    (2, 4, 200, 200, True, True, True),
]


@pytest.mark.parametrize("b,h,n_q,n_k,masked,causal,has_bias", ATTN_CASES)
def test_attn_dropout_vs_fp32(b, h, n_q, n_k, masked, causal, has_bias):
    from audiolm_pytorch_b200 import ops

    torch.manual_seed(n_q + 13 * n_k + h)
    p, seed, site = 0.1, 0xDEADBEEF_01234567, 11
    q = torch.randn(b, n_q, h * 64, device=DEV).to(bf16)
    k = torch.randn(b, n_k, 64, device=DEV).to(bf16)
    v = torch.randn(b, n_k, 64, device=DEV).to(bf16)
    d_o = torch.randn(b, n_q, h * 64, device=DEV).to(bf16)
    mask = None
    if masked:
        mask = torch.rand(b, n_k, device=DEV) > 0.15
        mask[:, 0] = True
    bias = dbias = None
    if has_bias:
        bias = torch.zeros(h, n_q, (n_k + 3) // 4 * 4, device=DEV)
        bias[..., :n_k] = torch.randn(h, n_q, n_k, device=DEV)
        dbias = torch.zeros_like(bias)
    drop = (p, seed, site)
    o, lse = ops.mqa_attn_fwd(q, k, v, heads=h, key_mask=mask, causal=causal, bias=bias, dropout=drop)
    _, lse0 = ops.mqa_attn_fwd(q, k, v, heads=h, key_mask=mask, causal=causal, bias=bias)
    dq, dk, dv = ops.mqa_attn_bwd(q, k, v, o, d_o, lse, heads=h, key_mask=mask, causal=causal, bias=bias, dbias=dbias,
                                  dropout=drop)
    torch.cuda.synchronize()
    assert torch.equal(lse[..., :n_q], lse0[..., :n_q])  # the LSE is that of the un-dropped probabilities
    Z = attn_mask_factors(b, h, n_q, n_k, p, seed, site)
    ql, kl, vl = (t.float().clone().requires_grad_(True) for t in (q, k, v))
    bl = bias[..., :n_k].clone().requires_grad_(True) if has_bias else None
    qh = ql.reshape(b, n_q, h, 64).permute(0, 2, 1, 3)
    ref = attend_drop_ref(qh, kl, vl, mask, causal, Z, bl).permute(0, 2, 1, 3).reshape(b, n_q, h * 64)
    assert (o.float() - ref).abs().max().item() <= 2e-2 * max(1.0, ref.abs().max().item())
    (ref * d_o.float()).sum().backward()
    assert rel_err(dq, ql.grad) < 2e-2
    assert rel_err(dk, kl.grad) < 2e-2
    assert rel_err(dv, vl.grad) < 2e-2
    if has_bias:
        assert rel_err(dbias[..., :n_k], bl.grad) < 2e-2


def test_attn_dropout_unbiased():
    """E[O] over seeds is the dropout-free O (inverted dropout)"""
    from audiolm_pytorch_b200 import ops

    torch.manual_seed(4)
    b, h, n = 1, 2, 128
    q = torch.randn(b, n, h * 64, device=DEV).to(bf16)
    k = torch.randn(b, n, 64, device=DEV).to(bf16)
    v = torch.randn(b, n, 64, device=DEV).to(bf16)
    qh = q.float().reshape(b, n, h, 64).permute(0, 2, 1, 3)
    ref = attend_drop_ref(qh, k.float(), v.float(), None, True, 1.0).permute(0, 2, 1, 3).reshape(b, n, h * 64)
    S = 512
    outs = torch.stack([ops.mqa_attn_fwd(q, k, v, heads=h, dropout=(0.5, 1000 + s, 0))[0].float() for s in range(S)])
    mean, se = outs.mean(0), outs.std(0) / S ** 0.5
    z = (mean - ref).abs() / (se + 4e-3)          # + bf16 rounding of the outputs
    assert z.max().item() < 6, z.max().item()


# ---- 4. GEGLU + LayerNorm --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,inner", [(33, 170), (256, 2730), (64, 512)])
def test_geglu_ln_dropout(M, inner):
    from audiolm_pytorch_b200 import ops

    torch.manual_seed(inner)
    p, seed, site = 0.2, 77, 2
    ip = (inner + 7) // 8 * 8
    h = torch.randn(M, 2 * ip, device=DEV).to(bf16)
    gamma = 1 + 0.1 * torch.randn(inner, device=DEV)
    Z = mask_factors(M, inner, p, seed, site)
    hl = h.float().clone().requires_grad_(True)
    gml = gamma.clone().requires_grad_(True)
    a, gate = hl[:, :inner], hl[:, ip:ip + inner]
    ref = F.layer_norm(F.gelu(gate) * a, (inner,)) * gml * Z
    gn, stats = ops.geglu_ln_fwd(h, gamma, inner=inner, inner_pad=ip, dropout=(p, seed, site))
    assert rel_err(gn[:, :inner], ref) < 1.5e-2
    assert (gn[:, :inner][Z == 0] == 0).all()
    assert (gn[:, inner:] == 0).all()
    w = torch.randn(M, ip, device=DEV).to(bf16)
    (ref * w[:, :inner].float()).sum().backward()
    g_gamma = torch.zeros_like(gamma)
    dh = ops.geglu_ln_bwd(h, gamma, stats, w, g_gamma, inner=inner, inner_pad=ip, dropout=(p, seed, site))
    assert rel_err(dh[:, :inner], hl.grad[:, :inner]) < 2e-2
    assert rel_err(dh[:, ip:ip + inner], hl.grad[:, ip:ip + inner]) < 2e-2
    assert rel_err(g_gamma, gml.grad) < 2e-2


# ---- 5. the whole stack against the oracle with the same masks --------------------------------------------------
def _stack(num_streams, flash, p, seed=0):
    from audiolm_pytorch_b200.transformer import Transformer

    torch.manual_seed(seed)
    tr = Transformer(dim=128, depth=2, heads=2, attn_dropout=p, ff_dropout=p, flash_attn=flash,
                     num_residual_streams=num_streams)
    with torch.no_grad():
        for n_, prm in tr.named_parameters():
            if "dynamic_alpha_fn" in n_ or "dynamic_beta_fn" in n_:
                prm.normal_(0, 0.05)
            if "dynamic_alpha_scale" in n_ or "dynamic_beta_scale" in n_:
                prm.fill_(0.3)
    return tr.to(DEV)


def stack_vs_oracle(num_streams, flash, p, b=2, n=200):
    """loss / output / every parameter gradient of a training step vs the fp32 oracle given the same dropout masks;
    returns the output RMS-relative error, the loss relative error and {param: (error, tolerance)}"""
    from audiolm_pytorch_b200.transformer import _draw_dropout_seed

    d, H, depth = 128, 2, 2
    tr = _stack(num_streams, flash, p).train()
    torch.manual_seed(21)
    x = torch.randn(b, n, d, device=DEV)
    W_logits = torch.randn(d, 64, device=DEV) / d ** 0.5   # a cross-entropy head, as in test_models_gpu.py
    labels = torch.randint(0, 64, (b * n,), device=DEV)
    st = {k: v.detach().clone().float().requires_grad_(v.is_floating_point()) for k, v in tr.state_dict().items()}
    torch.manual_seed(1234)
    seed = _draw_dropout_seed()
    inner = tr.layers[0][2].branch.inner
    masks = [(attn_mask_factors(b, H, n, n, p, seed, 3 * i), mask_factors(b * n, d, p, seed, 3 * i + 1).view(b, n, d),
              mask_factors(b * n, inner, p, seed, 3 * i + 2).view(b, n, inner)) for i in range(depth)]
    out_ref = dropout_ref.transformer_with_dropout(st, x, heads=H, depth=depth, num_streams=num_streams,
                                                   dropout_masks=masks)
    loss_ref = F.cross_entropy((out_ref @ W_logits).view(-1, 64), labels)
    loss_ref.backward()
    torch.manual_seed(1234)   # the forward draws the same seed
    out = tr(x)
    loss = F.cross_entropy((out.float() @ W_logits).view(-1, 64), labels)
    loss.backward()
    named = dict(tr.named_parameters())
    golden = {k: st[k].grad.cpu() for k in named if st[k].grad is not None}
    kind_scale = {}
    for k, gr in golden.items():
        if gr.numel() <= 20:
            kind = k.split(".")[-1]
            kind_scale[kind] = max(kind_scale.get(kind, 0.0), gr.pow(2).mean().sqrt().item())
    errs = {}
    for k, gr in golden.items():
        got = named[k].grad.float().cpu()
        if gr.numel() <= 20:
            errs[k] = ((got - gr).pow(2).mean().sqrt().item() / kind_scale[k.split(".")[-1]], 0.30)
        else:
            errs[k] = (rms_rel(got, gr), 7e-2)
    return rms_rel(out, out_ref), abs(loss.item() - loss_ref.item()) / abs(loss_ref.item()), errs


def _is_hyper_connection(name):
    """the hyper-connection parameters of layer wrappers (not their branches): layers.{i}.{0,2}.<param>"""
    parts = name.split(".")
    return parts[0] == "layers" and parts[3] != "branch"


@pytest.mark.parametrize("num_streams", [1, 4])
@pytest.mark.parametrize("flash", [True, False])
def test_stack_with_dropout_vs_oracle(num_streams, flash):
    """Each bound is the static one of test_models_gpu.py (1e-2 on output and loss, 7e-2 RMS-relative per gradient,
    0.30 of the same-kind scale for the <= 20-element tensors), or twice the error the same step shows WITHOUT dropout
    when that is larger, as check_grads there does with the reference's own bf16 noise.  The hyper-connection and
    rel-pos-bias gradients are sums of strongly cancelling bf16 terms (the last rel-pos bias is exactly zero in exact
    arithmetic: softmax ignores a constant shift), so at this size their error without dropout exceeds 7e-2; the
    hyper-connection tensors get the 0.30 bound test_models_gpu.py gives the small ones of that kind."""
    out0, loss0, errs0 = stack_vs_oracle(num_streams, flash, 0.0)
    out_err, loss_err, errs = stack_vs_oracle(num_streams, flash, 0.1)
    assert out_err < max(1e-2, 2 * out0) and loss_err < max(1e-2, 2 * loss0)
    errs = {k: (e, max(tol, 2 * errs0[k][0], 0.30 if _is_hyper_connection(k) else 0.0)) for k, (e, tol) in errs.items()}
    for k, (e, tol) in sorted(errs.items(), key=lambda kv: -kv[1][0] / kv[1][1])[:5]:
        print(f"  grad err {e:.4f} (tol {tol:.4f}) {k}")
    bad = {k: v for k, v in errs.items() if v[0] >= v[1]}
    assert not bad, bad


# ---- 6. identity and reproducibility ----------------------------------------------------------------------------
@pytest.mark.parametrize("num_streams", [1, 4])
def test_eval_is_bitwise_dropout_free(num_streams):
    tr1 = _stack(num_streams, False, 0.1).eval()
    tr0 = _stack(num_streams, False, 0.0).eval()
    tr0.load_state_dict(tr1.state_dict())
    x = torch.randn(2, 150, 128, device=DEV)
    with torch.no_grad():
        assert torch.equal(tr1(x), tr0(x))
        o1, c1 = tr1(x[:, :100], return_kv_cache=True)
        o0, c0 = tr0(x[:, :100], return_kv_cache=True)
        assert torch.equal(tr1(x, kv_cache=c1), tr0(x, kv_cache=c0))


def test_training_without_dropout_draws_no_seed():
    tr = _stack(4, True, 0.0).train()
    x = torch.randn(2, 100, 128, device=DEV)
    state = torch.get_rng_state()
    tr(x).float().pow(2).mean().backward()
    assert torch.equal(torch.get_rng_state(), state)


def test_same_seed_same_step():
    from audiolm_pytorch_b200 import ops

    tr = _stack(4, False, 0.1).train()
    x = torch.randn(2, 180, 128, device=DEV)

    def step(s):
        torch.manual_seed(s)
        for prm in tr.parameters():
            prm.grad = None
        loss = tr(x).float().pow(2).mean()
        loss.backward()
        return loss.detach().clone()

    l1, l2, l3 = step(7), step(7), step(8)
    assert torch.equal(l1, l2) and not torch.equal(l1, l3)
    # dk / dv of the attention kernels are bitwise reproducible with dropout too
    torch.manual_seed(0)
    q = torch.randn(2, 256, 4 * 64, device=DEV).to(bf16)
    k = torch.randn(2, 256, 64, device=DEV).to(bf16)
    v = torch.randn(2, 256, 64, device=DEV).to(bf16)
    d_o = torch.randn(2, 256, 4 * 64, device=DEV).to(bf16)
    res = []
    for _ in range(2):
        o, lse = ops.mqa_attn_fwd(q, k, v, heads=4, dropout=(0.1, 5, 1))
        _, dk, dv = ops.mqa_attn_bwd(q, k, v, o, d_o, lse, heads=4, dropout=(0.1, 5, 1))
        res.append((o, dk, dv))
    assert all(torch.equal(a, c) for a, c in zip(*res))


def test_coarse_wrapper_trains_with_dropout_then_generates():
    from audiolm_pytorch_b200.audiolm import CoarseTransformer, CoarseTransformerWrapper

    class _Codec:  # the wrapper constructors only read these
        rq_groups = 1
        num_quantizers = 8

    torch.manual_seed(5)
    m = CoarseTransformer(num_semantic_tokens=50, codebook_size=64, num_coarse_quantizers=2, dim=64, depth=2, heads=2,
                          flash_attn=True, attn_dropout=0.1, ff_dropout=0.1).to(DEV)
    cw = CoarseTransformerWrapper(transformer=m, codec=_Codec(), unique_consecutive=False, mask_prob=0.0).train()
    opt = torch.optim.Adam(m.parameters(), lr=1e-3)
    sem_ids = torch.randint(0, 50, (2, 10), device=DEV)
    loss = cw(semantic_token_ids=sem_ids, coarse_token_ids=torch.randint(0, 64, (2, 4, 2), device=DEV),
              return_loss=True)
    loss.backward()
    assert torch.isfinite(loss) and torch.isfinite(m.coarse_logit_weights.grad).all()
    opt.step()
    out = cw.generate(semantic_token_ids=sem_ids, max_time_steps=3)
    assert out.shape == (2, 3, 2)


# ---- 7. no stored masks -------------------------------------------------------------------------------------------
def test_dropout_step_memory():
    x = torch.randn(4, 512, 256, device=DEV)
    peaks = []
    for p in (0.0, 0.1):
        from audiolm_pytorch_b200.transformer import Transformer

        torch.manual_seed(0)
        tr = Transformer(dim=256, depth=2, heads=4, attn_dropout=p, ff_dropout=p).to(DEV).train()
        tr(x).float().pow(2).mean().backward()       # warm-up: weight caches
        for prm in tr.parameters():
            prm.grad = None
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        tr(x).float().pow(2).mean().backward()
        torch.cuda.synchronize()
        peaks.append(torch.cuda.max_memory_allocated() - base)
        del tr
    assert abs(peaks[1] - peaks[0]) <= 0.01 * peaks[0], peaks
