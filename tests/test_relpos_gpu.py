"""flash_attn=False path on the GPU (SURVEY §8 a7): attention kernels with an additive bias (+ d bias), the
bias gather / scatter-add kernels, and the three transformers against the reference goldens and the oracle."""

import pytest
import torch
import torch.nn.functional as F

from oracle import golden

pytestmark = pytest.mark.gpu
DEV = "cuda"


def rms_rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).pow(2).mean().sqrt() / b.pow(2).mean().sqrt().clamp(min=1e-12)).item()


def max_rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-6)


def attend_ref(q, k, v, mask, bias, causal=True):
    """attend.py:117-144 (math path) in fp32; q [b,h,i,d], k/v [b,j,d], bias [h,i,j]."""
    sim = torch.einsum("bhid,bjd->bhij", q, k) * q.shape[-1] ** -0.5
    if bias is not None:
        sim = sim + bias
    neg = -torch.finfo(sim.dtype).max
    if mask is not None:
        sim = sim.masked_fill(~mask[:, None, None, :], neg)
    if causal:
        i, j = sim.shape[-2:]
        sim = sim.masked_fill(torch.ones(i, j, dtype=torch.bool, device=q.device).triu(j - i + 1), neg)
    return torch.einsum("bhij,bjd->bhid", sim.softmax(-1), v)


@pytest.mark.parametrize("b,h,n_q,n_k,masked", [(2, 2, 34, 34, False), (2, 8, 300, 300, True), (1, 8, 1024, 1024, False),
                                                (2, 4, 1, 77, False), (2, 4, 5, 133, True)])
def test_attention_with_bias_fwd_bwd(b, h, n_q, n_k, masked):
    from audiolm_pytorch_b200 import ops

    torch.manual_seed(n_q * 7 + n_k)
    q = torch.randn(b, n_q, h * 64, device=DEV).to(torch.bfloat16)
    k = torch.randn(b, n_k, 64, device=DEV).to(torch.bfloat16)
    v = torch.randn(b, n_k, 64, device=DEV).to(torch.bfloat16)
    ld = (n_k + 3) // 4 * 4
    bias_pad = torch.full((h, n_q, ld), float("nan"), device=DEV)   # pad columns must never be read into a result
    bias_pad[..., :n_k] = torch.randn(h, n_q, n_k, device=DEV) * 1.5
    mask = None
    if masked:
        mask = torch.rand(b, n_k, device=DEV) > 0.2
        mask[:, 0] = True
    o, lse = ops.mqa_attn_fwd(q, k, v, heads=h, key_mask=mask, causal=True, bias=bias_pad)
    # fp32 autograd reference on the same bf16-rounded inputs
    qf = q.float().view(b, n_q, h, 64).permute(0, 2, 1, 3).requires_grad_()
    kf, vf = k.float().requires_grad_(), v.float().requires_grad_()
    bf = bias_pad[..., :n_k].clone().requires_grad_()
    ref = attend_ref(qf, kf, vf, mask, bf).permute(0, 2, 1, 3).reshape(b, n_q, h * 64)
    assert (o.float() - ref).abs().max().item() <= 2e-2 * max(1.0, ref.abs().max().item())
    if n_q != n_k:
        return  # the backward is only used on full (training) sequences
    d_o = torch.randn_like(ref).to(torch.bfloat16)
    ref.backward(d_o.float())
    dbias = torch.zeros_like(bias_pad)
    dq, dk, dv = ops.mqa_attn_bwd(q, k, v, o, d_o, lse, heads=h, key_mask=mask, causal=True, bias=bias_pad, dbias=dbias)
    dq_ref = qf.grad.permute(0, 2, 1, 3).reshape(b, n_q, h * 64)
    # control: the same kernels without a bias against their own fp32 reference (bf16 P / dS staging noise)
    o0, lse0 = ops.mqa_attn_fwd(q, k, v, heads=h, key_mask=mask, causal=True)
    dq0, dk0, dv0 = ops.mqa_attn_bwd(q, k, v, o0, d_o, lse0, heads=h, key_mask=mask, causal=True)
    q0 = q.float().view(b, n_q, h, 64).permute(0, 2, 1, 3).requires_grad_()
    k0, v0 = k.float().requires_grad_(), v.float().requires_grad_()
    attend_ref(q0, k0, v0, mask, None).permute(0, 2, 1, 3).reshape(b, n_q, h * 64).backward(d_o.float())
    ctrl = rms_rel(dq0, q0.grad.permute(0, 2, 1, 3).reshape(b, n_q, h * 64))
    errs = dict(dq=rms_rel(dq, dq_ref), dk=rms_rel(dk, kf.grad), dv=rms_rel(dv, vf.grad),
                dbias=rms_rel(dbias[..., :n_k], bf.grad), dq_nobias_control=ctrl)
    print(errs)
    assert max_rel(dq, dq_ref) < 2e-2 and max_rel(dk, kf.grad) < 2e-2 and max_rel(dv, vf.grad) < 2e-2, errs
    assert max_rel(dbias[..., :n_k], bf.grad) < 2e-2, errs
    assert errs["dq"] < 5e-2 and errs["dk"] < 5e-2 and errs["dv"] < 5e-2 and errs["dbias"] < 5e-2, errs
    assert (dbias[..., n_k:] == 0).all()
    # accumulation semantics: a second call adds on top
    ops.mqa_attn_bwd(q, k, v, o, d_o, lse, heads=h, key_mask=mask, causal=True, bias=bias_pad, dbias=dbias)
    assert max_rel(dbias[..., :n_k], 2 * bf.grad) < 2e-2


def test_bias_gather_fwd_bwd():
    from audiolm_pytorch_b200 import ops

    torch.manual_seed(5)
    H, n_q, n_k, P = 8, 37, 50, 99
    table = torch.randn(P, H, device=DEV)
    over = torch.randn(H, device=DEV)
    idx = torch.randint(-1, P, (n_q, n_k), device=DEV, dtype=torch.int32)
    out = ops.bias_gather_fwd(table, idx, over)
    assert out.shape == (H, n_q, 52) and (out[..., n_k:] == 0).all()
    ref = torch.where((idx < 0)[None], over[:, None, None], table[idx.clamp(min=0).long()].permute(2, 0, 1))
    assert torch.equal(out[..., :n_k], ref)
    g = torch.randn(H, n_q, 52, device=DEV)
    dt, do = ops.bias_gather_bwd(g, idx, P, want_override=True)
    dt_ref = torch.zeros(P, H, device=DEV)
    gv = g[..., :n_k].permute(1, 2, 0).reshape(-1, H)
    flat = idx.reshape(-1).long()
    dt_ref.index_add_(0, flat.clamp(min=0), gv * (flat >= 0)[:, None])
    assert torch.allclose(dt, dt_ref, atol=1e-4)
    assert torch.allclose(do, (gv * (flat < 0)[:, None]).sum(0), atol=1e-4)


def _ce(lg, lb):
    from audiolm_pytorch_b200.heads import cross_entropy

    return cross_entropy(lg, lb)


def _check_grads(m, golden, tol=7e-2, noise=None):
    named = dict(m.named_parameters())
    kind_scale = {}
    for k, gr in golden.items():
        if gr.numel() <= 20:
            kind = k.split(".")[-1]
            kind_scale[kind] = max(kind_scale.get(kind, 0.0), gr.float().pow(2).mean().sqrt().item())
    bad = {}
    for k, gr in golden.items():
        assert named[k].grad is not None, k
        if gr.float().abs().max().item() < 1e-6:
            # e.g. the last bias of RelativePositionBias: a per-head constant shift leaves the softmax unchanged,
            # so the reference gradient is round-off; ours must be (absolutely) negligible too
            e, t = named[k].grad.float().abs().max().item(), 2e-3
        elif gr.numel() <= 20:
            e = (named[k].grad.float().cpu() - gr.float()).pow(2).mean().sqrt().item() / kind_scale[k.split(".")[-1]]
            t = 0.35
        else:
            e, t = rms_rel(named[k].grad, gr), max(tol, 2.0 * (noise or {}).get(k, 0.0))
        if e >= t:
            bad[k] = (e, t)
    assert not bad, bad


def test_semantic_rel_pos_bias_vs_reference_golden():
    from audiolm_pytorch_b200.audiolm import SemanticTransformer

    g = golden.load("relpos.pt")["semantic"]
    m = SemanticTransformer(**g["kwargs"])
    m.load_state_dict(g["state"])
    m = m.to(DEV).eval()
    ids = g["ids"].to(DEV)
    with torch.no_grad():
        lg = m(ids=ids)
        lgm = m(ids=ids, self_attn_mask=g["mask"].to(DEV))
        _, cache = m(ids=ids[:, :12], return_kv_cache=True)
        inc, _ = m(ids=ids[:, :13], kv_cache=cache, return_kv_cache=True)
    assert rms_rel(lg, g["logits"]) < 1e-2
    assert rms_rel(lgm, g["logits_masked"]) < 1e-2
    assert rms_rel(inc, g["logits_inc"]) < 1e-2
    m.zero_grad()
    loss = _ce(m(ids=ids), g["labels"].to(DEV))
    assert abs(loss.item() - g["loss"].item()) < 1e-2 * g["loss"].item()
    loss.backward()
    _check_grads(m, g["grads"], noise=g.get("bf16_noise"))


def test_coarse_rel_pos_bias_vs_reference_golden():
    from audiolm_pytorch_b200.audiolm import CoarseTransformer

    g = golden.load("relpos.pt")["coarse"]
    m = CoarseTransformer(**g["kwargs"])
    m.load_state_dict(g["state"])
    m = m.to(DEV).eval()
    sem, coarse = g["sem"].to(DEV), g["coarse"].to(DEV)
    with torch.no_grad():
        sl, cl = m(semantic_token_ids=sem, coarse_token_ids=coarse)
        (_, _), (kv_a, emb_a) = m(semantic_token_ids=sem, coarse_token_ids=coarse[:, :9], return_cache=True,
                                  return_only_coarse_logits=True)
        (_, cl_b), _ = m(semantic_token_ids=sem, coarse_token_ids=coarse[:, :10], return_cache=True, kv_cache=kv_a,
                         embed_cache=emb_a, return_only_coarse_logits=True)
    # control: the SAME weights on the flash path (no bias anywhere) against the oracle without the bias keys -
    # separates the bf16 noise floor of this d=64 toy model from anything the bias path adds
    from oracle import transformer as ot
    st_nb = {k: v for k, v in g["state"].items() if "rel_pos_bias" not in k and k != "cross_attn_bias"}
    m_nb = CoarseTransformer(**{**g["kwargs"], "flash_attn": True})
    m_nb.load_state_dict(st_nb)
    m_nb = m_nb.to(DEV).eval()
    with torch.no_grad():
        _, cl_nb = m_nb(semantic_token_ids=sem, coarse_token_ids=coarse)
    (_, ocl_nb), _ = ot.coarse_forward(st_nb, g["sem"], g["coarse"], heads=2, depth=2, codebook_size=64,
                                       num_coarse_quantizers=3)
    floor = rms_rel(cl_nb, ocl_nb)
    print("coarse relpos logits err", rms_rel(sl, g["sem_logits"]), rms_rel(cl, g["coarse_logits"]),
          rms_rel(cl_b, g["coarse_logits_b"]), "no-bias control (noise floor of these weights)", floor)
    assert rms_rel(sl, g["sem_logits"]) < 1e-2
    assert rms_rel(cl, g["coarse_logits"]) < max(1e-2, 1.3 * floor)
    assert rms_rel(cl_b, g["coarse_logits_b"]) < max(1e-2, 1.5 * floor)
    m.zero_grad()
    sl, cl = m(semantic_token_ids=sem, coarse_token_ids=coarse)
    loss = _ce(sl, g["sem_labels"].to(DEV)) + _ce(cl, g["coarse_labels"].to(DEV))
    assert abs(loss.item() - g["loss"].item()) < 1e-2 * g["loss"].item()
    loss.backward()
    # these weights sit at a 1.06e-2 forward noise floor (control above; the flash golden's is 0.76e-2), and the
    # gradient noise scales with it: 7e-2 * 1.06 / 0.76 ~ 0.1 -> 0.13.  The d=256 oracle test below keeps 7e-2.
    _check_grads(m, g["grads"], tol=0.13, noise=g.get("bf16_noise"))


def test_fine_rel_pos_bias_vs_reference_golden():
    from audiolm_pytorch_b200.audiolm import FineTransformer

    g = golden.load("relpos.pt")["fine"]
    m = FineTransformer(**g["kwargs"])
    m.load_state_dict(g["state"])
    m = m.to(DEV).eval()
    coarse, fine = g["coarse"].to(DEV), g["fine"].to(DEV)
    with torch.no_grad():
        cl, fl = m(coarse_token_ids=coarse, fine_token_ids=fine)
        (_, _), (kv_a, emb_a) = m(coarse_token_ids=coarse, fine_token_ids=fine[:, :7], return_cache=True,
                                  return_only_fine_logits=True)
        (_, fl_b), _ = m(coarse_token_ids=coarse, fine_token_ids=fine[:, :8], return_cache=True, kv_cache=kv_a,
                         embed_cache=emb_a, return_only_fine_logits=True)
    assert rms_rel(cl, g["coarse_logits"]) < 1e-2
    assert rms_rel(fl, g["fine_logits"]) < 1e-2
    assert rms_rel(fl_b, g["fine_logits_b"]) < 1e-2
    m.zero_grad()
    cl, fl = m(coarse_token_ids=coarse, fine_token_ids=fine)
    loss = _ce(cl, g["c_labels"].to(DEV)) + _ce(fl, g["f_labels"].to(DEV))
    assert abs(loss.item() - g["loss"].item()) < 1e-2 * g["loss"].item()
    loss.backward()
    _check_grads(m, g["grads"], noise=g.get("bf16_noise"))


def test_coarse_rel_pos_bias_larger_vs_oracle():
    """d256 L2 h4, 3 x 200 tokens: logits and the gradients of every bias parameter vs the fp32 oracle autograd."""
    from audiolm_pytorch_b200.audiolm import CoarseTransformer
    from oracle import transformer as ot

    torch.manual_seed(11)
    kw = dict(num_semantic_tokens=100, codebook_size=128, num_coarse_quantizers=3, dim=256, depth=2, heads=4)
    m = CoarseTransformer(**kw)  # flash_attn defaults to False -> rel_pos_bias + cross_attn_bias
    with torch.no_grad():
        m.cross_attn_bias.normal_(0, 0.5)
        for n_, p in m.named_parameters():
            if "dynamic_alpha_fn" in n_ or "dynamic_beta_fn" in n_:
                p.normal_(0, 0.02)
            if "logit_weights" in n_:
                p.mul_(0.1)
    st = {k: v.detach().clone().requires_grad_(v.is_floating_point()) for k, v in m.state_dict().items()}
    sem, coarse = torch.randint(0, 100, (3, 70)), torch.randint(0, 128, (3, 128))
    sl_l, cl_l = torch.randint(0, 101, (3, 70)), torch.randint(0, 129, (3, 129))
    (osl, ocl), _ = ot.coarse_forward(st, sem, coarse, heads=4, depth=2, codebook_size=128, num_coarse_quantizers=3)
    oloss = F.cross_entropy(osl.transpose(1, 2), sl_l) + F.cross_entropy(ocl.transpose(1, 2), cl_l)
    oloss.backward()
    m = m.to(DEV)
    sl, cl = m(semantic_token_ids=sem.to(DEV), coarse_token_ids=coarse.to(DEV))
    assert rms_rel(sl, osl.detach()) < 1e-2 and rms_rel(cl, ocl.detach()) < 1e-2
    loss = _ce(sl, sl_l.to(DEV)) + _ce(cl, cl_l.to(DEV))
    loss.backward()
    named = dict(m.named_parameters())
    for k in st:
        if "rel_pos_bias" in k or k == "cross_attn_bias":
            assert rms_rel(named[k].grad, st[k].grad) < 7e-2, (k, rms_rel(named[k].grad, st[k].grad))
