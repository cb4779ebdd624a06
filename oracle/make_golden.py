"""Generate tests/golden/*.pt by running the REAL reference (via oracle/ref_import.py) — build container only.

    python -m oracle.make_golden            # writes fixtures and checks the functional oracle against them

Each fixture holds: constructor kwargs, the reference module's state_dict, seeded inputs, and the
reference's outputs (and, for the coarse model, loss + parameter gradients).  The same run asserts
that oracle/transformer.py and oracle/codec.py reproduce the reference outputs to fp32 round-off,
which is what pins the oracle (the reference ships no tests or golden vectors of its own).
"""
from __future__ import annotations

import sys
import warnings

import torch

from . import codec as oc
from . import golden, ref_import
from . import third_party as tp
from . import transformer as ot

GOLDEN = golden.GOLDEN
TOL = 2e-4


def perturb(module, seed):
    """move every parameter off its init so each code path (HC dynamic maps, LN gains...) matters."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in module.named_parameters():
            leaf = name.split(".")[-1]
            if leaf in ("dynamic_alpha_fn", "dynamic_beta_fn"):
                p.copy_(torch.randn(p.shape, generator=g) * 0.05)
            elif leaf in ("dynamic_alpha_scale", "dynamic_beta_scale"):
                p.fill_(0.3)
            elif leaf in ("static_alpha", "static_beta"):
                p.add_(torch.randn(p.shape, generator=g) * 0.1)
            elif leaf == "gamma":
                p.add_(torch.randn(p.shape, generator=g) * 0.1)
            elif "logit_weights" in name:
                p.mul_(0.2)


def rms_rel(a, b):
    return ((a.float() - b.float()).pow(2).mean().sqrt() / b.float().pow(2).mean().sqrt().clamp(min=1e-20)).item()


def clone_state(m):
    return {k: v.detach().clone() for k, v in m.state_dict().items()}


def check(name, a, b, tol=TOL):
    err = (a.float() - b.float()).abs().max().item()
    scale = max(1.0, b.float().abs().max().item())
    status = "ok" if err <= tol * scale else "MISMATCH"
    print(f"  [{status}] {name}: max abs err {err:.3e} (scale {scale:.2f})")
    if status != "ok":
        raise SystemExit(f"oracle does not reproduce the reference for {name}")



def bf16_noise(m, loss_fn, grads):
    """per-parameter RMS-relative deviation of the REFERENCE's own gradients when the same loss runs under bf16
    autocast (the trainers wrap every step in accelerator.autocast(), trainer.py:577, 946, 1241, 1545).  Stored next to
    the fp32 gradients so the GPU tests can bound the CUDA path (bf16 activations) by the reference's own bf16 noise on
    these tiny, cancellation-heavy problems instead of by a hand-picked constant."""
    m.zero_grad()
    with torch.autocast("cpu", dtype=torch.bfloat16):
        loss = loss_fn()
    loss.float().backward()
    out = {}
    for k, p in m.named_parameters():
        if p.grad is not None and k in grads:
            g = grads[k].float()
            out[k] = ((p.grad.float() - g).pow(2).mean().sqrt() / g.pow(2).mean().sqrt().clamp(min=1e-20)).item()
    m.zero_grad()
    return out


def golden_attend(ref):
    torch.manual_seed(11)
    b, h, n, d = 2, 4, 37, 64
    q, k, v = torch.randn(b, h, n, d), torch.randn(b, n, d), torch.randn(b, n, d)
    mask = torch.rand(b, n) > 0.2
    mask[:, 0] = True
    bias = torch.randn(h, n, n)
    out = {}
    math = ref.attend.Attend(causal=True, flash=False)
    flash = ref.attend.Attend(causal=True, flash=True)
    with torch.no_grad(), warnings.catch_warnings():
        warnings.simplefilter("ignore")
        out["math_masked"] = math(q, k, v, mask=mask)
        out["math_bias"] = math(q, k, v, mask=mask, attn_bias=bias)
        out["flash_masked"] = flash(q, k, v, mask=mask)
        out["math_causal"] = math(q, k, v)
        # cached-decode style: 5 new queries against all keys
        out["math_cached"] = math(q[:, :, -5:], k, v, mask=mask)
    print("attend:")
    check("attend masked", ot.attend(q, k, v, mask=mask), out["math_masked"])
    check("attend bias", ot.attend(q, k, v, mask=mask, attn_bias=bias), out["math_bias"])
    check("attend vs flash", ot.attend(q, k, v, mask=mask), out["flash_masked"])
    check("attend causal", ot.attend(q, k, v), out["math_causal"])
    check("attend cached", ot.attend(q[:, :, -5:], k, v, mask=mask), out["math_cached"])
    golden.save(dict(q=q, k=k, v=v, mask=mask, bias=bias, out=out), "attend.pt")


def golden_semantic(ref):
    torch.manual_seed(21)
    kw = dict(num_semantic_tokens=50, dim=64, depth=2, heads=2, flash_attn=True)
    m = ref.lm.SemanticTransformer(**kw).eval()
    perturb(m, 1)
    ids = torch.randint(0, 50, (2, 19))
    mask = ot.fcm_mask((2, 19), 0.15, torch.Generator().manual_seed(3))
    with torch.no_grad():
        logits = m(ids=ids)
        logits_masked = m(ids=ids, self_attn_mask=mask)
        # incremental decode with KV cache: feed the first 12 ids, then all 19 with the cache.
        # Done on the math path (flash_attn=False, rel_pos_bias=False; identical state_dict): with
        # flash_attn=True and no key mask the reference hands SDPA is_causal=True with q_len != k_len
        # (attend.py:75-94), which torch aligns TOP-LEFT, i.e. a cached new token would see key 0 only.
        # attend.py:134 (math path) and :82 (masked flash path) are right-aligned; that is the contract.
        m_math = ref.lm.SemanticTransformer(**{**kw, "flash_attn": False, "rel_pos_bias": False}).eval()
        m_math.load_state_dict(m.state_dict())
        l12, cache = m_math(ids=ids[:, :12], return_kv_cache=True)
        l_inc, cache2 = m_math(ids=ids, kv_cache=cache, return_kv_cache=True)
    st = clone_state(m)
    print("semantic:")
    hk = dict(heads=2, depth=2)
    check("logits", ot.semantic_forward(st, ids, **hk)[0], logits)
    check("logits masked", ot.semantic_forward(st, ids, self_attn_mask=mask, **hk)[0], logits_masked)
    o12, oc12 = ot.semantic_forward(st, ids[:, :12], **hk)
    check("kv cache tensor", oc12, cache)
    oinc, _ = ot.semantic_forward(st, ids, kv_cache=oc12, **hk)
    check("incremental logits", oinc, l_inc)
    check("incremental == full tail", l_inc, logits[:, 13:], tol=1e-3)
    # wrapper loss (train mode appends EOS; no dedup, no FCM so it is deterministic)
    w = ref.lm.SemanticTransformerWrapper(transformer=m, unique_consecutive=False, mask_prob=0.0).train()
    loss = w(semantic_token_ids=ids, return_loss=True)
    loss.backward()
    grads = {k: p.grad.detach().clone() for k, p in m.named_parameters() if p.grad is not None}
    noise = bf16_noise(m, lambda: w(semantic_token_ids=ids, return_loss=True), grads)
    labels = torch.cat((ids, torch.full((2, 1), 50)), dim=1)
    ol, _ = ot.semantic_forward(st, labels[:, :-1], **hk)
    check("wrapper loss", ot.cross_entropy(ol, labels), loss.detach())
    golden.save(dict(kwargs=kw, state=st, ids=ids, mask=mask, logits=logits, logits_masked=logits_masked,
                    cache12=cache, logits_inc=l_inc, loss=loss.detach(), grads=grads, bf16_noise=noise),
               "semantic.pt")


def golden_semantic_plain(ref):
    """num_residual_streams=1 (hyper-connections disabled -> plain Residual wrappers, audiolm_pytorch.py:446)."""
    torch.manual_seed(22)
    kw = dict(num_semantic_tokens=50, dim=64, depth=2, heads=2, flash_attn=True, num_residual_streams=1)
    m = ref.lm.SemanticTransformer(**kw).eval()
    perturb(m, 5)
    ids = torch.randint(0, 50, (2, 19))
    mask = ot.fcm_mask((2, 19), 0.15, torch.Generator().manual_seed(4))
    with torch.no_grad():
        logits = m(ids=ids)
        logits_masked = m(ids=ids, self_attn_mask=mask)
    st = clone_state(m)
    print("semantic (1 residual stream):")
    hk = dict(heads=2, depth=2, num_streams=1)
    check("logits", ot.semantic_forward(st, ids, **hk)[0], logits)
    check("logits masked", ot.semantic_forward(st, ids, self_attn_mask=mask, **hk)[0], logits_masked)
    w = ref.lm.SemanticTransformerWrapper(transformer=m, unique_consecutive=False, mask_prob=0.0).train()
    loss = w(semantic_token_ids=ids, return_loss=True)
    loss.backward()
    grads = {k: p.grad.detach().clone() for k, p in m.named_parameters() if p.grad is not None}
    noise = bf16_noise(m, lambda: w(semantic_token_ids=ids, return_loss=True), grads)
    golden.save(dict(kwargs=kw, state=st, ids=ids, mask=mask, logits=logits, logits_masked=logits_masked,
                    loss=loss.detach(), grads=grads, bf16_noise=noise), "semantic_plain.pt")


def golden_coarse(ref):
    torch.manual_seed(31)
    kw = dict(num_semantic_tokens=50, codebook_size=64, num_coarse_quantizers=3, dim=64, depth=2, heads=2,
              flash_attn=True)
    m = ref.lm.CoarseTransformer(**kw).eval()
    perturb(m, 2)
    sem = torch.randint(0, 50, (2, 10))
    coarse = torch.randint(0, 64, (2, 22))  # 7 frames * 3 + 1 -> remainder head path
    n_total = 1 + 10 + 1 + 22
    mask = ot.fcm_mask((2, n_total), 0.15, torch.Generator().manual_seed(5))
    with torch.no_grad():
        sl, cl = m(semantic_token_ids=sem, coarse_token_ids=coarse)
        slm, clm = m(semantic_token_ids=sem, coarse_token_ids=coarse, self_attn_mask=mask)
        m_math = ref.lm.CoarseTransformer(**{**kw, "flash_attn": False, "rel_pos_bias": False}).eval()
        m_math.load_state_dict(m.state_dict())  # math path for cached decode (see golden_semantic)
        (_, cl_a), (kv_a, emb_a) = m_math(semantic_token_ids=sem, coarse_token_ids=coarse[:, :9], return_cache=True,
                                          return_only_coarse_logits=True)
        (_, cl_b), (kv_b, emb_b) = m_math(semantic_token_ids=sem, coarse_token_ids=coarse[:, :10],
                                          return_cache=True, kv_cache=kv_a, embed_cache=emb_a,
                                          return_only_coarse_logits=True)
    with torch.no_grad(), torch.autocast("cpu", dtype=torch.bfloat16):
        sl16, cl16 = m(semantic_token_ids=sem, coarse_token_ids=coarse)   # the reference's own bf16-autocast logits
    logits_bf16_noise = (rms_rel(sl16, sl), rms_rel(cl16, cl))
    st = clone_state(m)
    hk = dict(heads=2, depth=2, codebook_size=64, num_coarse_quantizers=3)
    print("coarse:")
    (osl, ocl), _ = ot.coarse_forward(st, sem, coarse, **hk)
    check("semantic logits", osl, sl)
    check("coarse logits", ocl, cl)
    (oslm, oclm), _ = ot.coarse_forward(st, sem, coarse, self_attn_mask=mask, **hk)
    check("coarse logits masked", oclm, clm)
    (_, ocl_a), (okv_a, oemb_a) = ot.coarse_forward(st, sem, coarse[:, :9], return_only_coarse_logits=True, **hk)
    check("kv cache", okv_a, kv_a)
    (_, ocl_b), _ = ot.coarse_forward(st, sem, coarse[:, :10], kv_cache=okv_a, embed_cache=oemb_a,
                                      return_only_coarse_logits=True, **hk)
    check("cached coarse logits", ocl_b, cl_b)
    # training loss through the reference wrapper (needs a codec instance for its ctor only)
    ss = ref.ss.SoundStream(codebook_size=64, rq_num_quantizers=8, channels=4, use_local_attn=False, codebook_dim=32)
    w = ref.lm.CoarseTransformerWrapper(transformer=m, codec=ss, unique_consecutive=False, mask_prob=0.0).train()
    coarse_frames = coarse[:, :21]
    loss = w(semantic_token_ids=sem, coarse_token_ids=coarse_frames, return_loss=True)
    loss.backward()
    grads = {k: p.grad.detach().clone() for k, p in m.named_parameters() if p.grad is not None}
    noise = bf16_noise(m, lambda: w(semantic_token_ids=sem, coarse_token_ids=coarse_frames, return_loss=True), grads)
    # oracle restatement of the wrapper arithmetic (audiolm_pytorch.py:1785-1854)
    sem_l = torch.cat((sem, torch.full((2, 1), 50)), 1)
    co_l = torch.cat((coarse_frames, torch.full((2, 1), 64)), 1)
    wmask = torch.nn.functional.pad(sem_l != 50, (1, co_l.shape[1]), value=True)
    (wsl, wcl), _ = ot.coarse_forward(st, sem_l.masked_fill(sem_l == 50, 0), co_l[:, :-1], self_attn_mask=wmask, **hk)
    check("wrapper loss", ot.coarse_wrapper_loss(wsl, wcl, sem_l, co_l), loss.detach())
    golden.save(dict(kwargs=kw, state=st, sem=sem, coarse=coarse, mask=mask, sem_logits=sl, coarse_logits=cl,
                    sem_logits_masked=slm, coarse_logits_masked=clm, kv_a=kv_a, emb_a=emb_a, coarse_logits_b=cl_b,
                    loss=loss.detach(), grads=grads, bf16_noise=noise, logits_bf16_noise=logits_bf16_noise),
               "coarse.pt")


def golden_fine(ref):
    torch.manual_seed(41)
    kw = dict(num_coarse_quantizers=3, num_fine_quantizers=5, codebook_size=64, dim=64, depth=2, heads=2,
              flash_attn=True)
    m = ref.lm.FineTransformer(**kw).eval()
    perturb(m, 3)
    coarse = torch.randint(0, 64, (2, 12))
    coarse[1, -3:] = -1  # padded frame -> key mask path (:1175-1184)
    fine = torch.randint(0, 64, (2, 18))  # 3 frames * 5 + 3 -> remainder head path
    with torch.no_grad():
        cl, fl = m(coarse_token_ids=coarse, fine_token_ids=fine)
    st = clone_state(m)
    hk = dict(heads=2, depth=2, codebook_size=64, num_coarse_quantizers=3, num_fine_quantizers=5)
    print("fine:")
    (ocl, ofl), _ = ot.fine_forward(st, coarse, fine, **hk)
    check("coarse logits", ocl, cl)
    check("fine logits", ofl, fl)
    golden.save(dict(kwargs=kw, state=st, coarse=coarse, fine=fine, coarse_logits=cl, fine_logits=fl),
               "fine.pt")


def golden_relpos(ref):
    """flash_attn=False models: RelativePositionBias (semantic), + cross_attn_bias (coarse), 2-D pos_bias_mlp +
    null_pos_bias (fine) - SURVEY §8 row a7.  Forward, masked forward, cached decode step, CE loss gradients."""
    import torch.nn.functional as F
    out = {}
    print("relative position bias (flash_attn=False):")

    def ce(logits, labels):
        return F.cross_entropy(logits.transpose(1, 2), labels)

    def bias_perturb(m, seed):
        g = torch.Generator().manual_seed(seed)
        with torch.no_grad():
            for name, p in m.named_parameters():
                if name in ("cross_attn_bias", "null_pos_bias"):
                    p.copy_(torch.randn(p.shape, generator=g) * 0.5)
                elif "rel_pos_bias" in name or "pos_bias_mlp" in name:
                    p.add_(torch.randn(p.shape, generator=g) * 0.05)

    # ---- semantic ----
    torch.manual_seed(71)
    kw = dict(num_semantic_tokens=50, dim=64, depth=2, heads=2, flash_attn=False)
    m = ref.lm.SemanticTransformer(**kw).eval()
    perturb(m, 4)
    bias_perturb(m, 5)
    ids = torch.randint(0, 50, (2, 19))
    labels = torch.randint(0, 51, (2, 20))
    mask = ot.fcm_mask((2, 19), 0.15, torch.Generator().manual_seed(6))
    with torch.no_grad():
        lg = m(ids=ids)
        lgm = m(ids=ids, self_attn_mask=mask.clone())
        l12, cache = m(ids=ids[:, :12], return_kv_cache=True)
        inc, _ = m(ids=ids[:, :13], kv_cache=cache, return_kv_cache=True)
    m.zero_grad()
    loss = ce(m(ids=ids), labels)
    loss.backward()
    grads = {k: p.grad.detach().clone() for k, p in m.named_parameters() if p.grad is not None}
    noise = bf16_noise(m, lambda: ce(m(ids=ids).float(), labels), grads)
    st = clone_state(m)
    hk = dict(heads=2, depth=2)
    o, _ = ot.semantic_forward(st, ids, **hk)
    check("semantic logits", o, lg)
    om, _ = ot.semantic_forward(st, ids, self_attn_mask=mask, **hk)
    check("semantic logits masked", om, lgm)
    _, oc = ot.semantic_forward(st, ids[:, :12], **hk)
    oi, _ = ot.semantic_forward(st, ids[:, :13], kv_cache=oc, **hk)
    check("semantic cached step", oi, inc)
    check("semantic loss", ce(o, labels), loss.detach())
    out["semantic"] = dict(kwargs=kw, state=st, ids=ids, labels=labels, mask=mask, logits=lg, logits_masked=lgm,
                           logits_inc=inc, loss=loss.detach(), grads=grads, bf16_noise=noise)

    # ---- coarse ----
    torch.manual_seed(72)
    kw = dict(num_semantic_tokens=50, codebook_size=64, num_coarse_quantizers=3, dim=64, depth=2, heads=2,
              flash_attn=False)
    m = ref.lm.CoarseTransformer(**kw).eval()
    perturb(m, 6)
    bias_perturb(m, 7)
    sem = torch.randint(0, 50, (2, 10))
    coarse = torch.randint(0, 64, (2, 22))
    sem_labels = torch.randint(0, 51, (2, 10))
    coarse_labels = torch.randint(0, 65, (2, 23))
    with torch.no_grad():
        sl, cl = m(semantic_token_ids=sem, coarse_token_ids=coarse)
        (_, cl_a), (kv_a, emb_a) = m(semantic_token_ids=sem, coarse_token_ids=coarse[:, :9], return_cache=True,
                                     return_only_coarse_logits=True)
        (_, cl_b), _ = m(semantic_token_ids=sem, coarse_token_ids=coarse[:, :10], return_cache=True, kv_cache=kv_a,
                         embed_cache=emb_a, return_only_coarse_logits=True)
    m.zero_grad()
    sl2, cl2 = m(semantic_token_ids=sem, coarse_token_ids=coarse)
    loss = ce(sl2, sem_labels) + ce(cl2, coarse_labels)
    loss.backward()
    grads = {k: p.grad.detach().clone() for k, p in m.named_parameters() if p.grad is not None}

    def _loss():
        a, b_ = m(semantic_token_ids=sem, coarse_token_ids=coarse)
        return ce(a.float(), sem_labels) + ce(b_.float(), coarse_labels)
    noise = bf16_noise(m, _loss, grads)
    st = clone_state(m)
    hk = dict(heads=2, depth=2, codebook_size=64, num_coarse_quantizers=3)
    (osl, ocl), _ = ot.coarse_forward(st, sem, coarse, **hk)
    check("coarse: semantic logits", osl, sl)
    check("coarse: coarse logits", ocl, cl)
    (_, _), (okv_a, oemb_a) = ot.coarse_forward(st, sem, coarse[:, :9], return_only_coarse_logits=True, **hk)
    (_, ocl_b), _ = ot.coarse_forward(st, sem, coarse[:, :10], kv_cache=okv_a, embed_cache=oemb_a,
                                      return_only_coarse_logits=True, **hk)
    check("coarse cached step", ocl_b, cl_b)
    check("coarse loss", ce(osl, sem_labels) + ce(ocl, coarse_labels), loss.detach())
    out["coarse"] = dict(kwargs=kw, state=st, sem=sem, coarse=coarse, sem_labels=sem_labels,
                         coarse_labels=coarse_labels, sem_logits=sl, coarse_logits=cl, coarse_logits_b=cl_b,
                         loss=loss.detach(), grads=grads, bf16_noise=noise)

    # ---- fine ----
    torch.manual_seed(73)
    kw = dict(num_coarse_quantizers=3, num_fine_quantizers=5, codebook_size=64, dim=64, depth=2, heads=2,
              flash_attn=False)
    m = ref.lm.FineTransformer(**kw).eval()
    perturb(m, 8)
    bias_perturb(m, 9)
    coarse = torch.randint(0, 64, (2, 12))
    coarse[1, -3:] = -1
    fine = torch.randint(0, 64, (2, 18))
    c_labels = torch.randint(0, 64, (2, 12))
    f_labels = torch.randint(0, 64, (2, 19))
    with torch.no_grad():
        cl, fl = m(coarse_token_ids=coarse, fine_token_ids=fine)
        (_, fl_a), (kv_a, emb_a) = m(coarse_token_ids=coarse, fine_token_ids=fine[:, :7], return_cache=True,
                                     return_only_fine_logits=True)
        (_, fl_b), _ = m(coarse_token_ids=coarse, fine_token_ids=fine[:, :8], return_cache=True, kv_cache=kv_a,
                         embed_cache=emb_a, return_only_fine_logits=True)
    m.zero_grad()
    cl2, fl2 = m(coarse_token_ids=coarse, fine_token_ids=fine)
    loss = ce(cl2, c_labels) + ce(fl2, f_labels)
    loss.backward()
    grads = {k: p.grad.detach().clone() for k, p in m.named_parameters() if p.grad is not None}

    def _loss():
        a, b_ = m(coarse_token_ids=coarse, fine_token_ids=fine)
        return ce(a.float(), c_labels) + ce(b_.float(), f_labels)
    noise = bf16_noise(m, _loss, grads)
    st = clone_state(m)
    hk = dict(heads=2, depth=2, codebook_size=64, num_coarse_quantizers=3, num_fine_quantizers=5)
    (ocl, ofl), _ = ot.fine_forward(st, coarse, fine, **hk)
    check("fine: coarse logits", ocl, cl)
    check("fine: fine logits", ofl, fl)
    (_, _), (okv_a, oemb_a) = ot.fine_forward(st, coarse, fine[:, :7], return_only_fine_logits=True, **hk)
    (_, ofl_b), _ = ot.fine_forward(st, coarse, fine[:, :8], kv_cache=okv_a, embed_cache=oemb_a,
                                    return_only_fine_logits=True, **hk)
    check("fine cached step", ofl_b, fl_b)
    check("fine loss", ce(ocl, c_labels) + ce(ofl, f_labels), loss.detach())
    out["fine"] = dict(kwargs=kw, state=st, coarse=coarse, fine=fine, c_labels=c_labels, f_labels=f_labels,
                       coarse_logits=cl, fine_logits=fl, fine_logits_b=fl_b, loss=loss.detach(), grads=grads,
                       bf16_noise=noise)
    golden.save(out, "relpos.pt")


fixed_fcm = ot.fixed_fcm


def golden_wrappers(ref):
    """training wrappers with the paths the plain goldens skip: FineTransformerWrapper.forward(return_loss=True)
    (audiolm_pytorch.py:2041-2137), and Semantic / Coarse / Fine wrappers with the forgetful causal mask
    (mask_prob=0.15) and unique_consecutive=True (:1513-1567, 1742-1854).  Loss + every parameter gradient."""
    out = {}
    print("wrappers (FCM mask, unique_consecutive, fine loss):")
    ss = ref.ss.SoundStream(codebook_size=64, rq_num_quantizers=8, channels=4, use_local_attn=False, codebook_dim=32)
    saved = ref.lm.generate_mask_with_prob
    ref.lm.generate_mask_with_prob = fixed_fcm
    try:
        def grads_of(m):
            return {k: p.grad.detach().clone() for k, p in m.named_parameters() if p.grad is not None}

        # ---- fine wrapper: plain (mask_prob=0) and with FCM ----
        torch.manual_seed(81)
        kw = dict(num_coarse_quantizers=3, num_fine_quantizers=5, codebook_size=64, dim=64, depth=2, heads=2,
                  flash_attn=True)
        m = ref.lm.FineTransformer(**kw).train()
        perturb(m, 11)
        coarse = torch.randint(0, 64, (2, 4, 3))
        fine = torch.randint(0, 64, (2, 4, 5))
        st = clone_state(m)
        hk = dict(heads=2, depth=2, codebook_size=64, num_coarse_quantizers=3, num_fine_quantizers=5)
        res = {}
        for tag, mp in (("plain", 0.0), ("fcm", 0.15)):
            m.zero_grad()
            w = ref.lm.FineTransformerWrapper(transformer=m, codec=ss, mask_prob=mp).train()
            loss = w(coarse_token_ids=coarse, fine_token_ids=fine, return_loss=True)
            loss.backward()
            gr = grads_of(m)
            res[tag] = dict(loss=loss.detach(), grads=gr, bf16_noise=bf16_noise(
                m, lambda: w(coarse_token_ids=coarse, fine_token_ids=fine, return_loss=True), gr))
            c2, f2 = coarse.reshape(2, -1), fine.reshape(2, -1)
            mask = fixed_fcm((2, c2.shape[1] + f2.shape[1] - 1 + 2), mp) if mp > 0 else None
            (ocl, ofl), _ = ot.fine_forward(st, c2, f2[:, :-1], self_attn_mask=mask, **hk)
            n_c, n_f = ocl.shape[1], ofl.shape[1]
            ol = (ot.cross_entropy(ocl, c2) * n_c + ot.cross_entropy(ofl, f2) * n_f) / (n_c + n_f)
            check(f"fine wrapper loss ({tag})", ol, loss.detach())
        out["fine"] = dict(kwargs=kw, state=st, coarse=coarse, fine=fine, **{f"{t}_{k}": v for t, r in res.items()
                                                                                for k, v in r.items()})

        # ---- semantic wrapper: unique_consecutive=True + FCM ----
        torch.manual_seed(82)
        kw = dict(num_semantic_tokens=50, dim=64, depth=2, heads=2, flash_attn=True)
        m = ref.lm.SemanticTransformer(**kw).train()
        perturb(m, 12)
        ids = torch.randint(0, 50, (2, 24))
        ids[0, 3:7] = ids[0, 3]           # runs of repeated ids -> ragged rows after unique_consecutive
        ids[1, 10:12] = ids[1, 10]
        ids[1, 15:20] = ids[1, 15]
        w = ref.lm.SemanticTransformerWrapper(transformer=m, unique_consecutive=True, mask_prob=0.15).train()
        loss = w(semantic_token_ids=ids, return_loss=True)
        loss.backward()
        gr = grads_of(m)
        out["semantic"] = dict(kwargs=kw, state=clone_state(m), ids=ids, loss=loss.detach(), grads=gr,
                               bf16_noise=bf16_noise(m, lambda: w(semantic_token_ids=ids, return_loss=True), gr))

        # ---- coarse wrapper: unique_consecutive=True + FCM ----
        torch.manual_seed(83)
        kw = dict(num_semantic_tokens=50, codebook_size=64, num_coarse_quantizers=3, dim=64, depth=2, heads=2,
                  flash_attn=True)
        m = ref.lm.CoarseTransformer(**kw).train()
        perturb(m, 13)
        sem = torch.randint(0, 50, (2, 14))
        sem[0, 2:6] = sem[0, 2]
        sem[1, 8:10] = sem[1, 8]
        coarse = torch.randint(0, 64, (2, 7, 3))
        w = ref.lm.CoarseTransformerWrapper(transformer=m, codec=ss, unique_consecutive=True, mask_prob=0.15).train()
        loss = w(semantic_token_ids=sem, coarse_token_ids=coarse, return_loss=True)
        loss.backward()
        gr = grads_of(m)
        out["coarse"] = dict(kwargs=kw, state=clone_state(m), sem=sem, coarse=coarse, loss=loss.detach(), grads=gr,
                             bf16_noise=bf16_noise(m, lambda: w(semantic_token_ids=sem, coarse_token_ids=coarse,
                                                                return_loss=True), gr))
    finally:
        ref.lm.generate_mask_with_prob = saved
    golden.save(out, "wrappers.pt")


def golden_sampling(ref):
    torch.manual_seed(51)
    logits = torch.randn(4, 65) * 3
    filt = ref.lm.top_k(logits, thres=0.9)
    torch.manual_seed(52)
    ids = ref.lm.gumbel_sample(filt, temperature=1.0)
    torch.manual_seed(52)
    u = torch.zeros_like(filt).uniform_(0, 1)
    print("sampling:")
    check("top_k", ot.top_k_filter(logits).nan_to_num(neginf=-1e30), filt.nan_to_num(neginf=-1e30))
    assert torch.equal(ot.gumbel_argmax(ot.top_k_filter(logits), u), ids), "gumbel sample ids differ"
    print("  [ok] gumbel ids bit-exact")
    seq = torch.tensor([[3, 7, 64, 5, 64, 1], [1, 2, 3, 4, 5, 6]])
    masked = ref.lm.mask_out_after_eos_id(seq, 64, keep_eos=False)
    golden.save(dict(logits=logits, filtered=filt, uniform=u, ids=ids, seq=seq, seq_masked=masked),
               "sampling.pt")


def golden_soundstream(ref):
    torch.manual_seed(61)
    kw = dict(codebook_size=64, rq_num_quantizers=4, channels=4, use_local_attn=False, codebook_dim=32,
              target_sample_hz=24000)
    ss = ref.ss.SoundStream(**kw).eval()
    tp.seed_codebooks(ss.rq, seed=7, std=0.5)
    wave = torch.randn(2, 3200)
    with torch.no_grad():
        enc = ss.encoder(wave[:, None, :])
        quant, idx, _ = ss(wave, return_encoded=True)
        codes = ss.tokenize(wave)
        recon = ss(wave, return_recons_only=True)
        recon_idx = ss.decode_from_codebook_indices(idx)
    st = {k: v for k, v in clone_state(ss).items() if k.split(".")[0] in ("encoder", "decoder", "rq")}
    print("soundstream:")
    check("encoder", oc.encoder(ot.sub(st, "encoder"), wave[:, None, :]), enc)
    oq, oi = oc.soundstream_tokenize(st, wave)
    assert torch.equal(oi, idx), "rvq indices differ"
    print("  [ok] rvq indices bit-exact")
    check("quantized", oq, quant)
    check("decode from indices", oc.soundstream_decode_indices(st, idx), recon_idx)
    check("round trip (README.md:100-113)", recon_idx, recon, tol=1e-5)
    # per-layer conv goldens: every (k, stride, dilation) the codec uses + pad modes
    convs = {}
    torch.manual_seed(62)
    for name, (cin, cout, k, s, d) in dict(k7=(3, 5, 7, 1, 1), k7d3=(4, 4, 7, 1, 3), k7d9=(4, 4, 7, 1, 9),
                                           k1=(4, 6, 1, 1, 1), s2=(4, 8, 4, 2, 1), s4=(4, 8, 8, 4, 1),
                                           s5=(4, 8, 10, 5, 1), s8=(4, 8, 16, 8, 1), k3=(8, 4, 3, 1, 1)).items():
        for mode in ("reflect", "constant"):
            c = ref.ss.CausalConv1d(cin, cout, k, stride=s, dilation=d, pad_mode=mode)
            x = torch.randn(2, cin, 80)
            with torch.no_grad():
                y = c(x)
            check(f"conv {name}/{mode}", oc.causal_conv1d(x, c.conv.weight, c.conv.bias, s, d, mode), y)
            convs[f"{name}/{mode}"] = dict(x=x, w=c.conv.weight.detach(), b=c.conv.bias.detach(), stride=s,
                                           dilation=d, mode=mode, y=y)
    for s in (2, 4, 5, 8):
        c = ref.ss.CausalConvTranspose1d(6, 4, 2 * s, s)
        x = torch.randn(2, 6, 11)
        with torch.no_grad():
            y = c(x)
        check(f"convT s{s}", oc.causal_conv_transpose1d(x, c.conv.weight, c.conv.bias, s), y)
        convs[f"convT{s}"] = dict(x=x, w=c.conv.weight.detach(), b=c.conv.bias.detach(), stride=s, y=y)
    golden.save(dict(kwargs=kw, state=st, wave=wave, enc=enc, quant=quant, idx=idx, codes=codes, recon=recon,
                    convs=convs), "soundstream.pt")


def golden_local_attn(ref):
    """SoundStream with its default bottleneck (use_local_attn=True, soundstream.py:397-440, 545, 613, 832-833, 857-858):
    the reference's LocalTransformer over the restated local-attention package (oracle/third_party.py, PARITY UNPINNED
    upstream).  Small sizes: window 8, 30 frames -> 4 buckets with a ragged last one."""
    torch.manual_seed(91)
    kw = dict(codebook_size=64, rq_num_quantizers=4, channels=4, codebook_dim=32, attn_window_size=8,
              target_sample_hz=24000)
    ss = ref.ss.SoundStream(**kw).eval()
    tp.seed_codebooks(ss.rq, seed=7, std=0.5)
    g = torch.Generator().manual_seed(92)
    with torch.no_grad():
        for n_, p_ in ss.named_parameters():   # move the attention block off its init (gates, scales, norms)
            if "_attn." in n_ and p_.ndim == 1:
                p_.add_(torch.randn(p_.shape, generator=g) * 0.1)
    wave = torch.randn(2, 9600)
    h = torch.randn(2, 30, 32)
    with torch.no_grad():
        enc_attn_out = ss.encoder_attn(h)
        quant, idx, _ = ss(wave, return_encoded=True)
        recon = ss(wave, return_recons_only=True)
        recon_idx = ss.decode_from_codebook_indices(idx)
    st = {k: v for k, v in clone_state(ss).items()
          if k.split(".")[0] in ("encoder", "decoder", "rq", "encoder_attn", "decoder_attn")}
    print("local attention bottleneck:")
    check("round trip with decoder_attn (README.md:100-113)", recon_idx, recon, tol=1e-5)
    golden.save(dict(kwargs=kw, state=st, wave=wave, h=h, enc_attn_out=enc_attn_out, quant=quant, idx=idx, recon=recon),
               "local_attn.pt")


def main():
    GOLDEN.mkdir(parents=True, exist_ok=True)
    import random
    ref = ref_import.load()
    fns = (golden_attend, golden_semantic, golden_semantic_plain, golden_coarse, golden_fine, golden_relpos,
           golden_wrappers, golden_sampling, golden_soundstream, golden_local_attn)
    only = set(sys.argv[1:])
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for fn in fns:
            if only and fn.__name__.replace("golden_", "") not in only:
                continue
            # hyper-connections picks its initial stream with `random.randrange` (third_party.py:60): seed per fixture
            # so each file is reproducible on its own, whatever ran before it
            random.seed(20240607 + sum(map(ord, fn.__name__)))
            fn(ref)
    files = sorted(GOLDEN.glob("*.pt*"))
    print(f"wrote {len(files)} fixture files, {sum(p.stat().st_size for p in files) / 1e6:.2f} MB")


if __name__ == "__main__":
    sys.exit(main())
