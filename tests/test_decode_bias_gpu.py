"""Decode engine for relative-position-bias (flash_attn=False) and plain-stream (num_residual_streams=1) models:
decode attention with a score bias, the bias-row kernel, the one-token step against the cached forward and the fp32
oracle, graph replay, and generate() on the engine."""

import pytest
import torch

from oracle import golden

pytestmark = pytest.mark.gpu
DEV = "cuda"
bf16 = torch.bfloat16


class _Codec:
    rq_groups = 1
    num_quantizers = 8


def rms_rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).pow(2).mean().sqrt() / b.pow(2).mean().sqrt().clamp(min=1e-12)).item()


@pytest.mark.parametrize("b,h,n,masked", [(1, 8, 1, False), (2, 8, 77, False), (3, 4, 300, True), (1, 8, 2047, False),
                                          (2, 8, 2047, True)])
def test_decode_attention_with_bias(b, h, n, masked):
    """softmax(q k^T scale + bias[h, j]) v over keys 0..len against fp32 (attend.py:117-144); everything past the fill
    level (cache rows and bias entries) is NaN and must be ignored; single pass == key-split."""
    from audiolm_pytorch_b200 import ops

    torch.manual_seed(n + b)
    max_len = 2048
    kc = torch.full((b, max_len, 64), float("nan"), device=DEV, dtype=bf16)
    vc = torch.full_like(kc, float("nan"))
    hist = torch.randn(b, n, 128, device=DEV).to(bf16)
    kc[:, :n] = hist[:, :, :64]
    vc[:, :n] = hist[:, :, 64:]
    ln = torch.tensor([n - 1], device=DEV, dtype=torch.int32)
    bias = torch.full((h, max_len), float("nan"), device=DEV)
    bias[:, :n] = torch.randn(h, n, device=DEV) * 2.0
    q = torch.randn(b, h * 64, device=DEV).to(bf16)
    mask = None
    if masked:
        mask = torch.ones(b, max_len, device=DEV, dtype=torch.uint8)
        mask[:, 1:n:3] = 0
    o = ops.mqa_attn_decode(q, kc, vc, ln, heads=h, key_mask=mask, bias=bias)
    o1 = ops.mqa_attn_decode(q, kc, vc, ln, heads=h, key_mask=mask, bias=bias, splits=1)
    assert torch.isfinite(o.float()).all() and torch.isfinite(o1.float()).all()
    assert (o.float() - o1.float()).abs().max().item() <= 1e-2   # key-split (flash-decoding) == single pass
    qf = q.float().view(b, h, 1, 64)
    sim = torch.einsum("bhid,bjd->bhij", qf, hist[:, :, :64].float()) * 0.125 + bias[None, :, None, :n]
    if masked:
        sim = sim.masked_fill(mask[:, None, None, :n] == 0, -torch.finfo(torch.float32).max)
    ref = torch.einsum("bhij,bjd->bhid", sim.softmax(-1), hist[:, :, 64:].float()).reshape(b, h * 64)
    for got in (o, o1):
        assert (got.float() - ref).abs().max().item() <= 2e-2 * max(1.0, ref.abs().max().item())
    # the bias changes the result (a zero bias row reproduces the bias-free kernel bit for bit)
    zero = torch.zeros(h, max_len, device=DEV)
    assert torch.equal(ops.mqa_attn_decode(q, kc, vc, ln, heads=h, key_mask=mask, bias=zero),
                       ops.mqa_attn_decode(q, kc, vc, ln, heads=h, key_mask=mask))


def _rules(max_len):
    """(name, u, cls, c, table rows) for the three models' bias rules (CPU-built coordinates)"""
    from audiolm_pytorch_b200.audiolm import CoarseTransformer, FineTransformer, SemanticTransformer

    kw = dict(dim=32, depth=1, heads=4)
    out = []
    s = SemanticTransformer(num_semantic_tokens=20, **kw)
    out.append(("semantic", *s.decode_bias_coords(max_len), 2 * max_len - 1))
    c = CoarseTransformer(num_semantic_tokens=20, codebook_size=16, num_coarse_quantizers=3, **kw)
    out.append(("coarse", *c.decode_bias_coords(37, max_len), 2 * max_len - 1))
    f = FineTransformer(num_coarse_quantizers=3, num_fine_quantizers=5, codebook_size=16, **kw)
    u, cls, cc = f.decode_bias_coords(151, 50 * 5, max_len)
    _, mlp_in = f._pos_bias_index(151, 50 * 5, "cpu")
    out.append(("fine", u, cls, cc, mlp_in.shape[0]))
    return out


def test_bias_row_kernel_matches_host_gather():
    from audiolm_pytorch_b200 import ops

    torch.manual_seed(2)
    H, max_len = 4, 512
    for name, u, cls, c, rows in _rules(max_len):
        table = torch.randn(rows, H, device=DEV)
        for override in (torch.randn(H, device=DEV), None):
            uu, cc_ = u.to(DEV), cls.to(DEV)
            fill = [0, 1, 37, 38, 39, 150, 152, 300, 403] if name == "fine" else [0, 1, 37, 38, 39, 300, 511]
            for L in fill:
                out = torch.full((H, max_len), 12345.0, device=DEV)
                ops.decode_bias_row(table, override, uu, cc_, c, torch.tensor([L], device=DEV, dtype=torch.int32), out)
                ul, cl = u.long(), cls.long()
                idx = ul[L] - ul[:L + 1] + c
                over = (cl[:L + 1] != cl[L]) | (cl[L] < 0)
                assert ((idx >= 0) & (idx < rows) | over).all()
                ov = torch.zeros(H, device=DEV) if override is None else override
                ref = torch.where(over.to(DEV)[None], ov[:, None], table[idx.clamp(0, rows - 1).to(DEV)].t())
                assert torch.equal(out[:, :L + 1], ref), (name, L)
                assert (out[:, L + 1:] == 12345.0).all(), (name, L)    # nothing past the fill level is written


def _model(fixture, cls_name, key=None):
    from audiolm_pytorch_b200 import audiolm

    g = golden.load(fixture)
    g = g[key] if key else g
    m = getattr(audiolm, cls_name)(**g["kwargs"])
    m.load_state_dict(g["state"])
    return m.to(DEV).eval(), g


def _oracle_kw(g):
    return dict(heads=g["kwargs"]["heads"], depth=g["kwargs"]["depth"],
                num_streams=g["kwargs"].get("num_residual_streams", 4))


def _semantic_case(fixture, key):
    from oracle import transformer as ot

    m, g = _model(fixture, "SemanticTransformer", key)
    ids = g["ids"].to(DEV)
    b, max_len = ids.shape[0], 64
    with torch.no_grad():
        oracle = ot.semantic_forward(g["state"], g["ids"], **_oracle_kw(g))[0][:, 1:]   # [b, t] follows ids[:, t]

    def prefill(n):
        _, kv = m(ids=ids[:, :n], return_kv_cache=True)
        return kv

    def want(t, kv):
        lg, kv = m(ids=ids[:, :t + 1], kv_cache=kv, return_kv_cache=True)
        return lg[:, -1], kv

    def feed(t):
        return m.semantic_embedding(ids[:, t])

    def head(out, t):
        return m._heads.linear(out, m.to_logits.weight, m.to_logits.bias, "sem")

    return m, b, max_len, prefill, want, feed, head, m.decode_bias(max_len), None, range(9, ids.shape[1]), oracle


def _coarse_case():
    from oracle import transformer as ot

    m, g = _model("relpos.pt", "CoarseTransformer", "coarse")
    sem, coarse = g["sem"].to(DEV), g["coarse"].to(DEV)
    b, max_len, q, cb = sem.shape[0], 64, m.num_coarse_quantizers, m.codebook_size
    with torch.no_grad():
        (_, oracle), _ = ot.coarse_forward(g["state"], g["sem"], g["coarse"], codebook_size=cb,
                                           num_coarse_quantizers=q, **_oracle_kw(g))
    oracle = oracle[:, 1:]
    kw = dict(semantic_token_ids=sem, return_cache=True, return_only_coarse_logits=True)

    def prefill(n):
        _, (kv, emb) = m(coarse_token_ids=coarse[:, :n], **kw)
        return kv, emb

    def want(t, cache):
        (_, cl), cache = m(coarse_token_ids=coarse[:, :t + 1], kv_cache=cache[0], embed_cache=cache[1], **kw)
        return cl[:, -1], cache

    def feed(t):
        qi = t % q
        return m.coarse_embedding(coarse[:, t] + qi * cb) + m.coarse_quantize_embedding.weight[qi]

    def head(out, t):
        qn = (t + 1) % q
        return m._heads.linear_decode(out, m.coarse_logit_weights[qn], None, ("coarse", qn))

    bias = m.decode_bias(sem.shape[1], max_len)
    return m, b, max_len, prefill, want, feed, head, bias, None, range(9, coarse.shape[1]), oracle


def _fine_case():
    import torch.nn.functional as F

    from oracle import transformer as ot

    m, g = _model("relpos.pt", "FineTransformer", "fine")
    coarse, fine = g["coarse"].to(DEV), g["fine"].to(DEV)
    b, max_len, qc, qf, cb = coarse.shape[0], 64, m.num_coarse_quantizers, m.num_fine_quantizers, m.codebook_size
    with torch.no_grad():
        (_, oracle), _ = ot.fine_forward(g["state"], g["coarse"], g["fine"], codebook_size=cb,
                                         num_coarse_quantizers=qc, num_fine_quantizers=qf, **_oracle_kw(g))
    oracle = oracle[:, 1:]
    kw = dict(coarse_token_ids=coarse, return_cache=True, return_only_fine_logits=True)

    def prefill(n):
        _, (kv, emb) = m(fine_token_ids=fine[:, :n], **kw)
        return kv, emb

    def want(t, cache):
        (_, fl), cache = m(fine_token_ids=fine[:, :t + 1], kv_cache=cache[0], embed_cache=cache[1], **kw)
        return fl[:, -1], cache

    def feed(t):
        qi = t % qf
        return m.fine_embedding(fine[:, t] + qi * cb) + m.fine_quantize_embedding.weight[qi]

    def head(out, t):
        qn = (t + 1) % qf
        return m._heads.linear_decode(out, m.fine_logit_weights[qn], None, ("fine", qn))

    n = coarse.shape[1]
    bias = m.decode_bias(n, -(-n // qc) * qf, max_len)
    keep = F.pad((coarse != m.pad_id) & (coarse != m.eos_id), (1, 0), value=True)
    return m, b, max_len, prefill, want, feed, head, bias, keep, range(7, fine.shape[1]), oracle


CASES = {
    "semantic_relpos": lambda: _semantic_case("relpos.pt", "semantic"),
    "coarse_relpos": _coarse_case,
    "fine_relpos": _fine_case,
    "semantic_plain": lambda: _semantic_case("semantic_plain.pt", None),
}


@pytest.mark.parametrize("case", list(CASES))
def test_stack_decoder_step_matches_cached_forward(case):
    """teacher-forced: each engine step + head against Transformer.forward(..., kv_cache=...) on the same prefix.

    Both are bf16 paths; on these d=64 toy weights their distance from the fp32 oracle reaches ~1e-2 at some steps,
    so a step may exceed 1e-2 by as much as 1.5x the cached forward's own distance from the oracle at that step;
    over the whole window the engine must be as close to the oracle as the cached forward (within 1.3x)."""
    from audiolm_pytorch_b200.decode import StackDecoder

    m, b, max_len, prefill, want, feed, head, bias, keep, window, oracle = CASES[case]()
    assert (bias is None) == (case == "semantic_plain")
    with torch.no_grad():
        cache = prefill(window[0])
        kv = cache[0] if isinstance(cache, tuple) else cache
        dec = StackDecoder(m.transformer, b, max_len)
        dec.load_cache(kv)
        dec.set_key_mask(keep)
        if bias is not None:
            dec.set_bias(*bias)
        n0 = dec.host_len
        gots, refs = [], []
        for t in window:
            ref, cache = want(t, cache)
            got = head(dec.step(feed(t)), t)
            floor = rms_rel(ref, oracle[:, t])
            print(case, t, "engine vs cached forward", rms_rel(got, ref), "cached forward vs oracle", floor)
            assert rms_rel(got, ref) < max(1e-2, 1.5 * floor), (case, t, rms_rel(got, ref), floor)
            gots.append(got)
            refs.append(ref)
        assert int(dec.len.item()) == n0 + len(window)
    o = oracle[:, list(window)].transpose(0, 1)
    e_engine, e_dense = rms_rel(torch.stack(gots), o), rms_rel(torch.stack(refs), o)
    print(case, "window vs oracle: engine", e_engine, "cached forward", e_dense)
    assert e_engine < max(1e-2, 1.3 * e_dense), (e_engine, e_dense)


def test_coarse_engine_vs_fp32_oracle_with_key_splits():
    """d256 L2 h4 with cross_attn_bias, 302 cached positions (the decode attention splits its keys): teacher-forced
    engine logits against the fp32 oracle on the full sequence (same bound as the dense path on these weights)"""
    from audiolm_pytorch_b200.audiolm import CoarseTransformer
    from audiolm_pytorch_b200.decode import StackDecoder
    from oracle import transformer as ot

    torch.manual_seed(11)
    kw = dict(num_semantic_tokens=100, codebook_size=128, num_coarse_quantizers=3, dim=256, depth=2, heads=4)
    m = CoarseTransformer(**kw)
    with torch.no_grad():
        m.cross_attn_bias.normal_(0, 0.5)
        for n_, p in m.named_parameters():
            if "dynamic_alpha_fn" in n_ or "dynamic_beta_fn" in n_:
                p.normal_(0, 0.02)
            if "logit_weights" in n_:
                p.mul_(0.1)
    st = {k: v.detach().clone() for k, v in m.state_dict().items()}
    b, S, n0, n1 = 2, 200, 100, 130
    sem, coarse = torch.randint(0, 100, (b, S)), torch.randint(0, 128, (b, n1))
    with torch.no_grad():
        (_, ocl), _ = ot.coarse_forward(st, sem, coarse, heads=4, depth=2, codebook_size=128, num_coarse_quantizers=3)
    m = m.to(DEV).eval()
    semd, coarsed = sem.to(DEV), coarse.to(DEV)
    max_len = 512
    with torch.no_grad():
        _, (kv, _) = m(semantic_token_ids=semd, coarse_token_ids=coarsed[:, :n0], return_cache=True,
                       return_only_coarse_logits=True)
        dec = StackDecoder(m.transformer, b, max_len)
        dec.load_cache(kv)
        dec.set_bias(*m.decode_bias(S, max_len))
        assert dec.host_len == S + 2 + n0 >= 300
        got, ref = [], []
        for t in range(n0, n1 - 1):
            qi, qn = t % 3, (t + 1) % 3
            x = m.coarse_embedding(coarsed[:, t] + qi * 128) + m.coarse_quantize_embedding.weight[qi]
            out = dec.step(x)
            got.append(m._heads.linear_decode(out, m.coarse_logit_weights[qn], None, ("coarse", qn)))
            ref.append(ocl[:, t + 1])
    err = rms_rel(torch.stack(got), torch.stack(ref))
    print("engine vs oracle", err)
    assert err < 1e-2, err


@pytest.mark.parametrize("fixture,key", [("relpos.pt", "semantic"), ("semantic_plain.pt", None)])
def test_graph_replay_is_bitwise_equal_to_eager(fixture, key):
    from audiolm_pytorch_b200.decode import GraphedStep, StackDecoder

    m, g = _model(fixture, "SemanticTransformer", key)
    ids = g["ids"].to(DEV)
    b, max_len = ids.shape[0], 64
    with torch.no_grad():
        _, kv = m(ids=ids[:, :9], return_kv_cache=True)
        outs = []
        for use_graph in (False, True):
            dec = StackDecoder(m.transformer, b, max_len)
            dec.load_cache(kv)
            bias = m.decode_bias(max_len)
            if bias is not None:
                dec.set_bias(*bias)
            x = torch.zeros(b, m.transformer.dim, device=DEV)
            y = torch.zeros(b, m.transformer.dim, device=DEV, dtype=bf16)

            def fn():
                y.copy_(dec.step(x))

            step = GraphedStep(fn, [dec.len, y]) if use_graph else fn
            got = []
            for t in range(9, 15):
                x.copy_(m.semantic_embedding(ids[:, t]))
                step()
                got.append(y.clone())
            outs.append(torch.stack(got))
            assert int(dec.len.item()) == 16
    assert torch.equal(outs[0], outs[1])


def _check_eos_masked(out, vocab):
    """ids in [0, vocab) or -1 (EOS and everything after it is masked out, keep_eos=False), -1 only as a suffix"""
    assert ((out >= -1) & (out < vocab)).all()
    pad = (out == -1).int()
    assert (pad.cummax(dim=-1).values == pad).all()


def _check_argmax_agreement(seq, logits, start, tag):
    """argmax-mode tokens of the engine against what the uncached path (use_kv_cache=False: the full forward) picks
    on the same prefix.  logits [b, n, V]: row p of the full forward over seq[:, :p] scores seq[:, p] (EOS rule
    applied).  Comparing prefix by prefix keeps one argmax near-tie (the toy weights have top-2 gaps of a few 1e-3,
    below the bf16 noise of either path) from turning every later token of a free-running comparison into a
    mismatch.  >= 90 % must be the exact argmax, and every pick must be within the bf16 noise of the maximum."""
    seq = seq.reshape(seq.shape[0], -1)
    valid = (seq != -1)
    valid[:, :start] = False
    chosen = logits.gather(-1, seq.clamp(min=0)[..., None])[..., 0]
    top = logits.max(dim=-1).values
    exact = (logits.argmax(-1) == seq)[valid].float().mean().item()
    gap = (top - chosen)[valid]
    tol = 2e-2 * logits.abs().amax(-1)[valid]
    print(tag, "argmax agreement", exact, "largest gap", gap.max().item())
    assert valid.sum() > 0 and exact >= 0.9 and (gap <= tol).all(), (tag, exact, gap.max().item())


def _frame_eos_rule(logits, q):
    """EOS (the last class) only at a frame boundary after the first frame, as the samplers apply it"""
    p = torch.arange(logits.shape[1], device=logits.device)
    logits[:, (p % q != 0) | (p == 0), -1] = float("-inf")
    return logits


@pytest.mark.parametrize("fixture,key", [("relpos.pt", "semantic"), ("semantic_plain.pt", None)])
def test_semantic_generate_on_engine(fixture, key):
    from audiolm_pytorch_b200.audiolm import SemanticTransformerWrapper

    m, g = _model(fixture, "SemanticTransformer", key)
    ids = g["ids"].to(DEV)
    w = SemanticTransformerWrapper(transformer=m, unique_consecutive=False)
    torch.manual_seed(3)
    out = w.generate(max_length=40, prime_ids=ids[:, :5])
    assert w._engine[1]._graphs   # the captured graph was used
    assert torch.equal(out[:, :5], ids[:, :5]) and 5 < out.shape[1] <= 40
    _check_eos_masked(out, m.num_semantic_tokens)
    kw = dict(max_length=40, prime_ids=ids[:, :5], temperature=1e-4, filter_thres=0.0)
    fast = w.generate(**kw)
    slow = w.generate(use_kv_cache=False, **kw)
    n = min(fast.shape[1], slow.shape[1])
    print("free-running agreement", (fast[:, :n] == slow[:, :n]).float().mean().item())
    with torch.no_grad():
        lg = m(ids=fast[:, :-1].clamp(min=0)).float()
    _check_argmax_agreement(fast, lg, 5, fixture)


def test_coarse_and_fine_generate_on_engine():
    from audiolm_pytorch_b200.audiolm import CoarseTransformerWrapper, FineTransformerWrapper

    m, g = _model("relpos.pt", "CoarseTransformer", "coarse")
    w = CoarseTransformerWrapper(transformer=m, codec=_Codec(), unique_consecutive=False)
    sem = g["sem"].to(DEV)
    torch.manual_seed(4)
    out = w.generate(semantic_token_ids=sem, max_time_steps=6)
    assert len(w._engine[1]._graphs) == 3 and out.shape == (2, 6, 3)
    _check_eos_masked(out.reshape(2, -1), m.codebook_size)
    kw = dict(semantic_token_ids=sem, max_time_steps=4, temperature=1e-4, filter_thres=0.0)
    fast = w.generate(**kw)
    slow = w.generate(use_kv_cache=False, **kw)
    assert fast.shape == slow.shape == (2, 4, 3)
    print("coarse free-running agreement", (fast == slow).float().mean().item())
    with torch.no_grad():
        _, cl = m(semantic_token_ids=sem, coarse_token_ids=fast.reshape(2, -1)[:, :-1].clamp(min=0),
                  return_only_coarse_logits=True)
    _check_argmax_agreement(fast, _frame_eos_rule(cl.float(), 3), 0, "coarse")

    f, g = _model("relpos.pt", "FineTransformer", "fine")
    fw = FineTransformerWrapper(transformer=f, codec=_Codec())
    coarse = g["coarse"].to(DEV).view(2, 4, 3)
    out = fw.generate(coarse_token_ids=coarse)
    assert len(fw._engine[1]._graphs) == 5 and out.shape == (2, 4, 5)
    _check_eos_masked(out.reshape(2, -1), f.codebook_size)
    # primed with one fine frame: the engine starts mid-sequence
    out2 = fw.generate(coarse_token_ids=coarse, prime_fine_token_ids=g["fine"][:, :5].to(DEV))
    assert out2.shape == (2, 4, 5) and torch.equal(out2[:, 0], g["fine"][:, :5].to(DEV))
    fast = fw.generate(coarse_token_ids=coarse, temperature=1e-4, filter_thres=0.0)
    slow = fw.generate(coarse_token_ids=coarse, temperature=1e-4, filter_thres=0.0, use_kv_cache=False)
    assert fast.shape == slow.shape == (2, 4, 5)
    print("fine free-running agreement", (fast == slow).float().mean().item())
    with torch.no_grad():
        _, fl = f(coarse_token_ids=coarse.reshape(2, -1), fine_token_ids=fast.reshape(2, -1)[:, :-1].clamp(min=0),
                  return_only_fine_logits=True)
    _check_argmax_agreement(fast, _frame_eos_rule(fl.float(), 5), 0, "fine")
