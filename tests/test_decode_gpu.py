"""CUDA-graph decode engine (config C5): static-cache kernels vs the tile kernels, one-token stack step vs the
cached forward, graph replay vs eager."""

import pytest
import torch

from oracle import golden

pytestmark = pytest.mark.gpu
DEV = "cuda"
bf16 = torch.bfloat16


def rms_rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).pow(2).mean().sqrt() / b.pow(2).mean().sqrt().clamp(min=1e-12)).item()


@pytest.mark.parametrize("b,h,n,masked", [(1, 8, 1, False), (2, 8, 77, False), (3, 4, 300, True), (1, 8, 2047, False)])
def test_kv_append_and_decode_attention(b, h, n, masked):
    """append at a device-side position, then attend keys 0..len against the fp32 reference (attend.py:117-144)."""
    from audiolm_pytorch_b200 import ops

    torch.manual_seed(n)
    max_len = 2048
    kc = torch.zeros(b, max_len, 64, device=DEV, dtype=bf16)
    vc = torch.zeros_like(kc)
    hist = torch.randn(b, n, 128, device=DEV).to(bf16)
    kc[:, :n - 1] = hist[:, :n - 1, :64]
    vc[:, :n - 1] = hist[:, :n - 1, 64:]
    kc[:, n:] = float("nan")   # anything past the fill level must be ignored
    vc[:, n:] = float("nan")
    ln = torch.tensor([n - 1], device=DEV, dtype=torch.int32)
    ops.kv_append(hist[:, n - 1].contiguous(), kc, vc, ln)
    assert torch.equal(kc[:, :n], hist[:, :, :64]) and torch.equal(vc[:, :n], hist[:, :, 64:])
    q = torch.randn(b, h * 64, device=DEV).to(bf16)
    mask = None
    if masked:
        mask = torch.ones(b, max_len, device=DEV, dtype=torch.uint8)
        mask[:, 1:n:3] = 0
    o = ops.mqa_attn_decode(q, kc, vc, ln, heads=h, key_mask=mask)
    o1 = ops.mqa_attn_decode(q, kc, vc, ln, heads=h, key_mask=mask, splits=1)
    assert (o.float() - o1.float()).abs().max().item() <= 1e-2   # key-split (flash-decoding) == single pass
    qf = q.float().view(b, h, 1, 64)
    sim = torch.einsum("bhid,bjd->bhij", qf, hist[:, :, :64].float()) * 0.125
    if masked:
        sim = sim.masked_fill(mask[:, None, None, :n] == 0, -torch.finfo(torch.float32).max)
    ref = torch.einsum("bhij,bjd->bhid", sim.softmax(-1), hist[:, :, 64:].float()).reshape(b, h * 64)
    assert (o.float() - ref).abs().max().item() <= 2e-2 * max(1.0, ref.abs().max().item())


def _semantic_model():
    from audiolm_pytorch_b200.audiolm import SemanticTransformer

    g = golden.load("semantic.pt")
    m = SemanticTransformer(**g["kwargs"])
    m.load_state_dict(g["state"])
    return m.to(DEV).eval(), g["ids"].to(DEV)


def test_stack_decoder_step_matches_cached_forward():
    from audiolm_pytorch_b200.decode import StackDecoder

    m, ids = _semantic_model()
    with torch.no_grad():
        _, kv = m(ids=ids[:, :9], return_kv_cache=True)        # prompt: start token + 9 ids
        dec = StackDecoder(m.transformer, ids.shape[0], 64)
        dec.load_cache(kv)
        for t in range(9, 14):
            want, kv = m(ids=ids[:, :t + 1], kv_cache=kv, return_kv_cache=True)   # logits of the new position
            out = dec.step(m.semantic_embedding(ids[:, t]))
            got = m._heads.linear(out, m.to_logits.weight, m.to_logits.bias, "sem")
            assert rms_rel(got, want[:, -1]) < 1e-2, (t, rms_rel(got, want[:, -1]))
        assert int(dec.len.item()) == 15


def test_graph_replay_is_bitwise_equal_to_eager():
    from audiolm_pytorch_b200.decode import GraphedStep, StackDecoder

    m, ids = _semantic_model()
    with torch.no_grad():
        _, kv = m(ids=ids[:, :9], return_kv_cache=True)
        outs = []
        for use_graph in (False, True):
            dec = StackDecoder(m.transformer, ids.shape[0], 64)
            dec.load_cache(kv)
            x = torch.zeros(ids.shape[0], 64, device=DEV)
            y = torch.zeros(ids.shape[0], 64, device=DEV, dtype=bf16)

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


def test_semantic_generate_uses_engine_and_respects_eos():
    from audiolm_pytorch_b200 import audiolm
    from audiolm_pytorch_b200.audiolm import SemanticTransformerWrapper

    m, ids = _semantic_model()
    w = SemanticTransformerWrapper(transformer=m, unique_consecutive=False)
    torch.manual_seed(3)
    out = w.generate(max_length=40, prime_ids=ids[:, :5])
    assert out.shape[0] == ids.shape[0] and 5 < out.shape[1] <= 40
    assert torch.equal(out[:, :5], ids[:, :5])
    assert ((out >= -1) & (out < m.num_semantic_tokens)).all()      # eos itself is masked out (keep_eos=False)
    assert getattr(w, "_engine", None) is not None and w._engine[1]._graphs   # the captured graph was used
    audiolm.USE_DECODE_GRAPHS = False
    try:
        w._engine = None
        out2 = w.generate(max_length=40, prime_ids=ids[:, :5])
        assert out2.shape[0] == ids.shape[0] and ((out2 >= -1) & (out2 < m.num_semantic_tokens)).all()
    finally:
        audiolm.USE_DECODE_GRAPHS = True


def test_gemv_matches_gemm():
    from audiolm_pytorch_b200 import ops

    torch.manual_seed(1)
    for rows, N, K in [(1, 512, 1024), (3, 5472, 1024), (8, 1024, 2730), (2, 501, 64)]:
        Kp = (K + 7) // 8 * 8
        x = torch.randn(rows, K, device=DEV).to(bf16)
        w = torch.zeros(N, Kp, device=DEV, dtype=bf16)
        w[:, :K] = (torch.randn(N, K, device=DEV) * 0.05).to(bf16)
        bias = torch.randn(N, device=DEV)
        y = ops.gemv(x, w, out_dtype=torch.float32, bias=bias)
        ref = x.float() @ w[:, :K].float().t() + bias
        assert (y - ref).abs().max().item() <= 2e-3 * max(1.0, ref.abs().max().item())
        yb = ops.gemv(x, w)
        assert (yb.float() - (ref - bias)).abs().max().item() <= 2e-2 * max(1.0, ref.abs().max().item())


def test_coarse_and_fine_generate_on_engine_match_slow_path_statistics():
    """the engine path produces tokens from the same distribution machinery as the slow cached path: with the
    sampler forced to argmax (temperature -> tiny) both paths must emit the same token ids."""
    from audiolm_pytorch_b200 import audiolm
    from audiolm_pytorch_b200.audiolm import (CoarseTransformer, CoarseTransformerWrapper, FineTransformer,
                                              FineTransformerWrapper)

    class _Codec:
        rq_groups = 1
        num_quantizers = 8

    g = golden.load("coarse.pt")
    m = CoarseTransformer(**g["kwargs"])
    m.load_state_dict(g["state"])
    m = m.to(DEV).eval()
    w = CoarseTransformerWrapper(transformer=m, codec=_Codec(), unique_consecutive=False)
    sem = g["sem"].to(DEV)
    kw = dict(semantic_token_ids=sem, max_time_steps=4, temperature=1e-4, filter_thres=0.0)
    fast = w.generate(**kw)
    assert getattr(w, "_engine", None) is not None and len(w._engine[1]._graphs) == 3
    slow = w.generate(use_kv_cache=False, **kw)
    assert fast.shape == slow.shape == (2, 4, 3)
    assert (fast == slow).float().mean().item() > 0.9   # argmax ties / bf16 noise may flip an occasional id

    g = golden.load("fine.pt")
    f = FineTransformer(**g["kwargs"])
    f.load_state_dict(g["state"])
    f = f.to(DEV).eval()
    fw = FineTransformerWrapper(transformer=f, codec=_Codec())
    coarse = g["coarse"].to(DEV)
    fast = fw.generate(coarse_token_ids=coarse.view(2, 4, 3), temperature=1e-4, filter_thres=0.0)
    slow = fw.generate(coarse_token_ids=coarse.view(2, 4, 3), temperature=1e-4, filter_thres=0.0, use_kv_cache=False)
    assert fast.shape == slow.shape == (2, 4, 5)
    assert (fast == slow).float().mean().item() > 0.9


@pytest.mark.parametrize("b,d,heads,depth,n0", [(1, 1024, 8, 2, 300), (3, 256, 4, 3, 37), (4, 1024, 8, 1, 2040),
                                               (2, 64, 2, 2, 0)])
def test_fused_stack_step_matches_multi_kernel_step(b, d, heads, depth, n0):
    """alm_decode_stack_step (one cooperative kernel per token) vs the multi-kernel step it replaces: same outputs,
    same rows appended to the cache, same fill level; its device-wide barriers never time out."""
    from audiolm_pytorch_b200 import decode
    from audiolm_pytorch_b200.transformer import Transformer

    torch.manual_seed(d + b)
    tr = Transformer(dim=d, depth=depth, heads=heads, flash_attn=True).to(DEV).eval()
    with torch.no_grad():
        for name, p in tr.named_parameters():
            if "dynamic_alpha_fn" in name or "dynamic_beta_fn" in name:
                p.normal_(0, 0.05)
            elif name.endswith("_scale"):
                p.fill_(0.3)
            elif "gamma" in name:
                p.add_(torch.randn_like(p) * 0.1)
    max_len = 2048
    kv = torch.randn(depth, 2, b, n0, 64, device=DEV)
    mask = torch.rand(b, n0, device=DEV) > 0.2
    if n0:
        mask[:, 0] = True
    xs = torch.randn(3, b, d, device=DEV)
    res = []
    default = decode.FUSED_STACK_STEP
    for fused in (False, True):
        decode.FUSED_STACK_STEP = fused
        try:
            dec = decode.StackDecoder(tr, b, max_len)
            assert dec.fused_ok() == fused
            dec.load_cache(kv)
            dec.set_key_mask(mask)
            outs = [dec.step(xs[t]).clone() for t in range(3)]
            torch.cuda.synchronize()
            assert int(dec.len.item()) == n0 + 3
            assert dec.barrier_timeouts() == 0
            res.append((torch.stack(outs), dec.kc[:, :, n0:n0 + 3].clone(), dec.vc[:, :, n0:n0 + 3].clone()))
        finally:
            decode.FUSED_STACK_STEP = default
    (o0, k0, v0), (o1, k1, v1) = res
    assert torch.isfinite(o1.float()).all()
    assert rms_rel(o1, o0) < 2e-2, rms_rel(o1, o0)
    assert rms_rel(k1, k0) < 2e-2 and rms_rel(v1, v0) < 2e-2, (rms_rel(k1, k0), rms_rel(v1, v0))
