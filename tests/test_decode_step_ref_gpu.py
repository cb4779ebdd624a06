"""Decode engine (config C5): both one-token step paths - the one-kernel stack step (alm_decode_stack_step) and the
multi-kernel step - against the fp64 oracle of the cached forward, across the one-kernel step's envelope: weights
staged in shared memory or read from L2, one or several head passes, flash-decoding slice layouts, key masks, with and
without the value residual, up to 64 layers; shapes the one-kernel step refuses run on the multi-kernel step.

Every parameter, embedding and cached row is bf16-representable, so the reference sees exactly the engine's operands
and the error measured is the engine's own arithmetic (bf16 activations, fp32 accumulation)."""

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
bf16 = torch.bfloat16
f64 = torch.float64
MAX_LEN = 2048
STEPS = 3
KEYS_PER_SPLIT, MAX_SPLITS = 32, 16   # flash-decoding slices of csrc/decode_step.cu

# The one-kernel step may not be much worse than the multi-kernel step on the same vector (they round at the same
# points): its error must stay under RATIO x the multi-kernel step's, or under a third of the case's bound.
RATIO = 1.5


def case(b, d, heads, depth, n0, value_residual, mask, bound, *, id, streams=4, fused=True, dc=0.0):
    return pytest.param(b, d, heads, depth, n0, value_residual, mask, streams, fused, bound, dc, id=id)


# (b, d, heads, depth, n0 = cached positions before the first step, value residual, key mask, bound, streams,
# one-kernel step taken, DC offset added to every token vector).  `bound` caps the RMS-relative error of every vector checked (an output row, one layer's
# appended k or v row of one sequence) on both paths: about 3x the largest error either path showed in the case on an
# H100 SXM (132 SMs, 700 W power limit).  The 64-layer model is ill-conditioned: its fp64 forward already moves 15-25x
# as much as a bf16-sized change of its input, so both paths sit 0.1-0.4 from it and only gross errors show there.
CASES = [
    case(1, 1024, 8, 6, 600, True, "holes", 6e-2, id="c5-all-phases-staged"),
    case(4, 1024, 8, 2, 2045, True, "none", 2e-2, id="b4-w1-from-l2-16-slices-last-slot"),
    case(4, 1024, 64, 1, 100, True, "holes", 1.4e-2, id="h64-four-head-passes-out-w1-w2-from-l2"),
    case(2, 256, 24, 3, 95, False, "slice-blank", 2.8e-2, id="h24-partial-head-pass-no-value-residual-blank-slice"),
    *[case(3, 64, 3, 64, n0, True, "holes", 1.2, id=f"L64-h3-idle-warps-n{n0}") for n0 in (0, 31, 32, 33)],
    case(1, 256, 16, 2, 40, False, "all-cached", 1.7e-2, id="h16-every-cached-key-masked"),
    case(5, 64, 4, 2, 50, True, "holes", 1.8e-2, fused=False, id="b5-multi-kernel-gemv"),
    case(9, 64, 4, 2, 50, True, "holes", 1.7e-2, fused=False, id="b9-multi-kernel-gemm"),
    case(2, 64, 4, 2, 50, True, "holes", 1.2e-2, streams=1, fused=False, id="one-stream-multi-kernel"),
    case(2, 1024, 8, 1, 64, True, "holes", 1.2e-2, id="d1024-accepted"),
    case(2, 1280, 8, 1, 64, True, "holes", 1.1e-2, fused=False, id="d1280-refused-falls-back"),
    case(2, 1536, 8, 1, 64, True, "holes", 1.2e-2, fused=False, id="d1536-refused-falls-back"),
    # token vectors with a DC offset: the branch inputs' LayerNorms see mean / sigma of about dc.  Larger offsets drown
    # in the bf16 rounding of the residual streams (2^-9 dc per element), which both paths store and the oracle does not
    case(2, 1024, 8, 2, 64, True, "holes", 5.5e-2, dc=4.0, id="dc4-offset"),
    case(1, 256, 16, 3, 95, True, "holes", 5.6e-2, dc=16.0, id="dc16-offset"),
]


def _model(d, heads, depth, value_residual, streams):
    """random weights with the dynamic hyper-connection terms switched on.  The alpha scale stays at 0.1: at 0.3 the
    four stream weights of a branch input can nearly cancel, and the fp64 forward itself then amplifies a bf16-sized
    change of its input 10-20x at depth 2 (hundreds of times at depth 64), which no kernel error bound can separate
    from a bug."""
    from audiolm_pytorch_b200.transformer import Transformer

    tr = Transformer(dim=d, depth=depth, heads=heads, flash_attn=True, add_value_residual=value_residual,
                     num_residual_streams=streams)
    with torch.no_grad():
        for name, p in tr.named_parameters():
            if "dynamic_alpha_fn" in name or "dynamic_beta_fn" in name:
                p.normal_(0, 0.05)
            elif name.endswith("alpha_scale"):
                p.fill_(0.1)
            elif name.endswith("beta_scale"):
                p.fill_(0.3)
            elif "gamma" in name:
                p.add_(torch.randn_like(p) * 0.1)
            p.copy_(p.bfloat16().float())
    st = {k: v.detach().to(f64) for k, v in tr.state_dict().items()}
    return tr.to(DEV).eval(), st


def _slices(n_all, b):
    """[begin, end) of every flash-decoding slice the one-kernel step opens over n_all keys (decode_step.cu)"""
    from audiolm_pytorch_b200 import ops

    splits = min(max(1, min(MAX_SPLITS, ops.decode_stack_grid() // b)), max(1, -(-n_all // KEYS_PER_SPLIT)))
    chunk = (-(-n_all // splits) + 3) & ~3
    return [(s * chunk, min(n_all, (s + 1) * chunk)) for s in range(splits)]


def _key_mask(kind, b, n0):
    """bool [b, n0] (True = attend) over the cached keys, or None"""
    if kind == "none" or n0 == 0:
        return None
    mask = torch.rand(b, n0) > 0.2
    mask[:, 0] = True
    if kind == "all-cached":
        mask[:] = False
    elif kind == "slice-blank":   # row 0: one whole slice of every step blank; row 1: no holes
        mask[:] = True
        for t in range(STEPS):
            lo, hi = _slices(n0 + t + 1, b)[1]
            assert hi <= n0
            mask[0, lo:hi] = False
    return mask


def _rel_rows(got, want):
    """RMS-relative error of every vector along the last dimension"""
    got, want = got.to(f64).cpu(), want.to(f64).cpu()
    return (got - want).pow(2).mean(-1).sqrt() / want.pow(2).mean(-1).sqrt().clamp(min=1e-12)


def _reference(st, dec, x, n, *, heads, depth, streams, value_residual):
    """fp64 oracle of the cached forward for the token x [b, d] at position n over the engine's own cache rows [0, n)
    and key mask [0, n] -> (output [b, d], new k [depth, b, 64], new v [depth, b, 64])"""
    from oracle import transformer as ot

    b, d = x.shape
    xs = x.to(f64).cpu()[:, None].expand(b, n + 1, d)   # (only position n is read: the cache covers the others)
    kv = torch.stack((dec.kc[:, :, :n], dec.vc[:, :, :n]), dim=1).to(f64).cpu()
    out, cache = ot.transformer(st, xs, heads=heads, depth=depth, num_streams=streams,
                                self_attn_mask=dec.mask[:, :n + 1].bool().cpu(), kv_cache=kv,
                                add_value_residual=value_residual)
    return out[:, 0], cache[:, 0, :, n], cache[:, 1, :, n]


def _run_path(fused_flag, tr, st, b, n0, kv, mask, xs, ref_kw):
    """three consecutive steps on one path -> (fused_ok(), errors {quantity: [STEPS, ...]})"""
    from audiolm_pytorch_b200 import decode

    default = decode.FUSED_STACK_STEP
    decode.FUSED_STACK_STEP = fused_flag
    try:
        dec = decode.StackDecoder(tr, b, MAX_LEN)
        fused_on = dec.fused_ok()
        dec.load_cache(kv)
        dec.set_key_mask(mask)
        errs = {"out": [], "k": [], "v": []}
        for t in range(STEPS):
            n = n0 + t   # from t = 1 on, the step reads rows it appended itself
            want_out, want_k, want_v = _reference(st, dec, xs[t], n, **ref_kw)
            kc0, vc0 = dec.kc.clone(), dec.vc.clone()
            out = dec.step(xs[t].to(DEV))
            torch.cuda.synchronize()
            assert int(dec.len.item()) == n + 1
            assert dec.barrier_timeouts() == 0
            kc0[:, :, n], vc0[:, :, n] = dec.kc[:, :, n], dec.vc[:, :, n]
            assert torch.equal(kc0, dec.kc) and torch.equal(vc0, dec.vc), "a step wrote outside row n of the cache"
            errs["out"].append(_rel_rows(out, want_out))              # [b]
            errs["k"].append(_rel_rows(dec.kc[:, :, n], want_k))      # [depth, b]
            errs["v"].append(_rel_rows(dec.vc[:, :, n], want_v))
        return fused_on, {q: torch.stack(e) for q, e in errs.items()}
    finally:
        decode.FUSED_STACK_STEP = default


@pytest.mark.parametrize("b,d,heads,depth,n0,value_residual,mask_kind,streams,fused,bound,dc", CASES)
def test_step_matches_fp64_reference(b, d, heads, depth, n0, value_residual, mask_kind, streams, fused, bound, dc,
                                     request):
    torch.manual_seed(d * 7 + b * 3 + depth + n0)
    tr, st = _model(d, heads, depth, value_residual, streams)
    kv = torch.randn(depth, 2, b, n0, 64).to(bf16)
    mask = _key_mask(mask_kind, b, n0)
    xs = torch.randn(STEPS, b, d).to(bf16).float() + dc
    ref_kw = dict(heads=heads, depth=depth, streams=streams, value_residual=value_residual)
    multi_on, multi = _run_path(False, tr, st, b, n0, kv, mask, xs, ref_kw)
    fused_on, one = _run_path(True, tr, st, b, n0, kv, mask, xs, ref_kw)
    assert not multi_on and fused_on == fused
    tag = request.node.callspec.id
    for q in ("out", "k", "v"):
        print(f"[err] {tag} {q} multi={multi[q].max().item():.3e} fused={one[q].max().item():.3e} "
              f"ratio={(one[q] / multi[q].clamp(min=1e-12)).max().item():.2f}")
    for q in ("out", "k", "v"):
        assert (multi[q] <= bound).all(), (q, "multi-kernel", multi[q].max().item())
        assert (one[q] <= bound).all(), (q, "one-kernel" if fused else "fallback", one[q].max().item())
        worse = one[q] > torch.clamp(RATIO * multi[q], min=bound / 3)
        assert not worse.any(), (q, one[q][worse].tolist(), multi[q][worse].tolist())


def test_fused_cases_cover_staged_and_l2_weights():
    """over the one-kernel cases above, each of phases A, C, D, E (q|kv, out, W1, W2) reads its weights from shared
    memory at least once, and each of C, D, E from L2 at least once (A is placed first: only extreme shapes read it
    from L2); a change to the kernel's shared-memory plan that loses this coverage fails here"""
    from audiolm_pytorch_b200 import ops
    from audiolm_pytorch_b200.transformer import FeedForward

    seen = {True: set(), False: set()}
    for p in CASES:
        (b, d, heads, depth), fused = p.values[:4], p.values[8]
        if not fused:
            continue
        staged = ops.decode_stack_plan(b, d, heads, FeedForward(dim=d).inner, depth)
        assert staged is not None, p.id
        for phase, s in zip("ACDE", staged):
            seen[s].add(phase)
    assert seen[True] == set("ACDE") and seen[False] >= set("CDE"), seen
