"""Head widths 32 and 128 (dim_head) on the GPU: the attention kernels and the decode kernels against an fp64 reference,
and the three transformers against fixtures of the reference implementation (tests/golden/dim_head.pt).

Kernel level.  The fp64 reference and the per-row criterion are those of tests/test_attn_envelope_gpu.py with the head
width as an argument: every operand is bf16-representable, and each output vector (o, dq per (query, head); dk, dv per
key) is compared by its RMS-relative error over max(row RMS, 0.05 x tensor RMS).  The case list sits on both sides of
the tile edges of the tilings that are new at these widths: 128-key tiles and 128-query blocks in the forward at both
widths; in the backward 128-query iterations at D = 32 and 64-query iterations at D = 128 (sizes 63 / 64 / 65 / 127 /
128 / 129 / 191 / 192 / 193), right-aligned causal offsets that are not multiples of 64, key masks on 32-bit word
edges, -inf biases, dropout, strided operands, single-key probes and a batch past 65535."""
import math
import sys
from pathlib import Path

import pytest
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
import dropout_ref  # noqa: E402

DEV = "cuda"
bf16 = torch.bfloat16
f32 = torch.float32
f64 = torch.float64
LN2 = math.log(2.0)
FLOOR, FLOOR_ABS = 0.05, 1e-3
WIDTHS = [32, 128]
GOLDEN = Path(__file__).resolve().parent / "golden" / "dim_head.pt"

# Per-row bounds, about 3x the worst error measured over every case of this file on an H100 80GB HBM3 (700 W power
# limit).  Worst measured, D = 32 / D = 128: o 4.3e-3 (nq63) / 3.7e-3 (dropout-mask-bias), dq 5.7e-3 / 5.1e-3, dk 5.2e-3 /
# 4.7e-3, dv 5.2e-3 / 5.0e-3 (all three at b = 70,000), dbias 1.0e-5 / 1.2e-5, lse 7.3e-7 / 1.2e-6; single-key probes
# |dq| 1.3e-6 / 3.3e-6, |dk| 4.9e-6 / 1.6e-5; decode kernels o 2.5e-3 / 2.1e-3.  Against a reference that hides one
# key of every row the same kernels err by o 1.0 / 0.25, dq 1.6 / 0.31, dv 21 / 15 (test_a_dropped_key_would_fail).
BOUND = dict(o=1.3e-2, dq=1.7e-2, dk=1.6e-2, dv=1.6e-2, dbias=3.6e-5)
BOUND_LSE = 4e-6          # absolute, natural log
BOUND_PROBE_ABS = 5e-5    # |dq|, |dk| where the exact answer is 0


# ---- the reference ---------------------------------------------------------------------------------------------------
def attend_fp64(q, k, v, d_o=None, *, heads, key_mask=None, causal=True, scale=None, bias=None, keep=None, o_bwd=None):
    """fp64 multi-query attention with autograd for any head width D = k.shape[-1]: q [b, n_q, heads*D], k / v
    [b, n_k, D]; queries right-aligned against keys when causal; bias [heads, n_q, >= n_k]; keep [b, heads, n_q, n_k]
    dropout factors applied to the probabilities, not to the LSE.  A row that sees no key gets o = 0, lse = +inf and no
    gradient.  o_bwd: the output the backward is handed (delta = rowsum(dO o_bwd)), see test_attn_envelope_gpu.py."""
    b, n_q, hd = q.shape
    n_k, D = k.shape[1], k.shape[2]
    h = heads
    assert hd == h * D
    if scale is None:
        scale = D ** -0.5
    dev = q.device
    qh = q.detach().to(f64).view(b, n_q, h, D).permute(0, 2, 1, 3).requires_grad_()
    kf = k.detach().to(f64).requires_grad_()
    vf = v.detach().to(f64).requires_grad_()
    s = torch.einsum("bhid,bjd->bhij", qh, kf) * scale
    bf = None
    if bias is not None:
        bf = bias[..., :n_k].detach().to(f64).requires_grad_()
        s = s + bf
    vis = torch.ones(b, 1, n_q, n_k, dtype=torch.bool, device=dev)
    if key_mask is not None:
        vis = vis & key_mask.to(dev).bool()[:, None, None, :]
    if causal:
        i = torch.arange(n_q, device=dev)[:, None]
        j = torch.arange(n_k, device=dev)[None, :]
        vis = vis & (j <= i + (n_k - n_q))
    vis = vis & (s.detach() > -math.inf)
    seen = vis.any(-1, keepdim=True)
    s = torch.where(vis, s, -math.inf)
    s = torch.where(seen, s, 0.0)
    lse = torch.where(seen[..., 0], torch.logsumexp(s.detach(), -1), math.inf)
    p = torch.softmax(s, -1) * seen
    if keep is not None:
        p = p * keep.to(dev, f64)
    o = torch.einsum("bhij,bjd->bhid", p, vf).permute(0, 2, 1, 3).reshape(b, n_q, hd)
    out = dict(o=o.detach(), lse=lse)
    if d_o is not None:
        g = d_o.detach().to(dev, f64)
        loss = (o * g).sum()
        if o_bwd is not None:
            rowsum = lambda t: (t * g).view(b, n_q, h, D).sum(-1).permute(0, 2, 1)  # noqa: E731
            shift = rowsum(o.detach()) - rowsum(o_bwd.detach().to(dev, f64))
            loss = loss + (shift * torch.where(seen[..., 0], torch.logsumexp(s, -1), 0.0)).sum()
        loss.backward()
        out.update(dq=qh.grad.permute(0, 2, 1, 3).reshape(b, n_q, hd), dk=kf.grad, dv=vf.grad,
                   dbias=None if bf is None else bf.grad)
    return out


def keep_factors(b, h, n_q, n_k, p, seed, site):
    """[b, h, n_q, n_k] fp64 dropout factors from the numpy keep mask (tests/dropout_ref.py): counter row
    (batch * h + head) * n_q_pad + i, column = key, the same at every head width"""
    import numpy as np

    n_q_pad = (n_q + 127) // 128 * 128
    rows = (np.arange(b * h)[:, None] * n_q_pad + np.arange(n_q)[None, :]).reshape(-1)
    kept = dropout_ref.keep(seed, site, rows, np.arange(n_k), p)
    scale = float(np.float32(1.0 / (1.0 - float(np.float32(p)))))
    return torch.from_numpy(kept).view(b, h, n_q, n_k).to(f64) * scale


def row_err(got, want):
    got, want = got.to(f64), want.to(f64)
    num = (got - want).pow(2).mean(-1).sqrt()
    floor = max(FLOOR * want.pow(2).mean().sqrt().item(), FLOOR_ABS)
    return num / want.pow(2).mean(-1).sqrt().clamp(min=floor)


# ---- the cases -------------------------------------------------------------------------------------------------------
def case(b, h, n_q, n_k, causal, *, id, mask=None, bias=None, layout="contig", drop=0.0):
    return dict(b=b, h=h, n_q=n_q, n_k=n_k, causal=causal, mask=mask, bias=bias, layout=layout, drop=drop, id=id)


# mask: random | edges (only keys 31, 32, 63, 64, 95, 96, 127, 128); bias: rand | inf (-inf entries and whole rows)
# layout: qslice (q = columns [D, D + h*D) of a wider buffer) | kvsplit (k, v = halves of one [b, n_k, 2D] buffer)
SHAPES = [
    case(1, 1, 1, 1, True, id="nq1-nk1"),
    case(2, 3, 1, 129, True, mask="random", id="nq1-nk129-off128"),
    case(2, 3, 63, 63, True, id="nq63"),
    case(1, 3, 64, 64, False, mask="random", id="nq64-noncausal"),
    case(3, 2, 65, 65, True, id="nq65"),
    case(2, 3, 63, 190, True, id="nq63-nk190-off127"),
    case(1, 8, 127, 127, True, mask="random", id="nq127-h8"),
    case(2, 3, 128, 128, True, id="nq128"),
    case(2, 3, 129, 129, False, mask="random", id="nq129-noncausal"),
    case(2, 2, 130, 256, True, id="nq130-nk256-off126"),
    case(1, 4, 191, 191, True, id="nq191"),
    case(2, 2, 192, 193, True, mask="random", id="nq192-nk193-off1"),
    case(1, 3, 193, 257, True, id="nq193-nk257-off64"),
    case(1, 3, 129, 329, True, mask="random", id="nq129-nk329-off200"),
    case(2, 8, 257, 257, True, id="nq257-h8"),
    case(1, 8, 1024, 1024, True, mask="random", id="nq1024-h8-many-iters"),
    case(1, 2, 500, 1000, False, id="nq500-nk1000-noncausal"),
    case(2, 4, 300, 300, True, layout="qslice", mask="random", id="q-column-slice"),
    case(2, 3, 200, 456, True, layout="kvsplit", mask="random", id="kv-halves-right-aligned"),
    case(2, 3, 384, 384, True, mask="edges", id="mask-word-edges"),
    case(3, 2, 300, 300, False, mask="edges", id="mask-word-edges-noncausal"),
    case(2, 4, 300, 300, True, bias="rand", id="bias"),
    case(2, 4, 200, 333, True, bias="inf", mask="random", id="bias-inf-rows-right-aligned"),
    case(2, 3, 200, 200, True, drop=0.1, id="dropout"),
    case(2, 2, 300, 300, True, drop=0.1, mask="random", bias="rand", id="dropout-mask-bias"),
]
CASES = [pytest.param(D, c, id=f"d{D}-{c['id']}") for D in WIDTHS for c in SHAPES]


def _mask(kind, b, n_k, gen):
    if kind is None:
        return None
    m = torch.rand(b, n_k, generator=gen) > 0.15
    if kind == "edges":
        m[:] = False
        m[:, [31, 32, 63, 64, 95, 96, 127, 128]] = True
    return m


def _bias(kind, h, n_q, n_k, gen):
    if kind is None:
        return None
    ld = (n_k + 3) // 4 * 4 + 4
    bias = torch.full((h, n_q, ld), math.nan)
    val = torch.randn(h, n_q, n_k, generator=gen) * 1.5
    if kind == "inf":
        val[torch.rand(h, n_q, n_k, generator=gen) < 0.1] = -math.inf
        val[:, 5::17] = -math.inf
    bias[..., :n_k] = val.to(bf16).float()
    return bias


def make_operands(D, c, seed):
    gen = torch.Generator().manual_seed(seed)
    b, h, n_q, n_k = c["b"], c["h"], c["n_q"], c["n_k"]
    q = torch.randn(b, n_q, h * D, generator=gen)
    k = torch.randn(b, n_k, D, generator=gen)
    v = torch.randn(b, n_k, D, generator=gen)
    d_o = torch.randn(b, n_q, h * D, generator=gen)
    q, k, v, d_o = (t.to(bf16).to(DEV) for t in (q, k, v, d_o))
    if c["layout"] == "qslice":
        buf = torch.randn(b, n_q, h * D + 2 * D, generator=gen).to(bf16).to(DEV)
        buf[..., D:D + h * D] = q
        q = buf[..., D:D + h * D]
    elif c["layout"] == "kvsplit":
        kv = torch.cat((k, v), dim=-1)
        k, v = kv[..., :D], kv[..., D:]
    mask = _mask(c["mask"], b, n_k, gen)
    bias = _bias(c["bias"], h, n_q, n_k, gen)
    drop = (c["drop"], 0x5EED_0000_0000_0000 + seed, 7) if c["drop"] > 0 else None
    return q, k, v, d_o, None if mask is None else mask.to(DEV), None if bias is None else bias.to(DEV), drop


def run_case(D, c, seed, *, check_repro=True, drop_last_key=False):
    """kernels and reference on one case -> per-quantity error tensors.  drop_last_key: the reference is run with the
    last key of every sequence hidden, i.e. the kernels are made to look like ones that attend one key too many."""
    from audiolm_pytorch_b200 import ops

    q, k, v, d_o, mask, bias, drop = make_operands(D, c, seed)
    b, h, n_q, n_k = c["b"], c["h"], c["n_q"], c["n_k"]
    kw = dict(heads=h, key_mask=mask, causal=c["causal"], bias=bias, dropout=drop)
    o, lse = ops.mqa_attn_fwd(q, k, v, **kw)
    dbias = torch.zeros_like(bias) if bias is not None else None
    dq, dk, dv = ops.mqa_attn_bwd(q, k, v, o, d_o, lse, dbias=dbias, **kw)
    torch.cuda.synchronize()
    got = dict(o=o, lse=lse[..., :n_q].to(f64) * LN2, dq=dq, dk=dk, dv=dv,
               dbias=None if dbias is None else dbias[..., :n_k].clone())
    if check_repro:
        o2, lse2 = ops.mqa_attn_fwd(q, k, v, **kw)
        _, dk2, dv2 = ops.mqa_attn_bwd(q, k, v, o, d_o, lse, **kw)
        torch.cuda.synchronize()
        assert torch.equal(o, o2) and torch.equal(lse[..., :n_q], lse2[..., :n_q]), "forward not bitwise reproducible"
        assert torch.equal(dk, dk2) and torch.equal(dv, dv2), "dk / dv not bitwise reproducible"
    keep = keep_factors(b, h, n_q, n_k, *drop) if drop is not None else None
    ref_mask = mask
    if drop_last_key:
        ref_mask = torch.ones(b, n_k, dtype=torch.bool, device=DEV) if mask is None else mask.clone()
        ref_mask[:, -1] = False
    ref = attend_fp64(q, k, v, d_o, heads=h, key_mask=ref_mask, causal=c["causal"], bias=bias, keep=keep, o_bwd=o)
    for name in ("o", "dq", "dk", "dv"):
        assert torch.isfinite(got[name]).all(), f"{name} is not finite"
    dead = torch.isinf(ref["lse"])
    if not drop_last_key:
        assert torch.equal(torch.isinf(got["lse"]), dead), "rows without a visible key and rows with +inf lse differ"
    live = ~dead & torch.isfinite(got["lse"])
    errs = dict(
        o=row_err(got["o"].view(b, n_q, h, D), ref["o"].view(b, n_q, h, D)),
        dq=row_err(got["dq"].view(b, n_q, h, D), ref["dq"].view(b, n_q, h, D)),
        dk=row_err(got["dk"], ref["dk"]),
        dv=row_err(got["dv"], ref["dv"]),
        lse=(got["lse"][live].to(f64) - ref["lse"][live]).abs(),
    )
    if bias is not None:
        assert torch.isfinite(got["dbias"]).all() and (dbias[..., n_k:] == 0).all()
        errs["dbias"] = row_err(got["dbias"], ref["dbias"])
    return errs


def worst(errs):
    return {q: (e.max().item() if e.numel() else 0.0) for q, e in errs.items()}


def check_errs(errs, tag):
    w = worst(errs)
    print(f"[err] {tag} " + " ".join(f"{q}={x:.3e}" for q, x in w.items()))
    for q, x in w.items():
        bound = BOUND_LSE if q == "lse" else BOUND[q]
        assert x <= bound, (q, x, bound)


@pytest.mark.gpu
@pytest.mark.parametrize("D,c", CASES)
def test_attention_matches_fp64(D, c, request):
    seed = (D * 1009 + c["b"] * 131 + c["h"] * 17 + c["n_q"] * 7 + c["n_k"]) % 100003
    check_errs(run_case(D, c, seed), request.node.callspec.id)


@pytest.mark.gpu
@pytest.mark.parametrize("D", WIDTHS)
def test_a_dropped_key_would_fail(D):
    """the criterion's power: against a reference that hides the last key of every row, the same kernels are far
    outside the bounds, so a kernel that drops (or adds) one key cannot pass test_attention_matches_fp64"""
    c = case(2, 3, 193, 257, False, id="power")
    w = worst(run_case(D, c, 5, check_repro=False, drop_last_key=True))
    print(f"[err] d{D}-dropped-key " + " ".join(f"{q}={x:.3e}" for q, x in w.items()))
    assert w["o"] > 3 * BOUND["o"] and w["dv"] > 3 * BOUND["dv"] and w["dq"] > 3 * BOUND["dq"], w


PROBE_KEYS = [0, 31, 32, 63, 64, 95, 96, 127, 128, 260, 299]


@pytest.mark.gpu
@pytest.mark.parametrize("D", WIDTHS)
@pytest.mark.parametrize("causal,n_q", [(False, 300), (True, 170)], ids=["noncausal", "causal-off130"])
def test_single_visible_key_is_exact(D, causal, n_q):
    """batch row r masks every key except PROBE_KEYS[r]: o is v[j] bitwise on the rows that see j and 0 elsewhere, dv[j]
    is the sum of those dO rows, masked keys get no gradient, and dq, dk vanish up to rounding"""
    from audiolm_pytorch_b200 import ops

    n_k, h = 300, 3
    b = len(PROBE_KEYS)
    gen = torch.Generator().manual_seed(n_q + int(causal) + D)
    q = torch.randn(b, n_q, h * D, generator=gen).to(bf16).to(DEV)
    k = torch.randn(b, n_k, D, generator=gen).to(bf16).to(DEV)
    v = torch.randn(b, n_k, D, generator=gen).to(bf16).to(DEV)
    d_o = torch.randn(b, n_q, h * D, generator=gen).to(bf16).to(DEV)
    mask = torch.zeros(b, n_k, dtype=torch.bool, device=DEV)
    js = torch.tensor(PROBE_KEYS, device=DEV)
    rows = torch.arange(b, device=DEV)
    mask[rows, js] = True
    o, lse = ops.mqa_attn_fwd(q, k, v, heads=h, key_mask=mask, causal=causal)
    dq, dk, dv = ops.mqa_attn_bwd(q, k, v, o, d_o, lse, heads=h, key_mask=mask, causal=causal)
    torch.cuda.synchronize()
    off = n_k - n_q
    sees = (torch.arange(n_q, device=DEV)[None, :] + off >= js[:, None]) if causal else \
        torch.ones(b, n_q, dtype=torch.bool, device=DEV)
    oh = o.view(b, n_q, h, D)
    want = torch.where(sees[..., None, None], v[rows, js][:, None, None, :], torch.zeros((), dtype=bf16, device=DEV))
    assert torch.equal(oh, want.expand_as(oh)), "o is not v[j] bitwise on rows that see j, or not 0 on the others"
    score = torch.einsum("bihd,bd->bhi", q.view(b, n_q, h, D).to(f64), k[rows, js].to(f64)) * D ** -0.5
    lse_n = lse[..., :n_q].to(f64) * LN2
    seen3 = sees[:, None, :].expand(b, h, n_q)
    assert torch.isinf(lse_n[~seen3]).all() and (lse_n[seen3] - score[seen3]).abs().max().item() <= BOUND_LSE
    dv_j = (d_o.view(b, n_q, h, D).to(f64) * sees[..., None, None]).sum((1, 2))
    assert row_err(dv[rows, js], dv_j).max().item() <= BOUND["dv"]
    assert (dv[~mask] == 0).all() and (dk[~mask] == 0).all(), "a masked key received a gradient"
    print(f"[err] d{D}-probe dq={dq.float().abs().max().item():.3e} dk={dk.float().abs().max().item():.3e}")
    assert dq.float().abs().max().item() <= BOUND_PROBE_ABS and dk.float().abs().max().item() <= BOUND_PROBE_ABS


@pytest.mark.gpu
@pytest.mark.parametrize("D", WIDTHS)
def test_batch_past_grid_limit(D):
    c = case(70000, 1, 1, 2, True, mask="random", id="b70000")
    check_errs(run_case(D, c, 70000 + D, check_repro=False), f"d{D}-b70000")


@pytest.mark.gpu
def test_same_seed_same_mask_at_every_width():
    """the dropout counter addresses (row, key) only: with v = identity columns the output of a uniform-score row is
    the keep pattern itself, and it is the same at D = 32, 64 and 128"""
    from audiolm_pytorch_b200 import ops

    b, h, n = 1, 2, 32
    pats = []
    for D in (32, 64, 128):
        q = torch.zeros(b, n, h * D, device=DEV, dtype=bf16)
        k = torch.zeros(b, n, D, device=DEV, dtype=bf16)
        v = torch.zeros(b, n, D, device=DEV, dtype=bf16)
        v[0, torch.arange(n), torch.arange(n)] = 1.0            # v[j] = e_j: o[i, :n] = P[i, :] o Z[i, :]
        o, _ = ops.mqa_attn_fwd(q, k, v, heads=h, causal=False, dropout=(0.3, 1234, 3))
        pats.append((o.view(b, n, h, D)[..., :n] > 0).cpu())
    assert pats[0].any() and not pats[0].all()
    assert torch.equal(pats[0], pats[1]) and torch.equal(pats[1], pats[2])
    want = keep_factors(b, h, n, n, 0.3, 1234, 3) > 0           # [b, h, n_q, n_k]
    assert torch.equal(pats[1].permute(0, 2, 1, 3), want)


@pytest.mark.gpu
def test_backward_is_deterministic_at_128():
    """dk / dv accumulate in registers over the heads (no atomics): two runs are bit-identical"""
    from audiolm_pytorch_b200 import ops

    gen = torch.Generator().manual_seed(9)
    b, h, n, D = 2, 8, 700, 128
    q, d_o = (torch.randn(b, n, h * D, generator=gen).to(bf16).to(DEV) for _ in range(2))
    k, v = (torch.randn(b, n, D, generator=gen).to(bf16).to(DEV) for _ in range(2))
    mask = (torch.rand(b, n, generator=gen) > 0.1).to(DEV)
    o, lse = ops.mqa_attn_fwd(q, k, v, heads=h, key_mask=mask)
    runs = [ops.mqa_attn_bwd(q, k, v, o, d_o, lse, heads=h, key_mask=mask) for _ in range(2)]
    torch.cuda.synchronize()
    assert torch.equal(runs[0][1], runs[1][1]) and torch.equal(runs[0][2], runs[1][2])


def test_unsupported_width_is_an_error_not_a_trap():
    """the C entry points return ALM_ERR_UNSUPPORTED (-4) for a width they are not built for, before touching a pointer"""
    from audiolm_pytorch_b200 import _lib

    lib = _lib.load()
    assert lib.alm_mqa_attn_fwd_dh(*([0] * 16), 1, 1, 1, 1, 1, 1.0, 0.0, 0, 0, 48, None) == -4
    assert lib.alm_kv_append_dh(0, 0, 0, 0, 0, 0, 1, 1, 256, None) == -4
    assert lib.alm_decode_stack_plan_dh(1, 512, 8, 1365, 6, 128, None) == -4


# ---- decode kernels --------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("D", WIDTHS)
@pytest.mark.parametrize("splits", [1, 4])
def test_decode_kernels_match_fp64(D, splits):
    """kv_append + mqa_attn_decode against the reference at cache lengths around the key-split edges (a split covers a
    multiple of 32 keys), with a key mask and a bias row"""
    from audiolm_pytorch_b200 import ops

    b, h, max_len = 3, 5, 300
    gen = torch.Generator().manual_seed(D + splits)
    kc = torch.zeros(b, max_len, D, device=DEV, dtype=bf16)
    vc = torch.zeros_like(kc)
    hist = torch.randn(b, max_len, 2 * D, generator=gen).to(bf16).to(DEV)
    mask = (torch.rand(b, max_len, generator=gen) > 0.2).to(DEV)
    mask[:, 0] = True
    bias = (torch.randn(h, max_len + 4, generator=gen) * 1.5).to(bf16).float().to(DEV)
    worst_o = 0.0
    for L in (0, 1, 31, 32, 33, 63, 64, 127, 128, 129, 255, 299):
        kc[:, :L] = hist[:, :L, :D]
        vc[:, :L] = hist[:, :L, D:]
        ln = torch.tensor([L], device=DEV, dtype=torch.int32)
        ops.kv_append(hist[:, L], kc, vc, ln)
        assert torch.equal(kc[:, L], hist[:, L, :D]) and torch.equal(vc[:, L], hist[:, L, D:])
        q = torch.randn(b, h * D, generator=gen).to(bf16).to(DEV)
        for use_bias in (False, True):
            o = ops.mqa_attn_decode(q, kc, vc, ln, heads=h, key_mask=mask.to(torch.uint8), splits=splits,
                                    bias=bias if use_bias else None)
            ref = attend_fp64(q[:, None], kc[:, :L + 1], vc[:, :L + 1], heads=h, key_mask=mask[:, :L + 1], causal=True,
                              bias=bias[:, None, :L + 1].contiguous() if use_bias else None)["o"]
            e = row_err(o.view(b, h, D), ref.view(b, h, D)).max().item()
            worst_o = max(worst_o, e)
    print(f"[err] d{D}-decode-splits{splits} o={worst_o:.3e}")
    assert worst_o <= BOUND["o"]


# ---- model level: the three transformers against the reference's fixtures -------------------------------------------
def unpack(p, device="cpu"):
    """inverse of oracle/make_golden_dim_head.py::_pack: {name: fp32 tensor} (values left out of the file are zeros)"""
    out, at = {}, 0
    for name, shape in zip(p["names"], p["shapes"]):
        n = math.prod(shape)
        if name in p["unused"]:
            out[name] = torch.zeros(shape)
        else:
            out[name] = p["flat"][at:at + n].float().view(shape)
            at += n
    assert at == p["flat"].numel()
    out.update(p["other"])
    return {k: v.to(device) for k, v in out.items()}


def fixture(D, model):
    from oracle import golden
    return golden.load(GOLDEN.name)[D][model]


def rms_rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).pow(2).mean().sqrt() / b.pow(2).mean().sqrt().clamp(min=1e-12)).item()


def build(cls, g, *, math_path=False, **over):
    kw = {**g["kwargs"], **over}
    state = unpack(g["state"])
    if math_path:
        kw["flash_attn"] = False
        state.update(unpack(g["math_extra"]))
    m = cls(**kw)
    m.load_state_dict(state, strict=True)
    return m.to(DEV)


def check_grads(named, grads, noise):
    """as tests/test_models_gpu.py::check_grads: RMS-relative error of every parameter gradient below max(7e-2, 2 x the
    reference's own deviation under bf16 autocast); the tiny hyper-connection tensors against their kind's largest,
    below max(0.35, 2 x that deviation)"""
    kind_scale = {}
    for k, gr in grads.items():
        if gr.numel() <= 20:
            kind = k.split(".")[-1]
            kind_scale[kind] = max(kind_scale.get(kind, 0.0), gr.float().pow(2).mean().sqrt().item())
    bad = {}
    for k, gr in grads.items():
        assert named[k].grad is not None, k
        if gr.numel() <= 20:
            e = (named[k].grad.float().cpu() - gr.float()).pow(2).mean().sqrt().item() / kind_scale[k.split(".")[-1]]
            tol = max(0.35, 2.0 * noise.get(k, 0.0))   # a few dozen tokens: the reference's own bf16 spread reaches 1.6
        else:
            e, tol = rms_rel(named[k].grad, gr), max(7e-2, 2.0 * noise.get(k, 0.0))
        if e >= tol:
            bad[k] = (e, tol)
    assert not bad, bad


class _Codec:
    rq_groups = 1
    num_quantizers = 5


def _model_io(model, g):
    """(class, wrapper factory, forward kwargs, logits keys, loss kwargs) of one fixture"""
    from audiolm_pytorch_b200 import audiolm as A

    if model == "semantic":
        ids = g["ids"].to(DEV)
        return (A.SemanticTransformer, lambda m: A.SemanticTransformerWrapper(transformer=m, unique_consecutive=False,
                                                                               mask_prob=0.0),
                dict(ids=ids), ("logits",), dict(semantic_token_ids=ids))
    if model == "coarse":
        sem, coarse = g["sem"].to(DEV), g["coarse"].to(DEV)
        return (A.CoarseTransformer, lambda m: A.CoarseTransformerWrapper(transformer=m, codec=_Codec(),
                                                                           unique_consecutive=False, mask_prob=0.0),
                dict(semantic_token_ids=sem, coarse_token_ids=coarse), ("sem_logits", "coarse_logits"),
                dict(semantic_token_ids=sem, coarse_token_ids=coarse[:, :12]))
    coarse, fine = g["coarse"].to(DEV), g["fine"].to(DEV)
    return (A.FineTransformer, lambda m: A.FineTransformerWrapper(transformer=m, codec=_Codec(), mask_prob=0.0),
            dict(coarse_token_ids=coarse.reshape(2, -1), fine_token_ids=fine.reshape(2, -1)[:, :-1]),
            ("coarse_logits", "fine_logits"), dict(coarse_token_ids=coarse, fine_token_ids=fine))


MODELS = ["semantic", "coarse", "fine"]


@pytest.mark.gpu
@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("D", WIDTHS)
def test_model_matches_reference(D, model):
    """logits on the flash and on the score-bias path, the wrapper's loss and every parameter gradient"""
    g = fixture(D, model)
    cls, wrap, fwd, keys, loss_kw = _model_io(model, g)
    m = build(cls, g).eval()
    mm = build(cls, g, math_path=True).eval()
    with torch.no_grad():
        got, got_math = m(**fwd), mm(**fwd)
    got, got_math = (((t,) if torch.is_tensor(t) else tuple(t)) for t in (got, got_math))
    for key, a, b in zip(keys, got, got_math):
        ea, eb = rms_rel(a, g[key]), rms_rel(b, g[key + "_math"])
        print(f"[err] d{D}-{model} {key} flash={ea:.3e} bias={eb:.3e}")
        assert ea < 1.5e-2 and eb < 1.5e-2, (key, ea, eb)
    w = wrap(m).train()
    loss = w(return_loss=True, **loss_kw)
    assert abs(loss.item() - g["loss"].item()) < 2e-2 * abs(g["loss"].item()), (loss.item(), g["loss"].item())
    loss.backward()
    check_grads(dict(m.named_parameters()), unpack(g["grads"]), g["bf16_noise"])


@pytest.mark.gpu
@pytest.mark.parametrize("D", WIDTHS)
def test_kv_cache_forward_matches_full_forward(D):
    """Transformer(..., kv_cache=...) on the score-bias path: the reference's outputs, its cache tensor
    [depth, 2, b, n, dim_head], and the cached positions equal to the full forward's"""
    from audiolm_pytorch_b200.audiolm import SemanticTransformer

    g = fixture(D, "semantic")
    t = build(SemanticTransformer, g, math_path=True).eval().transformer
    f = g["transformer"]
    x = f["x"].to(DEV)
    with torch.no_grad():
        full = t(x)
        _, cache = t(x[:, :9], return_kv_cache=True)
        inc, cache2 = t(x, kv_cache=cache, return_kv_cache=True)
    assert cache.shape == (2, 2, 2, 9, D) and cache2.shape == (2, 2, 2, 14, D)
    assert rms_rel(full, f["out"]) < 1.5e-2 and rms_rel(inc, f["out_inc"]) < 1.5e-2
    assert rms_rel(cache, f["cache9"]) < 1e-2
    assert rms_rel(inc, full[:, 9:]) < 1e-2


def _teacher_forced(tr, b, n0, n1, *, graphed=True):
    """decode engine vs the full forward of the same stack, per step: positions n0..n1-1 of random embeddings"""
    from audiolm_pytorch_b200.decode import GraphedStep, StackDecoder

    gen = torch.Generator().manual_seed(n1)
    xs = torch.randn(b, n1, tr.dim, generator=gen).to(DEV)
    with torch.no_grad():
        full = tr(xs)
        _, kv = tr(xs[:, :n0], return_kv_cache=True)
        dec = StackDecoder(tr, b, 64)
        assert dec.kc.shape == (tr.depth, b, 64, tr.dim_head)
        dec.load_cache(kv)
        x = torch.zeros(b, tr.dim, device=DEV)
        y = torch.zeros(b, tr.dim, device=DEV, dtype=bf16)

        def fn():
            y.copy_(dec.step(x))

        step = GraphedStep(fn, [dec.len, y]) if graphed else fn
        errs = []
        for t in range(n0, n1):
            x.copy_(xs[:, t])
            step()
            errs.append(rms_rel(y, full[:, t]))
    assert int(dec.len.item()) == n1
    return dec, max(errs)


@pytest.mark.gpu
@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("D", WIDTHS)
def test_graphed_engine_matches_full_forward(D, model):
    """the graphed multi-kernel decode step, teacher-forced over the stack of each of the three models"""
    g = fixture(D, model)
    m = build(_model_io(model, g)[0], g).eval()
    _, e = _teacher_forced(m.transformer, 2, 5, 14)
    print(f"[err] d{D}-{model}-engine {e:.3e}")
    assert e < 1.5e-2, e


@pytest.mark.gpu
@pytest.mark.parametrize("D,streams", [(32, 1), (128, 4), (128, 1)])
def test_residual_stream_counts(D, streams):
    """num_residual_streams 1 and 4 at the new widths: training gradients flow and the engine follows the forward"""
    from audiolm_pytorch_b200.transformer import Transformer

    torch.manual_seed(D + streams)
    tr = Transformer(dim=64, depth=2, heads=2, dim_head=D, flash_attn=True, num_residual_streams=streams).to(DEV)
    x = torch.randn(2, 20, 64, device=DEV, requires_grad=True)
    tr.train()(x).float().pow(2).mean().backward()
    assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in tr.parameters())
    assert tr.layers[0][0].branch.to_kv.weight.grad.abs().max() > 0
    _, e = _teacher_forced(tr.eval(), 2, 5, 14)
    assert e < 1.5e-2, e


@pytest.mark.gpu
def test_one_kernel_step_falls_back_at_128():
    """the one-kernel decode step is built for dim_head 64: with it switched on, a dim_head-128 stack still runs the
    multi-kernel step and gives that step's result bitwise"""
    from audiolm_pytorch_b200 import decode, ops
    from audiolm_pytorch_b200.transformer import Transformer

    torch.manual_seed(7)
    tr = Transformer(dim=256, depth=2, heads=4, dim_head=128, flash_attn=True).to(DEV).eval()
    assert ops.decode_stack_plan(2, 256, 4, tr.layers[0][2].branch.inner, 2, dim_head=64) is not None
    assert ops.decode_stack_plan(2, 256, 4, tr.layers[0][2].branch.inner, 2, dim_head=128) is None
    xs = torch.randn(3, 2, 256, device=DEV)
    outs = []
    default = decode.FUSED_STACK_STEP
    for fused in (False, True):
        decode.FUSED_STACK_STEP = fused
        try:
            dec = decode.StackDecoder(tr, 2, 64)
            assert not dec.fused_ok()
            outs.append(torch.stack([dec.step(xs[t]).clone() for t in range(3)]))
            assert dec._fused is None
        finally:
            decode.FUSED_STACK_STEP = default
    assert torch.equal(outs[0], outs[1])


@pytest.mark.gpu
@pytest.mark.parametrize("D", WIDTHS)
def test_wrappers_generate_on_the_engine(D):
    """generate() of the three wrappers at the new widths runs on captured graphs; with the sampler forced to argmax
    the coarse and fine engines emit the ids of the slow (re-forwarding) path"""
    from audiolm_pytorch_b200 import audiolm as A

    g = fixture(D, "semantic")
    m = build(A.SemanticTransformer, g).eval()
    w = A.SemanticTransformerWrapper(transformer=m, unique_consecutive=False)
    ids = g["ids"].to(DEV)
    out = w.generate(max_length=30, prime_ids=ids[:, :5])
    assert torch.equal(out[:, :5], ids[:, :5]) and ((out >= -1) & (out < m.num_semantic_tokens)).all()
    assert w._engine is not None and w._engine[1]._graphs

    g = fixture(D, "coarse")
    c = build(A.CoarseTransformer, g).eval()
    cw = A.CoarseTransformerWrapper(transformer=c, codec=_Codec(), unique_consecutive=False)
    kw = dict(semantic_token_ids=g["sem"].to(DEV), max_time_steps=4, temperature=1e-4, filter_thres=0.0)
    fast, slow = cw.generate(**kw), cw.generate(use_kv_cache=False, **kw)
    assert cw._engine is not None and fast.shape == slow.shape == (2, 4, 3)
    assert (fast == slow).float().mean().item() > 0.9

    g = fixture(D, "fine")
    f = build(A.FineTransformer, g).eval()
    fw = A.FineTransformerWrapper(transformer=f, codec=_Codec())
    kw = dict(coarse_token_ids=g["coarse"].to(DEV), temperature=1e-4, filter_thres=0.0)
    fast, slow = fw.generate(**kw), fw.generate(use_kv_cache=False, **kw)
    assert fast.shape == slow.shape == (2, 4, 3) and (fast == slow).float().mean().item() > 0.9


@pytest.mark.gpu
def test_full_width_model_trains_and_samples():
    """the usual heads * dim_head == dim scaling: dim 1024, 8 heads of 128"""
    from audiolm_pytorch_b200.audiolm import SemanticTransformer, SemanticTransformerWrapper

    torch.manual_seed(0)
    m = SemanticTransformer(dim=1024, depth=6, heads=8, dim_head=128, num_semantic_tokens=500, flash_attn=True).to(DEV)
    w = SemanticTransformerWrapper(transformer=m, unique_consecutive=False)
    opt = torch.optim.SGD(m.parameters(), lr=1e-3)
    ids = torch.randint(0, 500, (2, 300), device=DEV)
    loss = w.train()(semantic_token_ids=ids, return_loss=True)
    loss.backward()
    opt.step()
    assert torch.isfinite(loss) and abs(loss.item() - math.log(501)) < 1.5
    out = w.eval().generate(max_length=64, prime_ids=ids[:, :8])
    assert out.shape[0] == 2 and 8 < out.shape[1] <= 64 and w._engine is not None and w._engine[1]._graphs
