"""Attention forward and backward (ops.mqa_attn_fwd / ops.mqa_attn_bwd) against an fp64 reference across the kernels'
envelope: n_q / n_k on both sides of every 128-row tile edge, right-aligned causal offsets that are not multiples of
128, backward key blocks that walk 1, 2, 3, 4 or many (head, query block) iterations and start past query block 0,
strided q / k / v, key masks on every 32-bit word edge of a tile, -inf and NaN-padded score biases, dropout, peaked
softmaxes whose row max jumps in the last tile, exact single-key probes, NaN in the LSE pads, and batches past the
65535 limit of a grid's y / z dimension.

Every operand is bf16-representable, so the reference sees exactly the kernels' inputs and the error measured is the
kernels' own arithmetic (fp32 scores, P and dS rounded to bf16 for the tensor cores, bf16 outputs).  The criterion is
per row: the RMS-relative error of every output vector (o, dq and dbias per (query, head); dk, dv per key) over
max(row RMS, 0.05 x tensor RMS), and the absolute error of every row's natural-log LSE.  A bug confined to a few keys
of a long causal row hardly moves a whole-tensor max-error criterion; a per-row one sees it.

The GPU tests are marked individually; the reference's own check against torch SDPA and the case-list coverage checks
run without a GPU."""
import math
import sys
from pathlib import Path

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, str(Path(__file__).resolve().parent))
import dropout_ref  # noqa: E402

DEV = "cuda"
bf16 = torch.bfloat16
f64 = torch.float64
LN2 = math.log(2.0)
TILE = 128        # query / key tile edge of both kernels
AB_STAGES = 3     # Q / dO pipeline depth of the backward (csrc/attn_bwd_wgmma.cu)
FLOOR = 0.05      # row-RMS floor of the relative error, as a fraction of the tensor RMS
FLOOR_ABS = 1e-3  # and in absolute terms, for gradients that vanish exactly (dq, dk over a single key)

# Per-row bounds, one per quantity, about 3x the worst error measured over every case of this file on an H100 80GB
# HBM3 (400 W power limit).  Worst measured: o 4.2e-3 (dropout), dq 8.7e-3 and dk 7.5e-3 (late-max-noncausal-bias),
# dv 5.3e-3 (b = 70,000), dbias 6.9e-6 (fp32 dS, no bf16 staging), lse 6.9e-6; single-key probes |dq| 1.8e-6,
# |dk| 7.7e-6.  A kernel that drops one key of every row (the last) errs by 0.11-0.17 per row.
BOUND = dict(o=1.3e-2, dq=2.6e-2, dk=2.2e-2, dv=1.6e-2, dbias=2e-5)
BOUND_LSE = 2e-5  # absolute, natural log
BOUND_PROBE_ABS = 2.5e-5  # |dq|, |dk| where the exact answer is 0 (single-key probes)


# ---- the reference ---------------------------------------------------------------------------------------------------
def attend_fp64(q, k, v, d_o=None, *, heads, key_mask=None, causal=True, scale=None, bias=None, keep=None,
                o_bwd=None):
    """fp64 multi-query attention with autograd, on the device of q.

    q [b, n_q, heads*64], k / v [b, n_k, 64], d_o like q or None; key_mask bool [b, n_k] (True = attend); queries are
    right-aligned against keys (query i sees keys j <= i + n_k - n_q when causal); bias [heads, n_q, >= n_k] added to
    the scaled scores (columns past n_k are ignored); keep [b, heads, n_q, n_k] dropout factors (0 or 1/(1-p)) applied
    to the probabilities, not to the LSE.  A key whose score is -inf (a -inf bias) is hidden as a masked key is.  A row
    that sees no key gets o = 0, lse = +inf and no gradient, the kernels' definition.
    o_bwd: the output the backward is handed, or None for the exact o.  The backward takes o as an input and forms
    dS = P (dP - delta) with delta = rowsum(dO o) over it, so its gradients are those of that o; where dP nearly cancels
    delta (peaked rows, few keys) the bf16 rounding of o alone moves dq / dk far more than the kernel's own arithmetic.
    The term sum_i (delta_exact - delta_given)_i lse_i added to the loss makes autograd produce exactly those.
    Returns {o, lse [b, heads, n_q] (natural log)} and, with d_o, {dq, dk, dv, dbias}."""
    b, n_q, hd = q.shape
    n_k = k.shape[1]
    h = heads
    if scale is None:
        scale = 64 ** -0.5
    dev = q.device
    qh = q.detach().to(f64).view(b, n_q, h, 64).permute(0, 2, 1, 3).requires_grad_()
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
    s = torch.where(seen, s, 0.0)                  # a dead row: any finite values, its P is zeroed below
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
            rowsum = lambda t: (t * g).view(b, n_q, h, 64).sum(-1).permute(0, 2, 1)  # noqa: E731  [b, h, n_q]
            shift = rowsum(o.detach()) - rowsum(o_bwd.detach().to(dev, f64))
            loss = loss + (shift * torch.where(seen[..., 0], torch.logsumexp(s, -1), 0.0)).sum()
        loss.backward()
        out.update(dq=qh.grad.permute(0, 2, 1, 3).reshape(b, n_q, hd), dk=kf.grad, dv=vf.grad,
                   dbias=None if bf is None else bf.grad)
    return out


def keep_factors(b, h, n_q, n_k, p, seed, site):
    """[b, h, n_q, n_k] fp64 dropout factors of the attention kernels from the numpy keep mask: counter row
    (batch * h + head) * n_q_pad + i, column = key; kept elements are scaled by float32(1 / (1 - p))"""
    import numpy as np

    n_q_pad = (n_q + TILE - 1) // TILE * TILE
    rows = (np.arange(b * h)[:, None] * n_q_pad + np.arange(n_q)[None, :]).reshape(-1)
    kept = dropout_ref.keep(seed, site, rows, np.arange(n_k), p)
    scale = float(np.float32(1.0 / (1.0 - float(np.float32(p)))))
    return torch.from_numpy(kept).view(b, h, n_q, n_k).to(f64) * scale


def row_err(got, want):
    """RMS-relative error of every vector along the last dimension, over max(row RMS, FLOOR x tensor RMS, FLOOR_ABS)"""
    got, want = got.to(f64), want.to(f64)
    num = (got - want).pow(2).mean(-1).sqrt()
    floor = max(FLOOR * want.pow(2).mean().sqrt().item(), FLOOR_ABS)
    return num / want.pow(2).mean(-1).sqrt().clamp(min=floor)


# ---- the cases -------------------------------------------------------------------------------------------------------
def case(b, h, n_q, n_k, causal, *, id, mask=None, bias=None, layout="contig", scale=None, qmul=1.0, late=False,
         drop=0.0):
    return pytest.param(dict(b=b, h=h, n_q=n_q, n_k=n_k, causal=causal, mask=mask, bias=bias, layout=layout,
                             scale=scale, qmul=qmul, late=late, drop=drop), id=id)


# mask: random | edges (only keys 31, 32, 63, 64, 95, 96, 127, 128) | tile-off (keys [128, 256) off) |
#       row-dead (batch row 0 sees no key, the others random) | first-block (keys [0, 128) off)
# bias: rand | inf (-inf entries and whole -inf rows); its pad columns are NaN
# layout: qslice (q = columns [64, 64 + h*64) of a [b, n, h*64 + 128] buffer) | kvsplit (k, v = halves of [b, n_k, 128])
CASES = [
    # shape envelope: n_q / n_k at tile residues, right-aligned offsets, heads, batch, n_iter of the backward
    case(1, 1, 1, 1, True, id="nq1-nk1-single-key"),
    case(2, 3, 1, 129, True, mask="random", id="nq1-nk129-off128-one-query"),
    case(1, 1, 1, 2048, True, id="nq1-nk2048-off2047-decode-row"),
    case(2, 3, 63, 63, True, id="nq63-nk63-b2-h3"),
    case(1, 3, 64, 64, False, mask="random", id="nq64-nk64-noncausal"),
    case(5, 1, 64, 65, True, mask="random", id="nq64-nk65-off1-b5"),
    case(1, 8, 65, 65, False, id="nq65-nk65-noncausal-h8"),
    case(2, 3, 63, 190, True, id="nq63-nk190-off127"),
    case(1, 16, 127, 127, True, mask="random", id="nq127-nk127-h16"),
    case(2, 16, 127, 255, True, id="nq127-nk255-off128"),
    # off = 126: the last key of a tile is one past the first query row of a block, so the tile must not be "full"
    case(1, 4, 2, 128, True, id="nq2-nk128-off126-diagonal-tile-edge"),
    case(2, 3, 130, 256, True, id="nq130-nk256-off126-diagonal-tile-edge"),
    case(1, 24, 128, 128, True, id="nq128-nk128-h24"),
    case(5, 3, 128, 129, True, mask="random", id="nq128-nk129-off1-b5"),
    case(1, 16, 128, 257, True, id="nq128-nk257-off129"),
    case(2, 1, 129, 129, False, mask="random", id="nq129-nk129-noncausal"),
    case(2, 1, 129, 257, True, id="nq129-nk257-off128-h1"),
    case(1, 3, 129, 329, True, mask="random", id="nq129-nk329-off200"),
    case(5, 3, 255, 256, True, id="nq255-nk256-off1-b5"),
    case(1, 8, 255, 255, False, id="nq255-nk255-noncausal"),
    case(1, 8, 256, 256, True, mask="random", id="nq256-nk256"),
    case(2, 1, 256, 383, True, id="nq256-nk383-off127"),
    case(2, 24, 257, 257, True, id="nq257-nk257-h24"),
    case(1, 3, 257, 2048, True, mask="random", id="nq257-nk2048-off1791"),
    case(1, 8, 2048, 2048, True, mask="random", id="nq2048-nk2048-h8-many-iters"),
    case(2, 8, 1000, 2048, False, id="nq1000-nk2048-noncausal"),
    case(1, 1, 512, 512, True, id="nq512-h1-iters-1-2-3-4"),
    case(1, 2, 384, 385, True, id="nq384-nk385-off1-h2-iters-2-4-6"),
    case(1, 3, 2048, 2048, True, id="nq2048-h3-iters-3-to-48"),
    # operand layouts and scale
    case(2, 8, 300, 300, True, layout="qslice", mask="random", id="q-column-slice"),
    case(2, 8, 300, 300, True, layout="kvsplit", id="kv-halves-of-one-buffer"),
    case(2, 3, 200, 456, True, layout="kvsplit", mask="random", id="kv-halves-right-aligned"),
    case(2, 4, 256, 256, False, layout="qslice", scale=0.3, id="scale-0.3-q-slice-noncausal"),
    case(2, 1, 128, 256, True, scale=8.0, qmul=0.125, id="scale-8"),
    # masks and bias
    case(2, 3, 384, 384, True, mask="edges", id="mask-word-edges"),
    case(3, 2, 300, 300, False, mask="edges", id="mask-word-edges-noncausal"),
    case(2, 8, 512, 512, True, mask="tile-off", id="mask-whole-tile-off"),
    case(3, 3, 300, 300, True, mask="row-dead", id="mask-dead-batch-row"),
    case(2, 8, 384, 384, True, mask="first-block", id="mask-first-block"),
    case(2, 4, 300, 300, True, bias="rand", id="bias-nan-pads"),
    case(2, 4, 200, 333, True, bias="inf", mask="random", id="bias-inf-rows-right-aligned"),
    case(1, 3, 129, 129, False, bias="inf", id="bias-inf-rows-noncausal"),
    case(2, 3, 200, 200, True, drop=0.1, id="dropout"),
    case(2, 2, 300, 300, True, drop=0.1, mask="random", bias="rand", id="dropout-mask-bias"),
    case(1, 4, 129, 200, False, drop=0.1, layout="kvsplit", id="dropout-noncausal-kv-halves"),
    # numerically hard inputs
    case(2, 8, 384, 384, True, qmul=4.0, id="peaked-q-x4"),
    case(2, 8, 300, 300, False, qmul=8.0, mask="random", id="peaked-q-x8"),
    case(1, 8, 2048, 2048, True, qmul=4.0, id="peaked-q-x4-long"),
    case(2, 4, 512, 512, True, late=True, id="late-max"),
    case(2, 4, 200, 456, True, late=True, mask="random", id="late-max-right-aligned"),
    case(1, 3, 257, 257, False, late=True, bias="rand", id="late-max-noncausal-bias"),
]


def _mask(kind, b, n_k, gen):
    if kind is None:
        return None
    m = torch.rand(b, n_k, generator=gen) > 0.15
    if kind == "edges":
        m[:] = False
        m[:, [31, 32, 63, 64, 95, 96, 127, 128]] = True
    elif kind == "tile-off":
        m[:] = True
        m[:, 128:256] = False
    elif kind == "row-dead":
        m[0] = False
    elif kind == "first-block":
        m[:] = True
        m[:, :128] = False
    return m


def _bias(kind, h, n_q, n_k, gen):
    """fp32 [h, n_q, ld] with ld > n_k a multiple of 4 and NaN in the pad columns"""
    if kind is None:
        return None
    ld = (n_k + 3) // 4 * 4 + 4
    bias = torch.full((h, n_q, ld), math.nan)
    val = torch.randn(h, n_q, n_k, generator=gen) * 1.5
    if kind == "inf":
        val[torch.rand(h, n_q, n_k, generator=gen) < 0.1] = -math.inf
        val[:, 5::17] = -math.inf                  # whole rows: those queries see no key
    bias[..., :n_k] = val.to(bf16).float()
    return bias


def make_operands(c, seed):
    """bf16 q, k, v, d_o (on the GPU, in the case's layout), key mask, bias and dropout tuple of one case"""
    gen = torch.Generator().manual_seed(seed)
    b, h, n_q, n_k = c["b"], c["h"], c["n_q"], c["n_k"]
    q = torch.randn(b, n_q, h * 64, generator=gen) * c["qmul"]
    k = torch.randn(b, n_k, 64, generator=gen)
    v = torch.randn(b, n_k, 64, generator=gen)
    d_o = torch.randn(b, n_q, h * 64, generator=gen)
    if c["late"]:
        # one score component that grows along the keys: each row's max sits at its last visible keys, 18 nats above
        # its first ones, so the running max jumps in every tile and the last tile decides the result.  The component
        # stays moderate in q and in k: a dominant one makes dq = scale sum_j dS_j k_j (or dk over q) cancel down to
        # the bf16 rounding of dS, which measures the inputs, not the kernel.
        q.view(b, n_q, h, 64)[..., 0] = 12.0
        k[..., 0] = 12.0 * torch.arange(n_k) / n_k
    q, k, v, d_o = (t.to(bf16).to(DEV) for t in (q, k, v, d_o))
    if c["layout"] == "qslice":
        buf = torch.randn(b, n_q, h * 64 + 128, generator=gen).to(bf16).to(DEV)
        buf[..., 64:64 + h * 64] = q
        q = buf[..., 64:64 + h * 64]
    elif c["layout"] == "kvsplit":
        kv = torch.cat((k, v), dim=-1)
        k, v = kv[..., :64], kv[..., 64:]
    mask = _mask(c["mask"], b, n_k, gen)
    bias = _bias(c["bias"], h, n_q, n_k, gen)
    drop = (c["drop"], 0x5EED_0000_0000_0000 + seed, 7) if c["drop"] > 0 else None
    return q, k, v, d_o, None if mask is None else mask.to(DEV), None if bias is None else bias.to(DEV), drop


def bwd_key_blocks(h, n_q, n_k, causal):
    """(n_iter, qb_min) of every key block of the backward, as csrc/attn_bwd_wgmma.cu walks them"""
    off = n_k - n_q
    n_qblocks = (n_q + TILE - 1) // TILE
    out = []
    for kb in range((n_k + TILE - 1) // TILE):
        k0 = kb * TILE
        qb_min = (k0 - off) // TILE if causal and k0 - off > 0 else 0
        out.append((max(n_qblocks - qb_min, 0) * h, qb_min))
    return out


def run_case(c, seed, *, check_repro=True):
    """kernels and reference on one case -> (per-quantity error tensors, kernel outputs, reference outputs)"""
    from audiolm_pytorch_b200 import ops

    q, k, v, d_o, mask, bias, drop = make_operands(c, seed)
    b, h, n_q, n_k = c["b"], c["h"], c["n_q"], c["n_k"]
    kw = dict(heads=h, key_mask=mask, causal=c["causal"], scale=c["scale"], bias=bias, dropout=drop)
    o, lse = ops.mqa_attn_fwd(q, k, v, **kw)
    dbias = torch.zeros_like(bias) if bias is not None else None
    dq, dk, dv = ops.mqa_attn_bwd(q, k, v, o, d_o, lse, dbias=dbias, **kw)
    torch.cuda.synchronize()
    got = dict(o=o, lse=lse[..., :n_q].to(f64) * LN2, dq=dq, dk=dk, dv=dv,
               dbias=None if dbias is None else dbias[..., :n_k].clone())
    if check_repro:
        o2, lse2 = ops.mqa_attn_fwd(q, k, v, **kw)
        _, dk2, dv2 = ops.mqa_attn_bwd(q, k, v, o, d_o, lse, dbias=dbias, **kw)   # dbias accumulates a second time
        torch.cuda.synchronize()
        assert torch.equal(o, o2) and torch.equal(lse[..., :n_q], lse2[..., :n_q]), "forward not bitwise reproducible"
        assert torch.equal(dk, dk2) and torch.equal(dv, dv2), "dk / dv not bitwise reproducible"
    keep = keep_factors(b, h, n_q, n_k, *drop) if drop is not None else None
    ref = attend_fp64(q, k, v, d_o, heads=h, key_mask=mask, causal=c["causal"], scale=c["scale"], bias=bias, keep=keep,
                      o_bwd=o)
    for name in ("o", "dq", "dk", "dv"):
        assert torch.isfinite(got[name]).all(), f"{name} is not finite"
    dead = torch.isinf(ref["lse"])
    assert torch.equal(torch.isinf(got["lse"]), dead), "rows without a visible key and rows with +inf lse differ"
    assert (got["lse"][dead] > 0).all() and torch.isfinite(got["lse"][~dead]).all()
    errs = dict(
        o=row_err(got["o"].view(b, n_q, h, 64), ref["o"].view(b, n_q, h, 64)),
        dq=row_err(got["dq"].view(b, n_q, h, 64), ref["dq"].view(b, n_q, h, 64)),
        dk=row_err(got["dk"], ref["dk"]),
        dv=row_err(got["dv"], ref["dv"]),
        lse=(got["lse"][~dead].to(f64) - ref["lse"][~dead]).abs(),
    )
    if bias is not None:
        assert torch.isfinite(got["dbias"]).all() and (dbias[..., n_k:] == 0).all()
        errs["dbias"] = row_err(got["dbias"], ref["dbias"])
        if check_repro:
            errs["dbias-2x"] = row_err(dbias[..., :n_k], 2 * ref["dbias"])
    return errs, got, ref


def check_errs(errs, tag):
    worst = {q: (e.max().item() if e.numel() else 0.0) for q, e in errs.items()}
    print(f"[err] {tag} " + " ".join(f"{q}={w:.3e}" for q, w in worst.items()))
    for q, w in worst.items():
        bound = BOUND_LSE if q == "lse" else BOUND[q.split("-")[0]]
        assert w <= bound, (q, w, bound)


@pytest.mark.gpu
@pytest.mark.parametrize("c", CASES)
def test_attention_matches_fp64(c, request):
    seed = (c["b"] * 131 + c["h"] * 17 + c["n_q"] * 7 + c["n_k"]) % 100003
    errs, _, _ = run_case(c, seed)
    check_errs(errs, request.node.callspec.id)


# ---- exact probes: one visible key per row ---------------------------------------------------------------------------
PROBE_KEYS = [0, 31, 32, 63, 64, 95, 96, 127, 128, 260, 299]   # every word edge of a tile; 260, 299: last partial tile


@pytest.mark.gpu
@pytest.mark.parametrize("causal,n_q", [(False, 300), (True, 300), (True, 170)], ids=["noncausal", "causal", "causal-off130"])
def test_single_visible_key_is_exact(causal, n_q):
    """batch row r masks every key except j = PROBE_KEYS[r]: a row that sees j gets P = ex2(0) = 1 and l = 1, so o is
    v[j] bitwise and the LSE is the scaled score of j; a row that cannot see j gets o = 0 and lse = +inf.  In the
    backward dv[j] is the sum of the dO rows that see j, every other dk / dv row is 0, and dq, dk vanish up to
    rounding (dS = P (dP - delta) with delta = dO . v[j] = dP)."""
    from audiolm_pytorch_b200 import ops

    n_k, h = 300, 3
    b = len(PROBE_KEYS)
    gen = torch.Generator().manual_seed(n_q + int(causal))
    q = torch.randn(b, n_q, h * 64, generator=gen).to(bf16).to(DEV)
    k = torch.randn(b, n_k, 64, generator=gen).to(bf16).to(DEV)
    v = torch.randn(b, n_k, 64, generator=gen).to(bf16).to(DEV)
    d_o = torch.randn(b, n_q, h * 64, generator=gen).to(bf16).to(DEV)
    mask = torch.zeros(b, n_k, dtype=torch.bool, device=DEV)
    js = torch.tensor(PROBE_KEYS, device=DEV)
    mask[torch.arange(b, device=DEV), js] = True
    o, lse = ops.mqa_attn_fwd(q, k, v, heads=h, key_mask=mask, causal=causal)
    dq, dk, dv = ops.mqa_attn_bwd(q, k, v, o, d_o, lse, heads=h, key_mask=mask, causal=causal)
    torch.cuda.synchronize()
    off = n_k - n_q
    sees = (torch.arange(n_q, device=DEV)[None, :] + off >= js[:, None]) if causal else torch.ones(b, n_q, dtype=torch.bool, device=DEV)
    vj = v[torch.arange(b, device=DEV), js]                                  # [b, 64]
    oh = o.view(b, n_q, h, 64)
    want = torch.where(sees[..., None, None], vj[:, None, None, :], torch.zeros((), dtype=bf16, device=DEV))
    assert torch.equal(oh, want.expand_as(oh)), "o is not v[j] bitwise on rows that see j, or not 0 on the others"
    kj = k[torch.arange(b, device=DEV), js].to(f64)
    score = torch.einsum("bihd,bd->bhi", q.view(b, n_q, h, 64).to(f64), kj) * 64 ** -0.5
    lse_n = lse[..., :n_q].to(f64) * LN2
    seen3 = sees[:, None, :].expand(b, h, n_q)
    assert torch.isinf(lse_n[~seen3]).all() and (lse_n[~seen3] > 0).all()
    assert (lse_n[seen3] - score[seen3]).abs().max().item() <= BOUND_LSE
    # backward
    dv_j = (d_o.view(b, n_q, h, 64).to(f64) * sees[..., None, None]).sum((1, 2))   # [b, 64]
    got_dv_j = dv[torch.arange(b, device=DEV), js]
    err = row_err(got_dv_j, dv_j)
    print(f"[err] probe causal={causal} n_q={n_q} dv={err.max().item():.3e} dq={dq.float().abs().max().item():.3e} "
          f"dk={dk.float().abs().max().item():.3e}")
    assert err.max().item() <= BOUND["dv"], err.tolist()
    others = ~mask
    assert (dv[others] == 0).all() and (dk[others] == 0).all(), "a masked key received a gradient"
    assert dq.float().abs().max().item() <= BOUND_PROBE_ABS
    assert dk.float().abs().max().item() <= BOUND_PROBE_ABS


# ---- hygiene: NaN in the LSE pads never reaches a result -------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("n_q,n_k,masked", [(100, 128, False), (300, 300, True)], ids=["one-key-block", "three-key-blocks"])
def test_lse_pad_nan_does_not_leak(n_q, n_k, masked):
    """the backward reads the LSE in 128-row blocks; rows n_q.. are padding that its branch-free selects must drop.
    With one key block every dq element has a single reduce-add, so dq is bitwise comparable too."""
    from audiolm_pytorch_b200 import ops

    b, h = 2, 3
    gen = torch.Generator().manual_seed(n_q)
    q = torch.randn(b, n_q, h * 64, generator=gen).to(bf16).to(DEV)
    k = torch.randn(b, n_k, 64, generator=gen).to(bf16).to(DEV)
    v = torch.randn(b, n_k, 64, generator=gen).to(bf16).to(DEV)
    d_o = torch.randn(b, n_q, h * 64, generator=gen).to(bf16).to(DEV)
    mask = (torch.rand(b, n_k, generator=gen) > 0.15).to(DEV) if masked else None
    o, lse = ops.mqa_attn_fwd(q, k, v, heads=h, key_mask=mask)
    assert lse.shape[-1] > n_q
    dq, dk, dv = ops.mqa_attn_bwd(q, k, v, o, d_o, lse, heads=h, key_mask=mask)
    lse_nan = lse.clone()
    lse_nan[..., n_q:] = math.nan
    dq2, dk2, dv2 = ops.mqa_attn_bwd(q, k, v, o, d_o, lse_nan, heads=h, key_mask=mask)
    torch.cuda.synchronize()
    assert torch.isfinite(dq2.float()).all() and torch.isfinite(dk2.float()).all() and torch.isfinite(dv2.float()).all()
    assert torch.equal(dk, dk2) and torch.equal(dv, dv2)
    if n_k <= TILE:
        assert torch.equal(dq, dq2)
    else:
        assert row_err(dq2.view(b, n_q, h, 64), dq.view(b, n_q, h, 64)).max().item() <= 1e-2


# ---- batches past the 65535 limit of grid.y / grid.z -----------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("masked", [False, True], ids=["no-mask", "key-mask"])
def test_batch_past_grid_yz_limit(masked):
    """the local attention calls the kernels with batch = clips x heads x windows (about 2,800 per 10-minute clip):
    b = 70,000 must run and match"""
    c = dict(b=70000, h=1, n_q=1, n_k=2, causal=True, mask="random" if masked else None, bias=None, layout="contig",
             scale=None, qmul=1.0, late=False, drop=0.0)
    errs, _, _ = run_case(c, 70000 + int(masked), check_repro=False)
    check_errs(errs, f"b70000-{'mask' if masked else 'nomask'}")


@pytest.mark.gpu
def test_local_attention_shape():
    """the call of LocalMHA (local_attn.py): one head, 128 queries against the 256 keys of two windows, unit-norm
    q / k with scale 8, a shared [1, 128, 256] bias with -1e30 entries, the look-back half of every first window
    masked; b = 8 heads x 64 windows"""
    from audiolm_pytorch_b200 import ops

    b, w, heads, windows = 512, 128, 8, 64
    gen = torch.Generator().manual_seed(512)
    q = F.normalize(torch.randn(b, w, 64, generator=gen), dim=-1).to(bf16).to(DEV)
    k = F.normalize(torch.randn(b, 2 * w, 64, generator=gen), dim=-1).to(bf16).to(DEV)
    v = torch.randn(b, 2 * w, 64, generator=gen).to(bf16).to(DEV)
    d_o = torch.randn(b, w, 64, generator=gen).to(bf16).to(DEV)
    j = torch.arange(2 * w)[None, :]
    r = torch.arange(w)[:, None]
    bias = torch.where(j < r, -1e30, 0.0)[None].float().to(DEV)               # [1, 128, 256]
    mask = torch.ones(b, 2 * w, dtype=torch.bool, device=DEV)
    mask.view(heads, windows, 2 * w)[:, 0, :w] = False
    kw = dict(heads=1, key_mask=mask, causal=True, scale=8.0, bias=bias)
    o, lse = ops.mqa_attn_fwd(q, k, v, **kw)
    dbias = torch.zeros_like(bias)
    dq, dk, dv = ops.mqa_attn_bwd(q, k, v, o, d_o, lse, dbias=dbias, **kw)
    torch.cuda.synchronize()
    ref = attend_fp64(q, k, v, d_o, o_bwd=o, **kw)
    errs = dict(o=row_err(o.view(b, w, 1, 64), ref["o"].view(b, w, 1, 64)),
                dq=row_err(dq.view(b, w, 1, 64), ref["dq"].view(b, w, 1, 64)),
                dk=row_err(dk, ref["dk"]), dv=row_err(dv, ref["dv"]),
                dbias=row_err(dbias, ref["dbias"]),
                lse=(lse[..., :w].to(f64) * LN2 - ref["lse"]).abs())
    check_errs(errs, "local-attention")


# ---- host: the reference against torch SDPA, and the case list's coverage -------------------------------------------
def _sdpa_fp64(q, k, v, d_o, *, heads, key_mask, causal, scale, bias):
    """torch SDPA in fp64 on the CPU over the same operands; rows that see no key are given an all-visible mask and a
    zero output gradient (SDPA returns NaN there) and are left out of the comparison by the caller"""
    b, n_q, hd = q.shape
    n_k = k.shape[1]
    qh = q.to(f64).view(b, n_q, heads, 64).permute(0, 2, 1, 3).requires_grad_()
    kf = k.to(f64).requires_grad_()
    vf = v.to(f64).requires_grad_()
    add = torch.zeros(b, heads, n_q, n_k, dtype=f64)
    bf = None
    if bias is not None:
        bf = bias[..., :n_k].to(f64).requires_grad_()
        add = add + bf
    vis = torch.ones(b, 1, n_q, n_k, dtype=torch.bool)
    if key_mask is not None:
        vis = vis & key_mask[:, None, None, :]
    if causal:
        vis = vis & ~torch.ones(n_q, n_k, dtype=torch.bool).triu(n_k - n_q + 1)
    vis = vis & (add.detach() > -math.inf)
    dead = ~vis.any(-1, keepdim=True)
    add = torch.where(vis | dead, add, -math.inf)
    add = torch.where(dead, 0.0, add)
    o = F.scaled_dot_product_attention(qh, kf[:, None].expand(b, heads, n_k, 64), vf[:, None].expand(b, heads, n_k, 64),
                                       attn_mask=add, scale=scale)
    g = d_o.to(f64).view(b, n_q, heads, 64).permute(0, 2, 1, 3) * ~dead
    o.backward(g)
    lse = torch.logsumexp(torch.einsum("bhid,bjd->bhij", qh.detach(), kf.detach()) * scale + add.detach(), -1)
    return dict(o=o.detach().permute(0, 2, 1, 3).reshape(b, n_q, hd), lse=lse, dead=dead[..., 0],
                dq=qh.grad.permute(0, 2, 1, 3).reshape(b, n_q, hd), dk=kf.grad, dv=vf.grad,
                dbias=None if bf is None else bf.grad)


@pytest.mark.parametrize("causal,n_q,n_k,masked,bias_kind,scale", [
    (True, 7, 7, False, None, None),
    (True, 5, 13, True, None, 0.3),
    (False, 6, 11, True, "rand", None),
    (True, 9, 20, True, "inf", 8.0),
    (False, 4, 4, False, "inf", None),
])
def test_reference_matches_sdpa(causal, n_q, n_k, masked, bias_kind, scale):
    """attend_fp64 against torch's SDPA in fp64, outputs, LSE and every gradient, on rows that see at least one key"""
    gen = torch.Generator().manual_seed(n_q * 31 + n_k)
    b, h = 3, 2
    q = torch.randn(b, n_q, h * 64, generator=gen).to(bf16)
    k = torch.randn(b, n_k, 64, generator=gen).to(bf16)
    v = torch.randn(b, n_k, 64, generator=gen).to(bf16)
    d_o = torch.randn(b, n_q, h * 64, generator=gen).to(bf16)
    mask = None
    if masked:
        mask = torch.rand(b, n_k, generator=gen) > 0.3
        mask[0] = False                        # a batch row that sees nothing
    bias = _bias(bias_kind, h, n_q, n_k, gen)
    kw = dict(heads=h, key_mask=mask, causal=causal, scale=scale if scale is not None else 64 ** -0.5, bias=bias)
    got = attend_fp64(q, k, v, d_o, **kw)
    want = _sdpa_fp64(q, k, v, d_o, **kw)
    dead = want["dead"]                                         # [b, h, n_q]
    assert dead.any() or not masked
    live_rows = ~dead.permute(0, 2, 1)                          # [b, n_q, h]
    go, wo = got["o"].view(b, n_q, h, 64), want["o"].view(b, n_q, h, 64)
    assert torch.allclose(go[live_rows], wo[live_rows], rtol=1e-10, atol=1e-12)
    assert (go[~live_rows] == 0).all()
    assert torch.allclose(got["lse"][~dead], want["lse"][~dead], rtol=1e-10, atol=1e-12)
    assert torch.isinf(got["lse"][dead]).all() and (got["lse"][dead] > 0).all()
    for name in ("dq", "dk", "dv") + (("dbias",) if bias is not None else ()):
        assert torch.allclose(got[name], want[name], rtol=1e-9, atol=1e-11), name
    gq = got["dq"].view(b, n_q, h, 64)
    assert (gq[~live_rows] == 0).all()


def test_reference_applies_keep_factors():
    """with dropout factors the output is (P o Z) V while the LSE stays that of P; all-ones factors change nothing"""
    gen = torch.Generator().manual_seed(3)
    b, h, n_q, n_k = 2, 2, 5, 9
    q = torch.randn(b, n_q, h * 64, generator=gen).to(bf16)
    k = torch.randn(b, n_k, 64, generator=gen).to(bf16)
    v = torch.randn(b, n_k, 64, generator=gen).to(bf16)
    base = attend_fp64(q, k, v, heads=h)
    ones = attend_fp64(q, k, v, heads=h, keep=torch.ones(b, h, n_q, n_k))
    assert torch.equal(base["o"], ones["o"])
    Z = keep_factors(b, h, n_q, n_k, 0.5, 1234, 5)
    assert set(Z.unique().tolist()) <= {0.0, 2.0} and (Z == 0).any() and (Z > 0).any()
    got = attend_fp64(q, k, v, heads=h, keep=Z)
    qh = q.to(f64).view(b, n_q, h, 64).permute(0, 2, 1, 3)
    s = torch.einsum("bhid,bjd->bhij", qh, k.to(f64)) / 8
    s = s.masked_fill(torch.ones(n_q, n_k, dtype=torch.bool).triu(n_k - n_q + 1), -math.inf)
    want = torch.einsum("bhij,bjd->bhid", s.softmax(-1) * Z, v.to(f64)).permute(0, 2, 1, 3).reshape(b, n_q, h * 64)
    assert torch.allclose(got["o"], want, rtol=1e-12, atol=1e-14)
    assert torch.equal(got["lse"], base["lse"])


def test_cases_cover_the_envelope():
    """the case list hits every n_q / n_k residue and causal offset named in the module docstring, both sides of every
    tile edge, 1-24 heads, batch 1 / 2 / 5, and backward key blocks with 1, 2, 3, 4 and more than 3 x AB_STAGES
    iterations starting past query block 0"""
    cs = [p.values[0] for p in CASES]
    n_q = {c["n_q"] for c in cs}
    n_k = {c["n_k"] for c in cs}
    sizes = {1, 63, 64, 65, 127, 128, 129, 255, 256, 257, 2048}
    assert sizes <= n_q and sizes <= n_k, (sizes - n_q, sizes - n_k)
    offs = {c["n_k"] - c["n_q"] for c in cs if c["causal"]}
    assert {0, 1, 126, 127, 128, 129, 200} <= offs, offs
    assert {1, 3, 8, 16, 24} <= {c["h"] for c in cs}
    assert {1, 2, 5} <= {c["b"] for c in cs}
    assert {True, False} == {c["causal"] for c in cs}
    for kind in ("random", "edges", "tile-off", "row-dead", "first-block"):
        assert any(c["mask"] == kind for c in cs), kind
    assert {"qslice", "kvsplit"} <= {c["layout"] for c in cs}
    assert any(c["drop"] > 0 for c in cs) and any(c["late"] for c in cs) and any(c["scale"] for c in cs)
    assert {4.0, 8.0} <= {c["qmul"] for c in cs}
    iters = set()
    for c in cs:
        iters |= {(n if n <= 4 else "many", qb_min > 0)
                  for n, qb_min in bwd_key_blocks(c["h"], c["n_q"], c["n_k"], c["causal"])
                  if n <= 4 or n > 3 * AB_STAGES}
    assert {(1, True), (2, True), (3, True), (4, True), ("many", True), ("many", False)} <= iters, iters


def test_reference_backward_from_a_given_output():
    """with o_bwd the gradients are those of dS = P (Z dP - delta), delta = rowsum(dO o_bwd), written out by hand"""
    gen = torch.Generator().manual_seed(11)
    b, h, n_q, n_k, scale = 2, 3, 6, 10, 0.2
    q = torch.randn(b, n_q, h * 64, generator=gen).to(bf16)
    k = torch.randn(b, n_k, 64, generator=gen).to(bf16)
    v = torch.randn(b, n_k, 64, generator=gen).to(bf16)
    d_o = torch.randn(b, n_q, h * 64, generator=gen).to(bf16)
    bias = _bias("rand", h, n_q, n_k, gen)
    mask = torch.rand(b, n_k, generator=gen) > 0.3
    mask[1] = False
    Z = keep_factors(b, h, n_q, n_k, 0.3, 77, 2)
    kw = dict(heads=h, key_mask=mask, causal=True, scale=scale, bias=bias, keep=Z)
    o_given = attend_fp64(q, k, v, **kw)["o"].to(bf16)
    got = attend_fp64(q, k, v, d_o, o_bwd=o_given, **kw)
    qh = q.to(f64).view(b, n_q, h, 64).permute(0, 2, 1, 3)
    s = torch.einsum("bhid,bjd->bhij", qh, k.to(f64)) * scale + bias[..., :n_k].to(f64)
    vis = mask[:, None, None, :] & ~torch.ones(n_q, n_k, dtype=torch.bool).triu(n_k - n_q + 1)
    P = torch.softmax(s.masked_fill(~vis, -math.inf), -1).nan_to_num(0.0)
    g = d_o.to(f64).view(b, n_q, h, 64).permute(0, 2, 1, 3)
    dP = torch.einsum("bhid,bjd->bhij", g, v.to(f64))
    delta = (g * o_given.to(f64).view(b, n_q, h, 64).permute(0, 2, 1, 3)).sum(-1, keepdim=True)
    dS = P * (Z * dP - delta)
    dq = (torch.einsum("bhij,bjd->bhid", dS, k.to(f64)) * scale).permute(0, 2, 1, 3).reshape(b, n_q, h * 64)
    dk = torch.einsum("bhij,bhid->bjd", dS, qh) * scale
    assert torch.allclose(got["dq"], dq, rtol=1e-10, atol=1e-12)
    assert torch.allclose(got["dk"], dk, rtol=1e-10, atol=1e-12)
    assert torch.allclose(got["dbias"], dS.sum(0), rtol=1e-10, atol=1e-12)
    assert torch.allclose(got["dv"], torch.einsum("bhij,bhid->bjd", P * Z, g), rtol=1e-10, atol=1e-12)


def test_keep_factors_follow_the_counter_rows():
    """keep_factors reads the numpy mask at row (batch * h + head) * n_q_pad + i, the kernels' counter row"""
    import numpy as np

    b, h, n_q, n_k, p = 2, 3, 130, 20, 0.25
    Z = keep_factors(b, h, n_q, n_k, p, 99, 4)
    for bb, hh, i in [(0, 0, 0), (1, 2, 129), (1, 0, 77)]:
        row = (bb * h + hh) * 256 + i
        want = dropout_ref.keep(99, 4, [row], np.arange(n_k), p)[0]
        assert np.array_equal(Z[bb, hh, i].numpy() > 0, want)
