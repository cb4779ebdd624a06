"""References for the nearest-code search (ops.rvq_encode_tc / nearest_centroid, ops.rvq_encode, ops.rvq_decode).

The rule every search kernel implements is vector-quantize-pytorch's eval path (restated in
oracle/third_party.py::euclid_nearest): per stage  id = argmin_c sqrt(max(|r|^2 + |e_c|^2 - 2 r.e_c, 0)) in fp32,
lowest index on ties;  r -= e_id;  quantized += e_id.

Two references:

* integer lattices (`lattice`): every operand is an integer and every intermediate of the fp32 expansion
  (|r|^2, |e|^2, any partial sum of r.e, |r|^2 + |e|^2, the difference) is an integer below 2^24, so the fp32
  distance is exact in any summation order and the kernel's rule has one answer: `exact_search`.  The values carry
  9 significant bits, one more than bf16 keeps, so the split-bf16 scores of the tensor-core GEMM drop r_lo * e_lo
  terms and rank the codes wrongly while the fp32 re-rank stays exact; codes are `base + small perturbations` and
  rows sit near `base`, so near-ties and exact ties are common.

* continuous inputs (`check_fp64`): the stages are replayed with the kernel's own ids (the residual in fp32, exactly
  as the kernels update it), each stage's distances are taken in fp64, and the chosen code must lie within the
  rigorous error band of the fp32 expansion around the fp64 minimum.

Band of the fp32 expansion.  With u = 2^-24 and gamma_n = n u / (1 - n u), any fp32 evaluation of an n-term dot
product in any order (FMA chains, lane partials, shuffle trees, the GEMM's accumulator) is within
gamma_n * sum |a_i b_i| of the exact value.  |r|^2, |e|^2 and r.e are D-term dot products; the sum |r|^2 + |e|^2 and
the subtraction of 2 r.e (exact scaling by 2) add one rounding each, so the computed f satisfies
    |f - |r - e|^2| <= gamma_{D+2} (|r|^2 + |e|^2 + 2 |r| |e|) = gamma_{D+2} (|r| + |e|)^2 =: tau(r, e).
The kernels compare fl(sqrt(max(f, 0))); a correctly rounded sqrt is monotone and moves by at most one rounding, so
sqrt32(f_a) <= sqrt32(f_b) implies f_a <= f_b (1 + u)^2 / (1 - u)^2 <= f_b (1 + 5u).  Hence the chosen code a and
the fp64 argmin b satisfy
    d2_a - d2_b <= tau_a + tau_b + 5u (d2_b + tau_b),
and where every other code is further than that from the minimum, the id must be the fp64 argmin.
"""

import torch

U = 2.0 ** -24
CAND_TOL = 1e-4        # rvq_tc.cu select_kernel: candidates within CAND_TOL * (|r|^2 + |e|^2) of the best score
SMEM_CAP = 200 * 1024  # shared-memory cap of alm_rvq_encode's two kernels (csrc/codec.cu)


def gamma(n):
    return n * U / (1 - n * U)


# ---- restated guards of the search entry points ---------------------------------------------------------------------
def rvq_encode_path(D, aligned=True):
    """the kernel alm_rvq_encode (csrc/codec.cu) launches for width D, or None where it returns an error:
    'v2' for D % 32 == 0, a 16-byte aligned codebook and its shared memory under the cap, else 'v1' (D % 4 == 0,
    float4 rows) under the cap."""
    if D <= 0 or D % 4:
        return None
    if D % 32 == 0 and aligned:
        smem2 = (32 * (D + 4) + 2 * 256 * 36 + 32 + 2 * 32) * 4 + 3 * 32 * 4
        if smem2 <= SMEM_CAP:
            return "v2"
    smem1 = ((32 + 32) * (D + 4) + 2 * 32) * 4
    return "v1" if smem1 <= SMEM_CAP else None


def search_width(D):
    """ops.rvq_search_width: the tensor-core search pads D to a multiple of 8 (3D is the score GEMM's row pitch)"""
    return -(-D // 8) * 8


# ---- integer lattices -------------------------------------------------------------------------------------------------
def lattice(D, C, N, Q=1, *, nnz=32, seed=0):
    """(x [N, D], codebooks [Q, C, D]) fp32 integer lattice; stage s lives on its own k = min(nnz, D) // Q columns
    (columns 0 and D - 1 always among them), so every stage sees a near-tie lattice of its own and the residual of the
    others is a constant that changes no argmin.  Per stage: base values +-[260, 500], codes base + [-2, 2], rows
    base + [-3, 3].  Special rows and codes: row 0 is x = 0; rows 1..3 equal codewords; codes 1, 129 and C - 1
    (where they exist) are one duplicated "dead" codeword, and row 4 equals it, so the lowest index must win across
    a 128-code group boundary and a 256-code tile."""
    g = torch.Generator().manual_seed(seed)
    k = max(1, min(nnz, D) // Q)
    assert k * Q <= D, "not enough columns for a support per stage"
    inner = torch.randperm(D - 2, generator=g)[: max(0, k * Q - 2)] + 1 if D > 2 else torch.empty(0, dtype=torch.long)
    cols = torch.cat([torch.tensor([0, D - 1][: min(2, k * Q)]), inner])
    cols = cols[torch.randperm(cols.numel(), generator=g)].view(Q, k)
    x = torch.zeros(N, D, dtype=torch.float64)
    cb = torch.zeros(Q, C, D, dtype=torch.float64)
    for s in range(Q):
        sign = torch.randint(0, 2, (k,), generator=g) * 2 - 1
        base = (sign * torch.randint(260, 501, (k,), generator=g)).double()
        codes = base + torch.randint(-2, 3, (C, k), generator=g).double()
        dead = [c for c in (1, 129, C - 1) if c < C]
        codes[dead] = base + torch.randint(-2, 3, (k,), generator=g).double()
        rows = base + torch.randint(-3, 4, (N, k), generator=g).double()
        for i, c in zip(range(1, 4), (0, C // 2, C - 1)):
            if i < N:
                rows[i] = codes[c]
        if N > 4:
            rows[4] = codes[dead[-1]]
        cb[s][:, cols[s]] = codes
        x[:, cols[s]] = rows
    x[0] = 0
    return x.float(), cb.float()


def exactness_violations(x, cb, ids):
    """the lattice invariants along the stages `ids` takes, False when they hold: integer operands; at every stage
    |r|^2 + |e|^2 < 2^24 (so |r|^2, |e|^2, every partial sum of r.e and the sum are exact) and r.e >= 0 (so the
    difference d^2 = |r|^2 + |e|^2 - 2 r.e lies in [0, |r|^2 + |e|^2] and is exact too)"""
    r, cb64 = x.double(), cb.double()
    if not (torch.equal(r, r.round()) and torch.equal(cb64, cb64.round())):
        return "non-integer operand"
    for s in range(cb.shape[0]):
        e = cb64[s]
        top = (r * r).sum(1).max() + (e * e).sum(1).max()
        if top >= 2 ** 24:
            return f"stage {s}: |r|^2 + |e|^2 = {top.item():.0f} >= 2^24"
        if (r @ e.T).min() < 0:
            return f"stage {s}: r.e < 0"
        r = r - e[ids[:, s]]
    return False


def bf16_split(v):
    """split_bf16 of ptx_sm90.cuh: hi = bf16(v), lo = bf16(v - hi) (round to nearest even, as __float2bfloat16_rn)"""
    hi = v.to(torch.bfloat16).float()
    return hi, (v - hi).to(torch.bfloat16).float()


def split_scores(r, e):
    """the score GEMM's product R' B'^T = r_hi.e_hi + r_lo.e_hi + r_hi.e_lo, in fp64 (no accumulation error)"""
    rh, rl = (t.double() for t in bf16_split(r.float()))
    eh, el = (t.double() for t in bf16_split(e.float()))
    return rh @ eh.T + rl @ eh.T + rh @ el.T


def _d2(r64, e64):
    return (r64 * r64).sum(1, keepdim=True) + (e64 * e64).sum(1)[None] - 2.0 * (r64 @ e64.T)


def exact_search(x, cb):
    """the kernels' rule on a lattice: fp32 sqrt of the exact d^2, first minimum; -> (quantized fp32, ids int64)"""
    r = x.double()
    quant = torch.zeros_like(x)
    ids = []
    for s in range(cb.shape[0]):
        e = cb[s].double()
        i = torch.sqrt(_d2(r, e).float()).argmin(1)
        ids.append(i)
        r = r - e[i]
        quant = quant + cb[s][i]
    return quant, torch.stack(ids, 1)


# ---- continuous inputs ----------------------------------------------------------------------------------------------
def replay(x, cb, ids):
    """quantized as the kernels accumulate it (fp32, q = 0; q = q + cb[s][id_s] in stage order) and the fp32
    residual before every stage"""
    r, q = x.float().clone(), torch.zeros_like(x, dtype=torch.float32)
    residuals = []
    for s in range(cb.shape[0]):
        residuals.append(r)
        e = cb[s][ids[:, s]]
        r = r - e
        q = q + e
    return q, residuals


def check_fp64(x, cb, ids, *, quant=None, margin=None, label=""):
    """asserts the band criterion of the module docstring at every stage, and (when given) quantized bit for bit
    against `replay`; with `margin`, also the fp64 argmin on every row whose best and second-best distances (not
    squared) are more than `margin` apart.  -> (share of (row, stage) pairs whose fp64 minimum is not isolated by
    the band, share of pairs farther apart than `margin`)"""
    D = x.shape[1]
    q, residuals = replay(x, cb, ids)
    if quant is not None:
        assert torch.equal(quant.view(torch.int32), q.view(torch.int32)), f"{label}: quantized != fp32 replay"
    g = gamma(D + 2)
    in_band = safe = 0
    for s, r in enumerate(residuals):
        r64, e64 = r.double(), cb[s].double()
        d2 = _d2(r64, e64)
        tau = g * (r64.norm(dim=1, keepdim=True) + e64.norm(dim=1)[None]) ** 2
        slack = 1e-13 * (r64.norm(dim=1, keepdim=True) + e64.norm(dim=1)[None]) ** 2   # fp64 expansion error
        best = d2.argmin(1, keepdim=True)
        d2b, taub = d2.gather(1, best), tau.gather(1, best)
        band = tau + taub + 5 * U * (d2b.abs() + taub) + slack
        i = ids[:, s:s + 1]
        gap = d2.gather(1, i) - d2b
        bad = gap > band.gather(1, i)
        assert not bad.any(), (f"{label} stage {s}: {int(bad.sum())} rows chose a code outside the fp32 band, worst "
                               f"gap / band {(gap / band.gather(1, i)).max().item():.3g}")
        near = ((d2 - d2b) <= band).sum(1) > 1
        assert torch.equal(i[~near], best[~near]), f"{label} stage {s}: isolated minimum not chosen"
        in_band += int(near.sum())
        if margin is not None and d2.shape[1] > 1:
            top2 = d2.clamp_min(0).sqrt().topk(2, dim=1, largest=False).values
            far = (top2[:, 1] - top2[:, 0]) > margin
            assert torch.equal(i[far], best[far]), f"{label} stage {s}: a row {margin} clear of the next code differs"
            safe += int(far.sum())
    pairs = x.shape[0] * cb.shape[0]
    return in_band / pairs, safe / pairs


# ---- continuous generators ------------------------------------------------------------------------------------------
def gaussian(N, C, D, Q=1, *, g, x_scale=1.0):
    return torch.randn(N, D, generator=g) * x_scale, torch.randn(Q, C, D, generator=g)


def clustered(N, C, D, Q=1, *, g, spread=1e-3):
    """k-means-like: centers = base + spread |base| noise per stage, rows near centers (the residual of stage s is
    what stage s + 1 clusters)"""
    base = torch.randn(Q, 1, D, generator=g)
    cb = base + spread * torch.randn(Q, C, D, generator=g)
    ids = torch.randint(0, C, (Q, N), generator=g)
    x = sum(cb[s][ids[s]] for s in range(Q)) + 0.5 * spread * torch.randn(N, D, generator=g)
    return x, cb


def offset(N, C, D, Q=1, *, g, level=30.0):
    """HuBERT-like features: one large common offset, |x| >> the spread of the centers"""
    common = level * torch.randn(D, generator=g)
    cb = common + torch.randn(Q, C, D, generator=g)
    return common + 1.2 * torch.randn(N, D, generator=g), cb


def shrinking(N, C, D, Q=8, *, g, ratio=0.6):
    """Q stages whose scales shrink geometrically (ratio^Q spans orders of magnitude): x = sum of one code per stage
    plus noise below the last stage's scale"""
    scales = ratio ** torch.arange(Q, dtype=torch.float32)
    cb = torch.randn(Q, C, D, generator=g) * scales[:, None, None]
    ids = torch.randint(0, C, (Q, N), generator=g)
    x = sum(cb[s][ids[s]] for s in range(Q)) + 0.3 * scales[-1] * torch.randn(N, D, generator=g)
    return x, cb


GENERATORS = {"gaussian": gaussian, "clustered": clustered, "offset": offset, "shrinking": shrinking}


# (D, C, N, Q) of the lattice cases the GPU suite runs; the host suite checks each one still stresses the kernels
LATTICE_GRID = [
    (8, 1, 7, 1), (8, 33, 37, 2), (24, 2, 1, 1), (24, 31, 4000, 1), (64, 320, 37, 8), (64, 500, 2000, 32),
    (128, 1024, 4000, 2), (128, 1024, 1000, 32), (256, 512, 4000, 1), (256, 33, 3000, 8), (512, 4096, 3000, 1),
    (512, 1024, 2000, 8), (512, 2, 7, 32), (768, 500, 4000, 1), (1024, 500, 3000, 2), (1024, 4096, 37, 1),
]
