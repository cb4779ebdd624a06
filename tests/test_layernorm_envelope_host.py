"""Host checks of the LayerNorm envelope tests (test_layernorm_envelope_gpu.py), without a GPU:

* the fp64 references of tests/layernorm_ref.py against an independent float64 NumPy LayerNorm, forward and backward;
* the criterion's sensitivity: an fp32 emulation of the kernels' statistics on the ill-conditioned family passes with
  a two-pass variance and is rejected by at least 10x the bound with a one-pass variance E[v^2] - mean^2;
* the case lists reach every template and launch layout alm_geglu_ln_fwd / _bwd select, and the row counts around
  their grid caps."""
import math
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
import layernorm_ref as lr  # noqa: E402
from test_layernorm_envelope_gpu import BOUND, GEGLU_CASES, RESID_CASES  # noqa: E402

bf16, f32, f64 = torch.bfloat16, torch.float32, torch.float64


# ---- an independent float64 NumPy LayerNorm --------------------------------------------------------------------------
def np_gelu(x):
    from scipy.special import erf

    return 0.5 * x * (1 + erf(x / math.sqrt(2)))


def np_ln_fwd_bwd(v, gamma, dy):
    """y = (v - mean) / sqrt(var + eps) gamma and (dv, dgamma) for the upstream gradient dy"""
    n = v.shape[-1]
    mean = v.sum(-1, keepdims=True) / n
    var = ((v - mean) ** 2).sum(-1, keepdims=True) / n
    rstd = 1.0 / np.sqrt(var + 1e-5)
    xh = (v - mean) * rstd
    g = dy * gamma
    dv = rstd / n * (n * g - g.sum(-1, keepdims=True) - xh * (g * xh).sum(-1, keepdims=True))
    return xh * gamma, dv, (dy * xh).sum(0)


@pytest.mark.parametrize("M,n,dc", [(5, 1, 0.0), (7, 33, 0.0), (4, 2730, 0.0), (3, 1000, 300.0)])
def test_geglu_reference_matches_numpy(M, n, dc):
    g = torch.Generator().manual_seed(n)
    a = (dc + torch.randn(M, n, generator=g)).to(bf16).double()
    gate = (2 * torch.randn(M, n, generator=g)).to(bf16).double()
    gamma = 1 + 0.1 * torch.randn(n, generator=g, dtype=f64)
    Z = (torch.rand(M, n, generator=g) > 0.3).double() / 0.7
    dgn = torch.randn(M, n, generator=g, dtype=f64)
    g0 = torch.randn(n, generator=g, dtype=f64)
    ref = lr.geglu_ln_ref(a, gate, gamma, Z, dgn, g0)
    an, gn_, gmn, zn, dn = (t.numpy() for t in (a, gate, gamma, Z, dgn))
    ge = np_gelu(gn_)
    y, dv, dgam = np_ln_fwd_bwd(ge * an, gmn, dn * zn)
    gp = 0.5 * (1 + __import__("scipy.special", fromlist=["erf"]).erf(gn_ / math.sqrt(2))) \
        + gn_ * np.exp(-0.5 * gn_ ** 2) / math.sqrt(2 * math.pi)
    np.testing.assert_allclose(ref["out"].numpy(), y * zn, rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(ref["da"].numpy(), dv * ge, rtol=1e-8, atol=1e-10)
    np.testing.assert_allclose(ref["dgate"].numpy(), dv * an * gp, rtol=1e-8, atol=1e-10)
    np.testing.assert_allclose(ref["g_gamma"].numpy(), dgam + g0.numpy(), rtol=1e-9, atol=1e-10)
    v = ge * an
    np.testing.assert_allclose(ref["rstd"].numpy(), 1 / np.sqrt(v.var(-1) + 1e-5), rtol=1e-12)


@pytest.mark.parametrize("with_y,out_scale", [(True, 0.5), (False, -2.0)])
def test_resid_reference_matches_numpy(with_y, out_scale):
    g = torch.Generator().manual_seed(3)
    M, d = 6, 1000
    r = 50 + torch.randn(M, d, generator=g, dtype=f64)
    y = torch.randn(M, d, generator=g).to(bf16) if with_y else None
    gamma = 1 + 0.1 * torch.randn(d, generator=g, dtype=f64)
    dxn, dr_out, dextra = (torch.randn(M, d, generator=g, dtype=f64) for _ in range(3))
    g0 = torch.randn(d, generator=g, dtype=f64)
    ref = lr.resid_ln_ref(r, y, gamma, dxn, dr_out, dextra, out_scale, g0)
    v = r.numpy() + (y.double().numpy() if with_y else 0)
    out, dv, dgam = np_ln_fwd_bwd(v, gamma.numpy(), dxn.numpy())
    np.testing.assert_allclose(ref["out"].numpy(), out, rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(ref["dr"].numpy(), out_scale * (dv + dr_out.numpy() + dextra.numpy()), rtol=1e-9,
                               atol=1e-10)
    np.testing.assert_allclose(ref["g_gamma"].numpy(), dgam + g0.numpy(), rtol=1e-9, atol=1e-10)


# ---- the criterion's sensitivity to a one-pass variance ----------------------------------------------------------------
def emulate_geglu_ln_fwd(a, gate, gamma, two_pass):
    """fp32 NumPy emulation of geglu_ln_fwd_kernel: the GELU of alm_common.cuh (gelu_parts), fp32 sums, and the
    variance in two passes or as the one-pass max(E[v^2] - mean^2, 0); rsqrtf as 1 / sqrt in fp32 -> bf16 output"""
    a, x, gm = (t.float().numpy() for t in (a, gate, gamma))
    h = np.float32
    ax = np.abs(x) * h(0.7071067811865476)
    t = h(1) / (h(0.3275911) * ax + h(1))
    e = np.exp2(h(-0.7213475204444817) * x * x, dtype=np.float32)
    p = t * h(1.061405429) + h(-1.453152027)
    for c in (1.421413741, -0.284496736, 0.254829592):
        p = t * p + h(c)
    ht = h(0.5) * p * t * e
    cdf = np.where(x >= 0, h(1) - ht, ht).astype(np.float32)
    v = (x * cdf * a).astype(np.float32)
    n = h(v.shape[-1])
    mean = v.sum(-1, dtype=np.float32, keepdims=True) / n
    if two_pass:
        var = ((v - mean) * (v - mean)).sum(-1, dtype=np.float32, keepdims=True) / n
    else:
        var = np.maximum((v * v).sum(-1, dtype=np.float32, keepdims=True) / n - mean * mean, h(0))
    rstd = h(1) / np.sqrt(var + h(1e-5))
    out = ((v - mean) * rstd * gm).astype(np.float32)
    return torch.from_numpy(out).to(bf16)


def worst_excess(M, n, family, two_pass, seed=0):
    gen = torch.Generator().manual_seed(seed)
    if family == "randn":
        a, gate = torch.randn(M, n, generator=gen), 2 * torch.randn(M, n, generator=gen)
    else:
        a, gate = lr.ill_conditioned(M, n, int(family[3:]), gen)
    a, gate = a.to(bf16), gate.to(bf16)
    gamma = (1 + 0.1 * torch.randn(n, generator=gen)).to(bf16).float()
    got = emulate_geglu_ln_fwd(a, gate, gamma, two_pass)
    ref = lr.geglu_ln_ref(a, gate, gamma)
    return lr.excess(got, ref["out"], ref["s_out"], True).max().item()


@pytest.mark.parametrize("n", [1000, 2730, 8000])
def test_one_pass_variance_is_rejected(n):
    """the two-pass emulation passes the GPU test's bound on every family; the one-pass emulation exceeds it by >= 10x
    on the ill-conditioned family (mean / sigma >= 4096: the variance is rounding noise, or clamped to 0)"""
    two = {f: worst_excess(64, n, f, True) for f in ("randn", "ill16", "ill256", "ill4096")}
    one = {f: worst_excess(64, n, f, False) for f in ("randn", "ill16", "ill256", "ill4096")}
    print(f"\nn={n} two-pass {two}\nn={n} one-pass {one}")
    assert max(two.values()) <= BOUND["gn"], two
    assert one["ill4096"] >= 10 * BOUND["gn"], one


def test_ill_conditioned_family_is_what_it_claims():
    gen = torch.Generator().manual_seed(1)
    for ratio in lr.ILL_RATIOS:
        for n in (1024, 2730, 8000):
            a, gate = lr.ill_conditioned(16, n, ratio, gen)
            assert torch.equal(a.to(bf16).float(), a) and torch.equal(gate.to(bf16).float(), gate)
            v = torch.nn.functional.gelu(gate.double()) * a.double()
            assert torch.equal(gate.float() * 1.0, torch.full_like(gate, 8.0))
            m, s = v.mean(-1).abs(), v.std(-1, unbiased=False)
            live = s > 0   # a row of the p = 0.5 families can come out constant
            assert (m[live] / s[live] >= 0.85 * ratio).all(), (ratio, n, (m / s).min().item())
            assert (s[live] ** 2 > 100 * lr.EPS).all()


# ---- case lists against the launch selection ---------------------------------------------------------------------------
def test_geglu_cases_cover_every_launch():
    fwd_tmpl, fwd_nch, bwd, mods, grid_edges = set(), set(), set(), set(), set()
    flags = set()
    for p in GEGLU_CASES:
        c = p.values[0]
        M, n, ip = c["M"], c["inner"], c["ip"]
        tmpl, grid = lr.geglu_fwd_launch(M, ip)
        fwd_tmpl.add(tmpl)
        fwd_nch.add(-(-(ip // 8) // lr.FF_THREADS))
        threads, btmpl, bgrid = lr.geglu_bwd_launch(M, ip)
        bwd.add((threads, btmpl))
        mods.add(n % 8)
        cap_f = lr.H100_SMS * 8
        cap_b = lr.H100_SMS * (2 if threads == 512 else 4)
        for cap, kind in ((cap_f, "fwd"), (cap_b, f"bwd{threads}-{btmpl}")):
            if abs(M - cap) <= 1:
                grid_edges.add((kind, M - cap))
        flags |= {k for k in ("ldh_extra", "ldg_extra") if c[k]}
        flags.add(c["family"])
        flags.add("dropout" if c["p"] > 0 else "no-dropout")
        if ip > (n + 7) // 8 * 8:
            flags.add("padded")
        if M in (1, 2, 7):
            flags.add(f"M{M}")
        if M > 2 * cap_f and M % min(M, cap_f):
            flags.add("large-M")
        if ip == 8192:
            flags.add("widest")
    assert fwd_tmpl == {1, 2, 4} and fwd_nch == {1, 2, 3, 4}, (fwd_tmpl, fwd_nch)
    # (256, 2) is only selected when ALM_GEGLU_BWD_THREADS turns the 512-thread layout off
    assert bwd == {(256, 1), (512, 1), (256, 4)}, bwd
    assert mods >= {0, 1, 7}, mods
    for kind in ("fwd", "bwd256-1", "bwd512-1", "bwd256-4"):
        need = {-1, 0, 1} if kind != "bwd256-4" else {1}
        assert {dm for k, dm in grid_edges if k == kind} >= need, (kind, grid_edges)
    assert flags >= {"ldh_extra", "ldg_extra", "saturated", "constant", "ill16", "ill256", "ill4096", "dropout",
                     "no-dropout", "padded", "M1", "M2", "M7", "large-M", "widest"}, flags
    assert lr.geglu_fwd_launch(2, 8200) is None and lr.geglu_bwd_launch(2, 8200) is None


def test_resid_cases_cover_options():
    seen = {k: set() for k in ("y", "want_r_new", "raw", "dr_out", "dextra", "dr_bf16")}
    dims, rows, scales, dc = set(), set(), set(), set()
    for p in RESID_CASES:
        c = p.values[0]
        for k in seen:
            seen[k].add(c[k])
        dims.add(c["d"])
        rows.add(c["M"])
        scales.add(c["out_scale"])
        dc.add(c["dc"] > 0)
    assert all(v == {True, False} for v in seen.values()), seen
    assert dims >= {1, 31, 32, 33, 1000, 1024, 2048} and rows >= {1, 7, 8, 9} and max(rows) > 1000
    assert len(scales) > 1 and any(s != 1.0 for s in scales) and dc == {True, False}
