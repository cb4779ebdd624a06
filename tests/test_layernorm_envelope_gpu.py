"""GEGLU + LayerNorm (alm_geglu_ln_fwd / _bwd) and the plain residual + LayerNorm (alm_resid_ln_fwd / _bwd) against the
fp64 references of tests/layernorm_ref.py across the kernels' envelope: every forward template (NCH = 1 / 2 / 4, and an
NCH = 3 width on the NCH = 4 template) and every backward layout (256 threads at NCH = 1 / 4, 512 threads) on both sides
of their width limits, inner % 8 in {0, 1, 7}, padded widths, row counts around the grid caps (the forward's
software-pipelined next row and L2 prefetch, the backward's per-CTA g_gamma partials), a strided h and dgn, saturated
gates, constant rows, rows with mean / sigma up to several thousand, dropout, and the refused width.

Every input is bf16- or fp32-exact, so the references see exactly the kernels' operands.  The criterion is per element
(layernorm_ref.excess): the output's own rounding plus BOUND x an error scale that a two-pass fp32 LayerNorm meets at any
mean / sigma.  Everything outside the logical outputs (a NaN sentinel) must stay unchanged, and two identical forward
calls give bitwise-identical results.  The references, the criterion's sensitivity to a one-pass variance and the case
lists' coverage are checked without a GPU in test_layernorm_envelope_host.py."""
import sys
from pathlib import Path

import pytest
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
import dropout_ref  # noqa: E402
import layernorm_ref as lr  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
bf16, f32, f64 = torch.bfloat16, torch.float32, torch.float64
INT = {bf16: torch.int16, f32: torch.int32}
SENT = {bf16: 0x7FA5, f32: 0x7FC0BEEF}   # NaN bit patterns that fill everything outside the outputs

# Bounds, about 3x the worst excess (error beyond the output's rounding over its scale, see layernorm_ref) measured over
# every case of this file on an H100 80GB HBM3 (700 W power limit), printed by `pytest -s` as [err] lines.  Worst
# measured: gn 1.08, da 0.84, dgate 0.51, g_gamma 1.75; resid_ln xn 1.54, dr 3.54, g_gamma 1.52.  With the variance
# taken in one pass (E[v^2] - mean^2), the ill-conditioned GEGLU rows exceeded these by 2e2 (mean / sigma 256) to 2.5e6
# (mean / sigma >= 4096) in gn and by up to 1.4e7 in da / dgate.
BOUND = dict(gn=3.5, da=2.5, dgate=1.6, gg=5.5, xn=4.5, dr=11.0, rgg=4.5)


def report(what, tag, err):
    worst = err.max().item() if err.numel() else 0.0
    print(f"[err] {what} {tag} {worst:.3e}")
    return worst


def sentinel(shape, dtype):
    return torch.full(shape, SENT[dtype], dtype=INT[dtype], device=DEV).view(dtype)


def bits(t):
    return t.view(INT[t.dtype])


# ---- GEGLU + LayerNorm -------------------------------------------------------------------------------------------------
def gcase(M, inner, *, ip=None, family="randn", ldh_extra=0, ldg_extra=0, p=0.0, id):
    ip = ip or (inner + 7) // 8 * 8
    return pytest.param(dict(M=M, inner=inner, ip=ip, family=family, ldh_extra=ldh_extra, ldg_extra=ldg_extra, p=p),
                        id=id)


GEGLU_CASES = [
    # forward NCH = 1 (inner_pad <= 2048); the backward's 256-thread NCH = 1 layout
    gcase(1, 1, id="nch1-inner1"),
    gcase(2, 7, id="nch1-inner7"),
    gcase(7, 1000, ip=1024, id="nch1-inner1000-padded-to-1024"),
    gcase(7, 2047, ldg_extra=16, id="nch1-inner2047-mod7"),
    gcase(2, 2048, id="nch1-inner2048-mod0"),
    gcase(527, 2048, id="nch1-bwd-grid-cap-minus1"),
    gcase(528, 2048, id="nch1-bwd-grid-cap"),
    gcase(529, 2041, ldg_extra=8, id="nch1-bwd-grid-cap-plus1-mod1"),
    # NCH = 2 (2048 < inner_pad <= 4096); the backward's 512-thread layout
    gcase(1, 2049, id="nch2-inner2049-mod1"),
    gcase(2, 2041, ip=2064, id="nch2-by-padding-only"),
    gcase(263, 2730, id="nch2-production-bwd512-grid-cap-minus1"),
    gcase(264, 2730, ldh_extra=64, id="nch2-bwd512-grid-cap-strided-h"),
    gcase(265, 2730, ldg_extra=24, id="nch2-bwd512-grid-cap-plus1"),
    gcase(1055, 4095, id="nch2-inner4095-fwd-grid-cap-minus1"),
    gcase(1056, 4096, id="nch2-inner4096-fwd-grid-cap"),
    gcase(1057, 2736, ldh_extra=8, id="nch2-fwd-grid-cap-plus1-strided-h"),
    gcase(5000, 2730, ldh_extra=40, ldg_extra=8, id="nch2-large-M-strided"),
    # NCH = 3 on the NCH = 4 template, and NCH = 4; the backward's 256-thread NCH = 4 layout
    gcase(7, 4097, id="nch3-inner4097-mod1"),
    gcase(529, 6143, id="nch3-inner6143-bwd-grid-cap-plus1"),
    gcase(1057, 6144, ldh_extra=16, id="nch3-fwd-grid-cap-plus1"),
    gcase(2, 8185, id="nch4-inner8185"),
    gcase(33, 8192, ldg_extra=8, id="nch4-inner8192-accepted"),
    # value families
    gcase(64, 2730, family="saturated", id="gates-to-10"),
    gcase(64, 8192, family="saturated", id="nch4-gates-to-10"),
    gcase(16, 2736, family="constant", id="constant-rows"),
    gcase(7, 1000, family="constant", id="nch1-constant-rows"),
    *[gcase(200, 2730, family=f"ill{r}", id=f"ill-conditioned-{r}") for r in lr.ILL_RATIOS],
    gcase(7, 2048, family="ill4096", id="nch1-ill-conditioned-4096"),
    gcase(300, 8000, family="ill4096", ldh_extra=16, id="nch4-ill-conditioned-4096"),
    gcase(65, 6144, family="ill256", id="nch3-ill-conditioned-256"),
    # dropout
    gcase(300, 2730, p=0.2, id="dropout-nch2"),
    gcase(33, 2047, p=0.5, ldg_extra=8, id="dropout-nch1"),
    gcase(529, 8185, p=0.1, family="ill4096", id="dropout-nch4-ill-conditioned"),
]


def geglu_inputs(c, seed):
    """h view [M, 2 ip] (a | gate, NaN in the padding columns and in the row-stride gap), gamma [n], the operands"""
    M, n, ip = c["M"], c["inner"], c["ip"]
    gen = torch.Generator().manual_seed(seed)
    fam = c["family"]
    if fam == "randn":
        a, gate = torch.randn(M, n, generator=gen), torch.randn(M, n, generator=gen) * 2
    elif fam == "saturated":
        a, gate = torch.randn(M, n, generator=gen), (torch.rand(M, n, generator=gen) * 20 - 10)
    elif fam == "constant":
        a, gate = torch.randn(M, 1, generator=gen).expand(M, n), torch.full((M, n), 8.0)
    else:
        a, gate = lr.ill_conditioned(M, n, int(fam[3:]), gen)
    a, gate = a.to(bf16), gate.to(bf16)
    gamma = (1 + 0.1 * torch.randn(n, generator=gen)).to(bf16).float()
    ldh = 2 * ip + c["ldh_extra"]
    buf = sentinel((M, ldh), bf16)
    buf[:, :n] = a.to(DEV)
    buf[:, ip:ip + n] = gate.to(DEV)
    return buf[:, :2 * ip], gamma.to(DEV), a.to(DEV), gate.to(DEV)


def dropout_factors(c, seed, site):
    if c["p"] == 0.0:
        return None
    keep = dropout_ref.keep(seed, site, range(c["M"]), range(c["inner"]), c["p"])
    return torch.from_numpy(keep).to(DEV, f64) / (1 - c["p"])


def run_geglu_fwd(c, h, gamma, drop):
    """alm_geglu_ln_fwd into sentinel-filled gn [M + 2, ldg] and stats [M + 1, 2]; checks everything outside
    gn[:M, :ip] and stats[:M] is unchanged and returns (gn [M, ip], stats [M, 2])"""
    M, ip = c["M"], c["ip"]
    ldg = ip + c["ldg_extra"]
    gn, stats = sentinel((M + 2, ldg), bf16), sentinel((M + 1, 2), f32)
    gn0, stats0 = gn.clone(), stats.clone()
    from audiolm_pytorch_b200 import _lib, ops

    _lib.call("alm_geglu_ln_fwd", h, h.stride(0), ip, gamma, gn, ldg, stats, M, c["inner"], ip,
              *ops._drop_args(drop))
    torch.cuda.synchronize()
    outside = torch.ones_like(gn, dtype=torch.bool)
    outside[:M, :ip] = False
    assert torch.equal(bits(gn)[outside], bits(gn0)[outside]), "alm_geglu_ln_fwd wrote outside gn[:M, :inner_pad]"
    assert torch.equal(bits(stats[M:]), bits(stats0[M:])), "alm_geglu_ln_fwd wrote past stats[M]"
    return gn[:M, :ip], stats[:M]


def run_geglu_bwd(c, h, gamma, stats, dgn, g_gamma, drop):
    """alm_geglu_ln_bwd into a sentinel-filled dh with h's row stride and one extra row; checks the stride gap and the
    extra row are unchanged and returns dh [M, 2 ip]"""
    M, ip = c["M"], c["ip"]
    ldh = h.stride(0)
    dh = sentinel((M + 1, ldh), bf16)
    dh0 = dh.clone()
    from audiolm_pytorch_b200 import _lib, ops

    _lib.call("alm_geglu_ln_bwd", h, ldh, ip, gamma, stats, dgn, dgn.stride(0), dh, g_gamma, M, c["inner"], ip,
              *ops._drop_args(drop))
    torch.cuda.synchronize()
    outside = torch.ones_like(dh, dtype=torch.bool)
    outside[:M, :2 * ip] = False
    assert torch.equal(bits(dh)[outside], bits(dh0)[outside]), "alm_geglu_ln_bwd wrote outside dh[:M, :2 inner_pad]"
    return dh[:M, :2 * ip]


@pytest.mark.parametrize("c", GEGLU_CASES)
def test_geglu_ln_fp64(c, request):
    tag = request.node.callspec.id
    M, n, ip = c["M"], c["inner"], c["ip"]
    seed = zlib_seed(tag)
    h, gamma, a, gate = geglu_inputs(c, seed)
    drop = (c["p"], 0x5EED + seed, 2) if c["p"] > 0 else None
    Z = dropout_factors(c, *drop[1:]) if drop else None
    gen = torch.Generator().manual_seed(seed + 1)
    dgn_buf = sentinel((M, ip + 16), bf16)   # a strided dgn: NaN in the padding columns and the stride gap
    dgn_buf[:, :n] = torch.randn(M, n, generator=gen).to(bf16).to(DEV)
    dgn = dgn_buf[:, :ip]
    g0 = torch.randn(n, generator=gen).to(DEV)

    gn, stats = run_geglu_fwd(c, h, gamma, drop)
    gn2, stats2 = run_geglu_fwd(c, h, gamma, drop)
    assert torch.equal(bits(gn), bits(gn2)) and torch.equal(bits(stats), bits(stats2)), "forward not deterministic"
    assert (bits(gn[:, n:]) == 0).all(), "gn columns >= inner must be +0"
    g_gamma = torch.cat((g0, torch.full((8,), float("nan"), device=DEV)))
    dh = run_geglu_bwd(c, h, gamma, stats, dgn, g_gamma, drop)
    torch.cuda.synchronize()
    assert torch.isnan(g_gamma[n:]).all(), "alm_geglu_ln_bwd wrote past g_gamma[inner]"
    assert (bits(dh[:, n:ip]) == 0).all() and (bits(dh[:, ip + n:]) == 0).all(), "dh padding columns must be +0"

    ref = lr.geglu_ln_ref(a, gate, gamma, Z, dgn[:, :n], g0)
    if Z is not None:
        assert (gn[:, :n][Z == 0] == 0).all()
    worst = dict(
        gn=report("gn", tag, lr.excess(gn[:, :n], ref["out"], ref["s_out"], True)),
        da=report("da", tag, lr.excess(dh[:, :n], ref["da"], ref["s_da"], True)),
        dgate=report("dgate", tag, lr.excess(dh[:, ip:ip + n], ref["dgate"], ref["s_dgate"], True)),
        gg=report("gg", tag, lr.excess(g_gamma[:n], ref["g_gamma"], ref["s_gg"], False)),
    )
    for k, v in worst.items():
        assert v <= BOUND[k], (k, v)   # NaN fails too


def zlib_seed(tag):
    import zlib

    return zlib.crc32(tag.encode()) & 0x7FFFFFFF


def test_geglu_ln_width_limit():
    """inner_pad 8192 is the widest width (the nch4 cases above run it); 8200 is refused in both directions"""
    from audiolm_pytorch_b200 import _lib, ops

    M, n = 2, 8200
    h = torch.zeros(M, 2 * n, dtype=bf16, device=DEV)
    gamma = torch.ones(n, device=DEV)
    stats = torch.zeros(M, 2, device=DEV)
    with pytest.raises(_lib.AlmError, match=r"\(-4\)"):
        ops.geglu_ln_fwd(h, gamma, inner=n, inner_pad=n)
    with pytest.raises(_lib.AlmError, match=r"\(-4\)"):
        ops.geglu_ln_bwd(h, gamma, stats, torch.zeros(M, n, dtype=bf16, device=DEV), torch.zeros_like(gamma),
                         inner=n, inner_pad=n)


# ---- plain residual + LayerNorm ----------------------------------------------------------------------------------------
RESID_D = (1, 31, 32, 33, 1000, 1024, 2048)
RESID_M = (1, 7, 8, 9, 3001)


def resid_case(i, d, M):
    """the optional operands cycle with the case index so that every combination of y / r_new / raw and
    dr_out / dextra / dr_bf16 meets several widths and row counts; every fourth case has a DC offset"""
    return pytest.param(dict(d=d, M=M, y=i % 2 == 0, want_r_new=i % 3 != 0, raw=i % 4 < 2, dr_out=i % 3 != 1,
                             dextra=i % 5 < 3, dr_bf16=i % 2 == 1, out_scale=(1.0, 0.5, -2.0)[i % 3],
                             dc=(0.0, 0.0, 0.0, 2048.0)[i % 4]), id=f"d{d}-M{M}-{i}")


RESID_CASES = [resid_case(i, d, M) for i, (d, M) in enumerate((d, M) for d in RESID_D for M in RESID_M)]
RESID_CASES += [pytest.param(dict(d=d, M=M, y=True, want_r_new=True, raw=True, dr_out=True, dextra=True, dr_bf16=True,
                                  out_scale=0.5, dc=dc), id=f"ill-conditioned-d{d}-dc{int(dc)}")
                for d, M in ((1024, 300), (33, 9), (2048, 64)) for dc in (16.0, 4096.0)]


@pytest.mark.parametrize("c", RESID_CASES)
def test_resid_ln_fp64(c, request):
    from audiolm_pytorch_b200 import _lib

    tag = request.node.callspec.id
    M, d = c["M"], c["d"]
    gen = torch.Generator().manual_seed(zlib_seed(tag))
    r = (c["dc"] + torch.randn(M, d, generator=gen)).to(DEV)          # fp32 inputs: exact as they are
    y = torch.randn(M, d, generator=gen).to(bf16).to(DEV) if c["y"] else None
    gamma = (1 + 0.1 * torch.randn(d, generator=gen)).to(DEV)
    dxn = torch.randn(M, d, generator=gen).to(bf16).to(DEV)
    dr_out = torch.randn(M, d, generator=gen).to(DEV) if c["dr_out"] else None
    dextra = torch.randn(M, d, generator=gen).to(bf16).to(DEV) if c["dextra"] else None
    g0 = torch.randn(d, generator=gen).to(DEV)

    def fwd():
        want_r_new = c["want_r_new"] and y is not None
        r_new = sentinel((M + 1, d), f32) if want_r_new else None
        xn, stats = sentinel((M + 1, d), bf16), sentinel((M + 1, 2), f32)
        rb = sentinel((M + 1, d), bf16) if c["raw"] else None
        _lib.call("alm_resid_ln_fwd", r, y, gamma, r_new, xn, rb, stats, M, d)
        torch.cuda.synchronize()
        for t in (r_new, xn, rb, stats):
            if t is not None:
                assert torch.equal(bits(t[M:]), bits(sentinel((1, t.shape[1]), t.dtype))), "wrote past row M"
        return [None if t is None else t[:M] for t in (r_new, xn, rb, stats)]

    r_new, xn, rb, stats = fwd()
    again = fwd()
    for t, u in zip((r_new, xn, rb, stats), again):
        assert t is None or torch.equal(bits(t), bits(u)), "forward not deterministic"
    v32 = r + (y.float() if y is not None else 0)
    if r_new is not None:
        assert torch.equal(r_new, v32)
    if rb is not None:
        assert torch.equal(bits(rb), bits(v32.to(bf16)))

    rn = r_new if r_new is not None else v32   # the backward reads the forward's r + y
    dr = sentinel((M + 1, d), f32)
    drb = sentinel((M + 1, d), bf16) if c["dr_bf16"] else None
    g_gamma = torch.cat((g0, torch.full((8,), float("nan"), device=DEV)))
    _lib.call("alm_resid_ln_bwd", rn, gamma, stats, dr_out, dxn, dextra, dr, drb, g_gamma, float(c["out_scale"]), M, d)
    torch.cuda.synchronize()
    assert torch.isnan(g_gamma[d:]).all(), "alm_resid_ln_bwd wrote past g_gamma[d]"
    for t in (dr, drb):
        if t is not None:
            assert torch.equal(bits(t[M:]), bits(sentinel((1, d), t.dtype))), "wrote past row M"
    if drb is not None:
        assert torch.equal(bits(drb[:M]), bits(dr[:M].to(bf16)))

    ref = lr.resid_ln_ref(r, y, gamma, dxn, dr_out, dextra, c["out_scale"], g0)
    worst = dict(
        xn=report("xn", tag, lr.excess(xn, ref["out"], ref["s_out"], True)),
        dr=report("dr", tag, lr.excess(dr[:M], ref["dr"], ref["s_dr"], False)),
        rgg=report("rgg", tag, lr.excess(g_gamma[:d], ref["g_gamma"], ref["s_gg"], False)),
    )
    for k, v in worst.items():
        assert v <= BOUND[k], (k, v)
