"""Test references for the transformer's LayerNorm kernels (csrc/ffn_loss_misc.cu): GEGLU + LayerNorm
(alm_geglu_ln_fwd / _bwd) and the plain residual + LayerNorm (alm_resid_ln_fwd / _bwd).

* fp64 references: F.layer_norm in fp64 (eps 1e-5), the erf-form GELU, fp64 autograd for the gradients.
* The per-element criterion: an element may differ from the reference by its output's own rounding (2^-8 |ref| for
  bf16) plus BOUND x its error scale x 2^-24.  The error scale of the normalised value x^_c = (v_c - mean) rstd is
      e_c = rstd (|v_c| + mean_j |v_j|),
  what an fp32 computation of v, of the mean and of a two-pass variance can reach at any mean / sigma.  A one-pass
  variance E[v^2] - mean^2 loses (mean / sigma)^2 2^-24 of the variance and cannot meet it on rows with a DC offset.
  For GEGLU, |v_c| is replaced by |a_c gate_c|: the kernels' GELU (Abramowitz-Stegun erf, alm_common.cuh) has an
  absolute error of about 2^-24 in the normal CDF, i.e. about |a_c gate_c| 2^-24 in v_c.
  The backward's scale follows the terms of rstd (gl_c - m1 - x^_c m2) (gl = dgn gamma, m1 = mean gl,
  m2 = mean gl x^) with x^ carrying e; the gradients of GEGLU's inputs multiply it by |gelu(gate)| or
  |a gelu'(gate)|, and g_gamma's scale is sum_rows |dgn| (|x^| + e).
* The ill-conditioned input family: bf16-exact rows with mean / sigma from 16 to several thousand.
* A host copy of alm_geglu_ln_fwd / _bwd's launch selection.
"""
import math

import torch
import torch.nn.functional as F

f64 = torch.float64
EPS = 1e-5
U = 2.0 ** -24     # fp32 unit roundoff
TINY = 1e-30
H100_SMS = 132


# ---- launch selection of alm_geglu_ln_fwd / alm_geglu_ln_bwd (csrc/ffn_loss_misc.cu) ------------------------------------
FF_THREADS, FF_MAX_CHUNKS = 256, 4


def geglu_fwd_launch(M, inner_pad, sms=H100_SMS):
    """(template NCH, grid), or None where the entry point refuses the width (ALM_ERR_UNSUPPORTED)"""
    nch = -(-(inner_pad // 8) // FF_THREADS)
    if nch > FF_MAX_CHUNKS:
        return None
    return (1 if nch <= 1 else 2 if nch == 2 else 4), min(M, sms * 8)


def geglu_bwd_launch(M, inner_pad, sms=H100_SMS):
    """(threads, template NCH, grid) with the default 512-thread layout enabled, or None where refused"""
    nch = -(-(inner_pad // 8) // FF_THREADS)
    if nch > FF_MAX_CHUNKS:
        return None
    threads = 512 if 2048 < inner_pad <= 4096 else 256
    tmpl = 1 if threads == 512 or nch <= 1 else 2 if nch == 2 else 4
    return threads, tmpl, min(M, sms * (2 if threads == 512 else 4))


# ---- references ----------------------------------------------------------------------------------------------------------
def gelu_grad(x):
    return 0.5 * (1 + torch.erf(x / math.sqrt(2))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2 * math.pi)


def _ln_stats(v):
    mean = v.mean(-1, keepdim=True)
    rstd = (v.var(-1, unbiased=False, keepdim=True) + EPS).rsqrt()
    return mean, rstd


def _bwd_scale(gl, xhat, rstd, e):
    """error scale (units of 2^-24) of dv = rstd (gl - m1 - x^ m2) when x^ carries e"""
    m2 = (gl * xhat).mean(-1, keepdim=True)
    return rstd * (gl.abs() + gl.abs().mean(-1, keepdim=True) + xhat.abs() * (gl * xhat).abs().mean(-1, keepdim=True)
                   + m2.abs() * e + xhat.abs() * (gl.abs() * e).mean(-1, keepdim=True))


def geglu_ln_ref(a, gate, gamma, Z=None, dgn=None, g0=None):
    """fp64 LayerNorm(gelu(gate) a) gamma (x Z, the dropout factors) over the last dim, and with dgn [M, n] the
    gradients.  Returns a dict of fp64 tensors: out, mean, rstd, and the error scales s_out (already x 2^-24);
    with dgn also da, dgate, g_gamma (+ g0) and s_da, s_dgate, s_gg."""
    a, gate, gamma = (t.to(f64).detach().clone().requires_grad_(dgn is not None) for t in (a, gate, gamma))
    Z = torch.ones_like(a) if Z is None else Z.to(f64)
    v = F.gelu(gate) * a
    out = F.layer_norm(v, v.shape[-1:], eps=EPS) * gamma * Z
    with torch.no_grad():
        mean, rstd = _ln_stats(v)
        xhat = (v - mean) * rstd
        e = rstd * ((a * gate).abs() + v.abs().mean(-1, keepdim=True))
        r = dict(out=out.detach(), mean=mean[:, 0], rstd=rstd[:, 0], s_out=(gamma.abs() * Z.abs() * e * U + TINY))
    if dgn is None:
        return r
    out.backward(dgn.to(f64))
    with torch.no_grad():
        dz = dgn.to(f64) * Z
        gl = dz * gamma
        dv = rstd * (gl - gl.mean(-1, keepdim=True) - xhat * (gl * xhat).mean(-1, keepdim=True))
        sdv = _bwd_scale(gl, xhat, rstd, e)
        ge, gp = F.gelu(gate), gelu_grad(gate)
        r.update(da=a.grad, dgate=gate.grad, g_gamma=gamma.grad + (0 if g0 is None else g0.to(f64)),
                 s_da=(sdv * ge.abs() + dv.abs() * gate.abs()) * U + TINY,
                 s_dgate=(sdv * (a * gp).abs() + (dv * a).abs() * (1 + gate.abs())) * U + TINY,
                 s_gg=((dz.abs() * (xhat.abs() + e)).sum(0) + (0 if g0 is None else g0.to(f64).abs())) * U + TINY)
    return r


def resid_ln_ref(r, y, gamma, dxn=None, dr_out=None, dextra=None, out_scale=1.0, g0=None):
    """fp64 v = r (+ y), LayerNorm(v) gamma, and with dxn the residual gradient
    out_scale (dr_out + LN_bwd(dxn) + dextra) and g_gamma (+ g0), with their error scales (x 2^-24)"""
    v = r.to(f64) + (0 if y is None else y.to(f64))
    v, gamma = v.detach().clone().requires_grad_(dxn is not None), gamma.to(f64).detach().clone().requires_grad_(dxn is not None)
    out = F.layer_norm(v, v.shape[-1:], eps=EPS) * gamma
    with torch.no_grad():
        mean, rstd = _ln_stats(v)
        xhat = (v - mean) * rstd
        e = rstd * (v.abs() + v.abs().mean(-1, keepdim=True))
        res = dict(v=v.detach(), out=out.detach(), mean=mean[:, 0], rstd=rstd[:, 0], s_out=gamma.abs() * e * U + TINY)
    if dxn is None:
        return res
    out.backward(dxn.to(f64))
    with torch.no_grad():
        dx = dxn.to(f64)
        gl = dx * gamma
        dv = v.grad
        extra = (0 if dr_out is None else dr_out.to(f64)) + (0 if dextra is None else dextra.to(f64))
        s_extra = (0 if dr_out is None else dr_out.to(f64).abs()) + (0 if dextra is None else dextra.to(f64).abs())
        sdv = _bwd_scale(gl, xhat, rstd, e)
        res.update(dr=out_scale * (dv + extra), g_gamma=gamma.grad + (0 if g0 is None else g0.to(f64)),
                   s_dr=abs(out_scale) * (sdv + dv.abs() + s_extra) * U + TINY,
                   s_gg=((dx.abs() * (xhat.abs() + e)).sum(0) + (0 if g0 is None else g0.to(f64).abs())) * U + TINY)
    return res


def excess(got, ref, scale, bf16_out):
    """per-element error beyond the output's own rounding (2^-8 |ref| for bf16) over the error scale; NaN stays NaN"""
    d = (got.to(f64) - ref).abs()
    if bf16_out:
        d = torch.where(torch.isnan(d), d, (d - 2.0 ** -8 * ref.abs()).clamp(min=0.0))
    return d / scale


# ---- inputs ----------------------------------------------------------------------------------------------------------
ILL_RATIOS = (16, 256, 4096)


def ill_conditioned(M, n, ratio, gen):
    """bf16-exact GEGLU operands (a, gate) [M, n] whose rows v = gelu(gate) a have mean / sigma of about `ratio` or more:
    gate = 8 (gelu(8) = 8 in fp32), a = A except on a random subset of channels at A (1 + s) (an exact bf16 step), with
    A = +-32 or +-64 so that the variance stays far above eps.  16: s = 1/8 on half the channels; 256: s = 1/128 on
    half; 4096: s = 1/128 on one channel in 1024 (at least one), mean / sigma = 128 / sqrt(p (1 - p)) >= 4096."""
    s, p = {16: (1 / 8, 0.5), 256: (1 / 128, 0.5), 4096: (1 / 128, None)}[ratio]
    A = torch.tensor([32.0, -32.0, 64.0, -64.0])[torch.randint(0, 4, (M, 1), generator=gen)]
    if p is None:
        k = max(1, n // 1024)
        odd = torch.zeros(M, n, dtype=torch.bool)
        idx = torch.argsort(torch.rand(M, n, generator=gen), dim=1)[:, :k]
        odd.scatter_(1, idx, True)
    else:
        odd = torch.rand(M, n, generator=gen) < p
    a = torch.where(odd, A * (1 + s), A)
    gate = torch.full((M, n), 8.0)
    return a, gate
