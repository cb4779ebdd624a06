"""Hyper-connection backward on the shared-memory ring (d <= 1024) and the forward without `bin`: C3-sized token counts
that wrap the ring many times, odd d, no dbin_extra, expand mode, and the in-kernel parameter gradients against an
fp64 restatement."""
import sys
from pathlib import Path

import pytest
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
from test_ops_gpu import DEV, bf16, hc_ref, make_hc, rel_err  # noqa: E402

pytestmark = pytest.mark.gpu

C3_TAIL = 8 * 2048 + 37  # every CTA walks the ring many times; the token count is not a multiple of the grid


def _inputs(M, d, expand, seed):
    torch.manual_seed(seed)
    S = 4
    if expand:
        x = torch.randn(M, d, device=DEV)
        return dict(x_expand=x), dict(x=x)
    R_in = torch.randn(M, S, d, device=DEV).to(bf16)
    Y = torch.randn(M, d, device=DEV).to(bf16)
    bp = 1 + 0.2 * torch.randn(M, S, device=DEV)
    return dict(R_in=R_in, Y=Y, beta_prev=bp), dict(R_in=R_in, Y=Y, bp=bp)


def _reference(hc, ln_gamma, raw, expand, d, M, dtype, w):
    """autograd of hc_ref in `dtype`: (leaf gradients of the data inputs, of hc, of ln_gamma)"""
    S = 4
    hc_leaf = {k: v.to(dtype).clone().requires_grad_(True) for k, v in hc.items()}
    lng_leaf = ln_gamma.to(dtype).clone().requires_grad_(True)
    if expand:
        x_leaf = raw["x"].to(dtype).clone().requires_grad_(True)
        R = x_leaf[:, None, :].expand(M, S, d)
        data = (x_leaf,)
    else:
        data = tuple(raw[k].to(dtype).clone().requires_grad_(True) for k in ("R_in", "Y", "bp"))
        R = data[0] + data[2][..., None] * data[1][:, None, :]
    r_out, r_bin, r_xn, r_beta = hc_ref(hc_leaf, lng_leaf, R, d)
    w1, w2, w3, w4 = w
    loss = (r_out * w1.to(dtype)).sum() + (r_xn * w2.to(dtype)).sum() + (r_beta * w4.to(dtype)).sum()
    if w3 is not None:
        loss = loss + (r_bin * w3.to(dtype)).sum()
    loss.backward()
    return [t.grad for t in data], {k: v.grad for k, v in hc_leaf.items()}, lng_leaf.grad


@pytest.mark.parametrize("M,d,expand,with_dbin", [(C3_TAIL, 1024, False, True), (C3_TAIL, 1024, False, False),
                                                  (3001, 1000, False, True), (517, 64, False, False),
                                                  (C3_TAIL, 1024, True, True), (777, 1000, True, False)])
def test_hc_pre_bwd_ring(M, d, expand, with_dbin):
    from audiolm_pytorch_b200 import ops

    S = 4
    hc, ln_gamma = make_hc(d, seed=d + 1)
    kin, raw = _inputs(M, d, expand, M + d)
    R_out, bin_, xn, beta, aux = ops.hc_pre_fwd(hc, ln_gamma, **kin, M=M, d=d)
    w1 = torch.randn(M, S, d, device=DEV).to(bf16)
    w2 = torch.randn(M, d, device=DEV).to(bf16)
    w3 = torch.randn(M, d, device=DEV).to(bf16) if with_dbin else None
    w4 = torch.randn(M, S, device=DEV)
    ref_data, ref_hc, ref_ln = _reference(hc, ln_gamma, raw, expand, d, M, torch.float32, (w1, w2, w3, w4))
    grads = {k: torch.zeros_like(v) for k, v in hc.items()}
    g_ln = torch.zeros_like(ln_gamma)
    if expand:
        dx = ops.hc_pre_bwd(hc, ln_gamma, grads, g_ln, aux, w1, w2, w4, dbin_extra=w3, x_expand=kin["x_expand"],
                            dx_scale=0.1, M=M, d=d)
        assert rel_err(dx, 0.1 * ref_data[0]) < 2e-2
    else:
        dR_in, dY, dbp = ops.hc_pre_bwd(hc, ln_gamma, grads, g_ln, aux, w1, w2, w4, dbin_extra=w3, **kin, M=M, d=d)
        assert rel_err(dR_in, ref_data[0]) < 2e-2
        assert rel_err(dY, ref_data[1]) < 2e-2
        assert rel_err(dbp, ref_data[2]) < 2e-2
    torch.cuda.synchronize()
    for k in hc:
        assert rel_err(grads[k], ref_hc[k]) < 3e-2, k
    assert rel_err(g_ln, ref_ln) < 3e-2


@pytest.mark.parametrize("M,d,expand", [(C3_TAIL, 1024, False), (3001, 1000, True)])
def test_hc_param_grads_vs_fp64(M, d, expand):
    """The per-channel parameter gradients are summed in fp32 inside the kernel; their error against an fp64
    restatement of the whole op is printed (pytest -s) and bounded."""
    from audiolm_pytorch_b200 import ops

    S = 4
    hc, ln_gamma = make_hc(d, seed=7)
    kin, raw = _inputs(M, d, expand, 11)
    _, _, _, _, aux = ops.hc_pre_fwd(hc, ln_gamma, **kin, M=M, d=d)
    w = (torch.randn(M, S, d, device=DEV).to(bf16), torch.randn(M, d, device=DEV).to(bf16),
         torch.randn(M, d, device=DEV).to(bf16), torch.randn(M, S, device=DEV))
    _, ref_hc, ref_ln = _reference(hc, ln_gamma, raw, expand, d, M, torch.float64, w)
    grads = {k: torch.zeros_like(v) for k, v in hc.items()}
    g_ln = torch.zeros_like(ln_gamma)
    ops.hc_pre_bwd(hc, ln_gamma, grads, g_ln, aux, w[0], w[1], w[3], dbin_extra=w[2], **kin,
                   **({"dx_scale": 1.0} if expand else {}), M=M, d=d)
    torch.cuda.synchronize()
    errs = {k: rel_err(grads[k], ref_hc[k]) for k in hc}
    errs["ln_gamma"] = rel_err(g_ln, ref_ln)
    print("\nparameter-gradient error vs fp64 (max abs / max |ref|):",
          " ".join(f"{k}={v:.2e}" for k, v in errs.items()))
    for k, v in errs.items():
        assert v < 1e-2, k


@pytest.mark.parametrize("M,d,expand", [(C3_TAIL, 1024, False), (300, 1000, False), (200, 1024, True)])
def test_hc_pre_fwd_without_bin(M, d, expand):
    from audiolm_pytorch_b200 import ops

    hc, ln_gamma = make_hc(d, seed=3)
    kin, _ = _inputs(M, d, expand, 5)
    full = ops.hc_pre_fwd(hc, ln_gamma, **kin, M=M, d=d)
    lean = ops.hc_pre_fwd(hc, ln_gamma, **kin, M=M, d=d, want_bin=False)
    assert full[1] is not None and lean[1] is None
    for i in (0, 2, 3, 4):
        assert torch.equal(full[i], lean[i]), i
