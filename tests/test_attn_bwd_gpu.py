"""Fused attention backward (ops.mqa_attn_bwd) vs an fp32 torch restatement with autograd, over the shapes the kernel
treats differently: the C3 length with a key mask, a ragged n_q, right-aligned n_k > n_q, non-causal, 1 / 8 / 16 heads
and a query block whose keys are all masked.  dk and dv must also be bitwise reproducible."""
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda"
bf16 = torch.bfloat16


def rel_err(a, b):
    a, b = a.float(), b.float()
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-6)


def attend_ref(q, k, v, mask, causal):
    """q [b, h, n_q, 64], k / v [b, n_k, 64]; queries right-aligned against keys.  A query that sees no key gets a
    zero output (and zero gradients), as the kernels define it."""
    scale = q.shape[-1] ** -0.5
    sim = torch.einsum("bhid,bjd->bhij", q, k) * scale
    n_q, n_k = sim.shape[-2:]
    vis = torch.ones(sim.shape[0], 1, n_q, n_k, dtype=torch.bool, device=q.device)
    if mask is not None:
        vis = vis & mask[:, None, None, :]
    if causal:
        vis = vis & ~torch.ones(n_q, n_k, dtype=torch.bool, device=q.device).triu(n_k - n_q + 1)
    any_vis = vis.any(-1, keepdim=True)
    sim = sim.masked_fill(~vis, float("-inf")).masked_fill(~any_vis, 0.0)
    p = sim.softmax(-1) * any_vis
    return torch.einsum("bhij,bjd->bhid", p, v)


@pytest.mark.parametrize("b,h,n_q,n_k,mask_kind,causal", [
    (2, 8, 2048, 2048, "random", True),     # C3 length, key mask
    (2, 8, 300, 300, "random", True),       # ragged n_q
    (2, 8, 200, 456, "random", True),       # right-aligned n_k > n_q
    (2, 8, 384, 384, None, False),          # non-causal
    (1, 1, 512, 512, "random", True),
    (1, 16, 256, 256, None, True),
    (2, 8, 384, 384, "first_block", True),  # keys [0, 128) masked: query block 0 sees no key
])
def test_attn_bwd_vs_fp32(b, h, n_q, n_k, mask_kind, causal):
    from audiolm_pytorch_b200 import ops

    torch.manual_seed(n_q + 7 * h + n_k)
    q = torch.randn(b, n_q, h * 64, device=DEV).to(bf16)
    k = torch.randn(b, n_k, 64, device=DEV).to(bf16)
    v = torch.randn(b, n_k, 64, device=DEV).to(bf16)
    d_o = torch.randn(b, n_q, h * 64, device=DEV).to(bf16)
    mask = None
    if mask_kind == "random":
        mask = torch.rand(b, n_k, device=DEV) > 0.15
        mask[:, 0] = True
    elif mask_kind == "first_block":
        mask = torch.ones(b, n_k, dtype=torch.bool, device=DEV)
        mask[:, :128] = False
    o, lse = ops.mqa_attn_fwd(q, k, v, heads=h, key_mask=mask, causal=causal)
    dq, dk, dv = ops.mqa_attn_bwd(q, k, v, o, d_o, lse, heads=h, key_mask=mask, causal=causal)
    _, dk2, dv2 = ops.mqa_attn_bwd(q, k, v, o, d_o, lse, heads=h, key_mask=mask, causal=causal)
    torch.cuda.synchronize()
    assert torch.equal(dk, dk2) and torch.equal(dv, dv2), "dk / dv are not bitwise reproducible"
    ql, kl, vl = (t.float().clone().requires_grad_(True) for t in (q, k, v))
    qh = ql.reshape(b, n_q, h, 64).permute(0, 2, 1, 3)
    ref = attend_ref(qh, kl, vl, mask, causal).permute(0, 2, 1, 3).reshape(b, n_q, h * 64)
    (ref * d_o.float()).sum().backward()
    assert torch.isfinite(dq.float()).all() and torch.isfinite(dk.float()).all() and torch.isfinite(dv.float()).all()
    assert rel_err(dq, ql.grad) < 2e-2
    assert rel_err(dk, kl.grad) < 2e-2
    assert rel_err(dv, vl.grad) < 2e-2
    if mask_kind == "first_block":
        assert (dk[:, :128] == 0).all() and (dv[:, :128] == 0).all()
        assert (dq[:, :128] == 0).all()
