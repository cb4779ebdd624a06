"""wgmma MQA attention vs an fp32 restatement of attend.py:98-146 (math path)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def attend_ref(q, k, v, mask, causal):
    # q [b,h,i,d], k/v [b,j,d] fp32; mask [b,j] bool  (attend.py:117-144)
    scale = q.shape[-1] ** -0.5
    sim = torch.einsum("bhid,bjd->bhij", q, k) * scale
    neg = -torch.finfo(sim.dtype).max
    if mask is not None:
        sim = sim.masked_fill(~mask[:, None, None, :], neg)
    if causal:
        i, j = sim.shape[-2:]
        cm = torch.ones(i, j, dtype=torch.bool, device=q.device).triu(j - i + 1)
        sim = sim.masked_fill(cm, neg)
    attn = sim.softmax(-1)
    return torch.einsum("bhij,bjd->bhid", attn, v), sim


CASES = [
    # b, h, n_q, n_k, masked, causal
    (1, 1, 128, 128, False, True),
    (2, 8, 256, 256, False, True),
    (2, 8, 300, 300, True, True),     # ragged + key mask
    (1, 8, 2048, 2048, True, True),   # config C3 length
    (2, 4, 128, 384, False, True),    # right-aligned queries (cache-style)
    (2, 2, 200, 200, True, False),    # non-causal
]


@pytest.mark.parametrize("b,h,n_q,n_k,masked,causal", CASES)
def test_attn_fwd(b, h, n_q, n_k, masked, causal):
    from audiolm_pytorch_b200 import ops

    torch.manual_seed(n_q + 13 * n_k + h)
    dev = "cuda"
    qkv = torch.randn(b, n_q, h * 64 + 128, device=dev).to(torch.bfloat16)
    q = qkv[..., : h * 64]
    if n_k == n_q:
        k, v = qkv[..., h * 64 : h * 64 + 64], qkv[..., h * 64 + 64 :]
    else:
        k = torch.randn(b, n_k, 64, device=dev).to(torch.bfloat16)
        v = torch.randn(b, n_k, 64, device=dev).to(torch.bfloat16)
    mask = None
    if masked:
        mask = torch.rand(b, n_k, device=dev) > 0.15
        mask[:, 0] = True
    o, lse = ops.mqa_attn_fwd(q, k, v, heads=h, key_mask=mask, causal=causal)
    torch.cuda.synchronize()
    qf = q.float().reshape(b, n_q, h, 64).permute(0, 2, 1, 3)
    ref, sim = attend_ref(qf, k.float(), v.float(), mask, causal)
    ref = ref.permute(0, 2, 1, 3).reshape(b, n_q, h * 64)
    err = (o.float() - ref).abs().max().item()
    assert err <= 2e-2 * max(1.0, ref.abs().max().item()), f"attention out err {err}"
    lse_ref = torch.logsumexp(sim, dim=-1)
    assert (lse[..., :n_q] * 0.6931471805599453 - lse_ref).abs().max().item() <= 2e-2  # kernel stores log2-domain LSE
