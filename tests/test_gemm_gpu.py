"""wgmma GEMM (alm_gemm_bf16) vs an fp32 torch reference of the same contraction."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _ref(a, b, a_mn, b_mn, alpha, bias):
    A = a.float().transpose(-1, -2) if a_mn else a.float()
    B = b.float().transpose(-1, -2) if b_mn else b.float()
    out = alpha * (A @ B.transpose(-1, -2))
    if bias is not None:
        out = out + bias
    return out


def _mk(shape, mn, dev, pad=0):
    """operand with logical (E, K); stored [E,K] or [K,E]; optional row padding to test ld != width"""
    E, K = shape[-2], shape[-1]
    st = (*shape[:-2], K, E) if mn else tuple(shape)
    if pad:
        pad = pad + (-(st[-1] + pad)) % 8  # keep the leading dimension a multiple of 8 elements (16 B)
    full = torch.randn(*st[:-1], st[-1] + pad, device=dev, dtype=torch.float32).to(torch.bfloat16)
    return full[..., : st[-1]]


CASES = [
    # M, N, K, a_mn, b_mn, batch
    (128, 256, 64, False, False, 1),
    (128, 256, 256, False, False, 1),
    (256, 512, 1024, False, False, 1),
    (300, 640, 1000, False, False, 1),     # ragged M / N / K tails
    (2048, 5460, 1024, False, False, 1),   # FFN W1 shape (N tail)
    (2048, 1024, 2736, False, False, 1),   # FFN W2 shape (padded K)
    (512, 128, 1024, False, False, 1),     # BLOCK_N = 128 path
    (512, 64, 512, False, False, 1),       # BLOCK_N = 64 path
    (128, 256, 64, False, True, 1),        # dgrad form: B MN-major
    (384, 1024, 5460, False, True, 1),
    (300, 1000, 520, False, True, 1),
    (128, 256, 64, True, True, 1),         # wgrad form: both MN-major
    (1024, 512, 4096, True, True, 1),
    (5460, 1024, 2048, True, True, 1),
    (200, 328, 1000, True, True, 1),
    (384, 1025, 1024, False, False, 3),    # batched (grouped logit heads), odd N
]


@pytest.mark.parametrize("M,N,K,a_mn,b_mn,batch", CASES)
def test_gemm_matches_fp32(M, N, K, a_mn, b_mn, batch):
    from audiolm_pytorch_b200 import ops

    torch.manual_seed(M * 7 + N * 3 + K)
    dev = "cuda"
    lead = (batch,) if batch > 1 else ()
    a = _mk((*lead, M, K), a_mn, dev, pad=8)
    b = _mk((*lead, N, K), b_mn, dev, pad=8)
    for out_dtype in (torch.bfloat16, torch.float32):
        bias = torch.randn(N, device=dev) if out_dtype == torch.float32 else None
        out = ops.gemm(a, b, a_mn=a_mn, b_mn=b_mn, out_dtype=out_dtype, alpha=0.5, bias=bias)
        torch.cuda.synchronize()
        ref = _ref(a, b, a_mn, b_mn, 0.5, bias)
        err = (out.float() - ref).abs().max().item()
        scale = ref.abs().max().item()
        tol = (2e-2 if out_dtype == torch.bfloat16 else 2e-3) * scale
        assert err <= tol, f"max err {err} vs scale {scale} ({out_dtype})"


def test_gemm_accumulate_and_splitk():
    from audiolm_pytorch_b200 import ops

    torch.manual_seed(0)
    M, N, K = 640, 1024, 8192
    a = _mk((M, K), True, "cuda")
    b = _mk((N, K), True, "cuda")
    base = torch.randn(M, N, device="cuda")
    ref = base + _ref(a, b, True, True, 1.0, None)
    out = base.clone()
    ops.gemm(a, b, a_mn=True, b_mn=True, out=out, acc_mode=1)
    assert (out - ref).abs().max().item() <= 2e-3 * ref.abs().max().item()
    out = base.clone()
    ops.gemm(a, b, a_mn=True, b_mn=True, out=out, acc_mode=2, split_k=4)
    assert (out - ref).abs().max().item() <= 2e-3 * ref.abs().max().item()
