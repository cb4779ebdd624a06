"""The dense GEMM (ops.gemm -> alm_gemm_bf16), the decode GEMV (ops.gemv -> alm_gemv_bf16), the fused logit head + cross
entropy (ops.head_ce_fwd / ops.head_ce_bwd -> alm_gemm_head_ce modes 1 and 2 + alm_ce_finish), the materialised cross
entropy (ops.ce_fwd_bwd) and their autograd wiring (heads.cross_entropy) against an fp64 reference across the kernels'
envelope: the three operand layouts at BLOCK_N 64, 128 and 256, M / N / K on both sides of every tile edge and of the
TMA boxes' K tails, persistent CTAs that run several tiles, every epilogue (TMA store, bf16 and fp32 register stores,
vector and scalar, accumulating, split-K atomics and the host's rewrite of split_k), batched operands with padded
strides, operand views with NaN in their padding, and C windows inside a sentinel-filled buffer.

Every operand is bf16-representable, so the reference sees exactly the kernels' inputs.  Operand rows carry scales
spread over 2^-8 .. 2^8, so output rows and columns differ in magnitude by up to 2^16 and a whole-tensor criterion
could not see an error confined to the small ones.  The criterion is per element instead:
    |got - ref| <= BOUND x (|alpha| sum_k |a_ik| |b_jk| + |bias_j| + |C0_ij|)  (+ 2^-8 |ref| for a bf16 output),
the dot product's own error scale, which neither hides one bad element nor blows up where a sum cancels.  The cross
entropy kernels are checked per row: the absolute error of the LSE and of the row loss in nats, and every dlogits
element against 2^-8 |ref| + BOUND x scale.  An exact-integer family (operands in {-2..2}, K <= 1024, integer bias and
C0) must match bitwise: every partial sum is an integer below 2^13, exact in fp32 in any summation order.

Everything outside the logical C (and outside [0, V) of dlogits) must be bitwise unchanged, and two identical calls
without split-K give bitwise-identical results.  The GPU tests are marked individually; the references' own checks,
the criterion's sensitivity to injected faults, the case lists' coverage and the host copy of the GEMM's BLOCK_N rule
run without a GPU."""
import math
import zlib

import pytest
import torch
import torch.nn.functional as F

DEV = "cuda"
bf16 = torch.bfloat16
f32 = torch.float32
f64 = torch.float64
BLOCK_M, BLOCK_K = 128, 64   # alm_gemm_bf16's tile (csrc/gemm_wgmma.cu)
H100_SMS = 132
TINY = 1e-30
INT = {bf16: torch.int16, f32: torch.int32}
SENT = {bf16: 0x7FA5, f32: 0x7FC0BEEF}   # NaN bit patterns that fill everything outside C / dlogits' [0, V)
LAYOUTS = {"kk": (False, False), "kmn": (False, True), "mnmn": (True, True)}   # forward, dgrad, wgrad

# Bounds, one per quantity, about 3x the worst error measured over every case of this file on an H100 80GB HBM3
# (700 W power limit).  Worst measured: gemm 1.3e-6 (K = 16400), gemv 6.7e-8; fused head + CE: lse 3.6e-4 and loss
# 2.7e-4 nats (V = 16385, K = 1024), dlogits 2.5e-6; materialised CE (exact fp32 logits): loss 7.7e-6 nats, dlogits
# 2.3e-7; autograd: mean loss 6.2e-7 nats, dx 4.8e-3, dw 3.7e-3, db 1.7e-3.  The exact-integer family matched bitwise.
# The fused LSE and loss carry the GEMM's error on logits of up to ~200 in dot-product scale (120-nat ramps plus
# sum_k |x_k| |w_k| ~ 80): about 1e-6 of that, where the materialised path starts from exact logits.  dx / dw / db
# carry the bf16 rounding of dlogits (at most 2^-8 of their scale) and, for dx, its own bf16 rounding.  Every injected
# fault of the host tests below exceeds its bound by more than 10x (a dropped k block or K tail by about 10^4x).
BOUND = dict(
    gemm=4e-6,           # per element, over the dot product's error scale (beyond 2^-8 |ref| for bf16 outputs)
    gemv=2e-7,
    lse=1.1e-3,          # nats, absolute, per row (fused)
    loss=8e-4,           # nats, absolute, per row (fused)
    dlogits=7.5e-6,      # per element, over the gradient scale, beyond 2^-8 |ref| (fused)
    loss_mat=2.5e-5,     # the same for ops.ce_fwd_bwd on exact fp32 logits
    dlogits_mat=7e-7,
    ce_mean=2e-6,        # nats: heads.cross_entropy's mean loss
    dx=1.45e-2, dw=1.1e-2, db=5.3e-3,   # per element, over |dlogits| contracted with |operand|
)


def report(what, tag, err):
    worst = err.max().item() if err.numel() else 0.0
    print(f"[err] {what} {tag} {worst:.3e}")
    return worst


# ---- references and the criterion -------------------------------------------------------------------------------------
def gemm_block_n():
    from audiolm_pytorch_b200.transformer import gemm_block_n as bn

    return bn


def split_after_rewrite(K, split):
    """the split-K factor gemm_common (csrc/gemm_wgmma.cu) runs: at most one split per k block, none empty"""
    kb = -(-K // BLOCK_K)
    s = min(split, kb)
    while s > 1 and (s - 1) * -(-kb // s) >= kb:
        s -= 1
    return s


def gemm_ref(a, b, *, alpha=1.0, bias=None, c0=None):
    """fp64 alpha A B^T (+ bias[n]) (+ C0) and the per-element error scale |alpha| |A| |B|^T + |bias| + |C0|.
    a [batch, M, K], b [batch, N, K] (fp64)"""
    ref = alpha * (a @ b.transpose(-1, -2))
    scale = abs(alpha) * (a.abs() @ b.abs().transpose(-1, -2))
    if bias is not None:
        ref = ref + bias.to(f64)
        scale = scale + bias.to(f64).abs()
    if c0 is not None:
        ref = ref + c0.to(f64)
        scale = scale + c0.to(f64).abs()
    return ref, scale + TINY


def excess(got, ref, scale, bf16_out):
    """per-element error beyond the output's own rounding (2^-8 |ref| for bf16) over the error scale; NaN stays NaN"""
    d = (got.to(f64) - ref).abs()
    if bf16_out:
        d = torch.where(torch.isnan(d), d, (d - 2.0 ** -8 * ref.abs()).clamp(min=0.0))
    return d / scale


def ce_ref(logits, labels, ignore, scale=1.0):
    """fp64 cross entropy per row: (lse, loss = lse - logit[label] or 0 where ignored,
    dlogits = (softmax - onehot) x scale, zero rows where ignored).  Labels are in [0, V) or ignore."""
    logits = logits.to(f64)
    R, V = logits.shape
    ign = labels == ignore
    safe = torch.where(ign, 0, labels)
    lse = torch.logsumexp(logits, -1)
    lab = logits.gather(1, safe[:, None])[:, 0]
    loss = torch.where(ign, 0.0, lse - lab)
    d = torch.softmax(logits, -1)
    d[torch.arange(R, device=logits.device), safe] -= 1.0
    d = torch.where(ign[:, None], 0.0, d * scale)
    return lse, loss, d


# ---- GEMM cases -----------------------------------------------------------------------------------------------------
def epilogue(dtype, acc_mode, base, ldc, strideC, batch):
    """the epilogue alm_gemm_bf16 runs for a C at byte address `base`: mirrors the p.tma_store condition of gemm_common
    (csrc/gemm_wgmma.cu) and the 8-B alignment test of its fp32 vector stores"""
    if dtype == bf16:
        tma = acc_mode == 0 and base % 16 == 0 and (2 * ldc) % 16 == 0 and (batch == 1 or (2 * strideC) % 16 == 0)
        return "tma" if tma else "bf16-reg"
    vec = base % 8 == 0 and ldc % 2 == 0 and (batch == 1 or strideC % 2 == 0)
    return "f32-vec" if vec else "f32-scalar"


def out_geometry(c):
    """(ldc, batch pitch) of the case's C window"""
    ldc = c["N"] + c["ldc_extra"]
    return ldc, (c["M"] + c["rows_extra"]) * ldc + c["gap"]


def gemm_case(M, N, K, lay="kk", *, out="bf16", acc=0, split=1, bias=False, alpha=1.0, batch=1, c_off=0, ldc_extra=0,
              rows_extra=2, gap=0, pad=0, exact=False):
    """one GEMM case.  out: C's dtype; c_off: C's base offset in elements; ldc_extra: columns past N in every row of
    the C buffer; rows_extra: rows past M; gap: elements between batches; pad: extra NaN columns (a multiple of 8) and
    NaN rows of the operand buffers; exact: the integer family"""
    c = dict(M=M, N=N, K=K, lay=lay, out=out, acc=acc, split=split, bias=bias, alpha=alpha, batch=batch, c_off=c_off,
             ldc_extra=ldc_extra, rows_extra=rows_extra, gap=gap, pad=pad, exact=exact)
    dtype = bf16 if out == "bf16" else f32
    ldc, pitch = out_geometry(c)
    c["path"] = epilogue(dtype, acc, c_off * dtype.itemsize, ldc, pitch, batch)
    return c


def g(*args, id, **kw):
    return pytest.param(gemm_case(*args, **kw), id=id)


GEMM_CASES = [
    # forward (K-major A and B): BLOCK_N 64 / 128 / 256, M / N / K residues
    g(1, 1, 8, id="kk-bn64-m1-n1-k8"),
    g(63, 8, 16, out="f32", id="kk-bn64-m63-n8-k16-f32"),
    g(64, 63, 56, bias=True, id="kk-bn64-m64-n63-k56-bias"),
    g(65, 64, 72, out="f32", alpha=-0.75, id="kk-bn64-m65-n64-k72-f32"),
    g(127, 65, 64, out="f32", bias=True, id="kk-bn128-m127-n65-k64-f32"),
    g(128, 127, 1000, id="kk-bn128-m128-n127-k1000"),
    g(129, 128, 5460, out="f32", bias=True, id="kk-bn128-m129-n128-k5460-f32"),
    g(200, 384, 520, alpha=0.5, id="kk-bn128-n384"),
    g(128, 257, 1000, out="f32", id="kk-bn128-n257-f32"),
    g(129, 129, 1000, bias=True, id="kk-bn256-m129-n129"),
    g(127, 255, 72, out="f32", id="kk-bn256-m127-n255-k72-f32"),
    g(65, 256, 16, id="kk-bn256-m65-n256-k16"),
    g(300, 1000, 1000, out="f32", bias=True, alpha=0.5, id="kk-bn256-n1000-f32"),
    g(64, 1025, 56, id="kk-bn256-m64-n1025-k56"),
    # dgrad (K-major A, MN-major B)
    g(1, 64, 64, "kmn", id="kmn-bn64-m1-n64"),
    g(63, 1, 1000, "kmn", out="f32", id="kmn-bn64-m63-n1-f32"),
    g(129, 8, 8, "kmn", bias=True, id="kmn-bn64-m129-n8-k8"),
    g(65, 128, 56, "kmn", id="kmn-bn128-m65-n128-k56"),
    g(128, 65, 72, "kmn", out="f32", id="kmn-bn128-m128-n65-k72-f32"),
    g(127, 384, 5460, "kmn", alpha=0.5, id="kmn-bn128-m127-n384-k5460"),
    g(64, 256, 1000, "kmn", out="f32", bias=True, id="kmn-bn256-m64-n256-f32"),
    g(129, 129, 16, "kmn", out="f32", id="kmn-bn256-m129-n129-k16-f32"),
    g(300, 1025, 64, "kmn", id="kmn-bn256-n1025-k64"),
    g(63, 255, 1000, "kmn", id="kmn-bn256-m63-n255"),
    g(1, 257, 1000, "kmn", out="f32", id="kmn-bn128-m1-n257-f32"),
    # wgrad (both MN-major)
    g(1, 1, 1000, "mnmn", out="f32", id="mnmn-bn64-m1-n1-f32"),
    g(64, 63, 8, "mnmn", id="mnmn-bn64-m64-n63-k8"),
    g(65, 64, 5460, "mnmn", out="f32", id="mnmn-bn64-m65-n64-k5460-f32"),
    g(127, 127, 64, "mnmn", bias=True, id="mnmn-bn128-m127-n127-k64"),
    g(128, 128, 56, "mnmn", out="f32", id="mnmn-bn128-m128-n128-k56-f32"),
    g(129, 384, 72, "mnmn", id="mnmn-bn128-m129-n384-k72"),
    g(63, 256, 16, "mnmn", id="mnmn-bn256-m63-n256-k16"),
    g(128, 1000, 1000, "mnmn", out="f32", bias=True, id="mnmn-bn256-n1000-f32"),
    g(129, 255, 5460, "mnmn", id="mnmn-bn256-m129-n255-k5460"),
    g(1, 129, 1000, "mnmn", id="mnmn-bn256-m1-n129"),
    # deep K
    g(128, 256, 16384, out="f32", id="kk-deep-k16384-f32"),
    g(256, 64, 16400, "mnmn", out="f32", id="mnmn-deep-k16400-f32"),
    g(128, 128, 16384, "kmn", id="kmn-deep-k16384"),
    # persistent CTAs: more tiles than SMs at each BLOCK_N (the epilogue staging buffers are reused)
    g(38400, 64, 256, id="persistent-bn64-m38400-tma-nbuf1"),
    g(20000, 128, 256, out="f32", bias=True, id="persistent-bn128-m20000-f32"),
    g(2048, 5460, 1024, bias=True, id="persistent-bn256-ffn-w1"),
    # epilogues: TMA store with and without bias, alpha != 1, NBUF 1 (BLOCK_N 64) and 2
    g(200, 64, 1000, bias=True, alpha=-1.5, id="tma-bn64-nbuf1-bias-alpha"),
    g(129, 128, 200, bias=True, id="tma-bn128-nbuf2-bias"),
    g(200, 200, 300, id="tma-bn256-nbuf2"),
    g(130, 200, 100, ldc_extra=8, rows_extra=5, bias=True, id="tma-ldc-past-n-rows-past-m"),
    # bf16 register path: base one element off, odd ldc
    g(130, 300, 200, c_off=1, bias=True, id="bf16-reg-base-off1"),
    g(129, 130, 100, ldc_extra=1, id="bf16-reg-odd-ldc"),
    g(65, 64, 72, c_off=1, ldc_extra=3, id="bf16-reg-bn64-off1-odd-ldc"),
    # fp32: vector stores (default) and scalar ones
    g(130, 300, 200, out="f32", c_off=1, bias=True, id="f32-scalar-base-off1"),
    g(129, 130, 100, out="f32", ldc_extra=1, id="f32-scalar-odd-ldc"),
    g(200, 384, 100, out="f32", ldc_extra=4, rows_extra=3, id="f32-vec-ldc-past-n"),
    # accumulation into C: read-modify-write, atomics, split-K and its host-side rewrite
    g(200, 300, 500, out="f32", acc=1, bias=True, id="acc1-f32"),
    g(200, 300, 500, acc=1, bias=True, id="acc1-bf16"),
    g(129, 130, 72, acc=1, c_off=1, ldc_extra=1, id="acc1-bf16-off1-odd-ldc"),
    g(131, 257, 300, "mnmn", out="f32", acc=1, ldc_extra=1, id="acc1-f32-odd-ldc"),
    g(128, 200, 600, "mnmn", out="f32", acc=2, id="acc2-split1"),
    g(128, 256, 2048, "mnmn", out="f32", acc=2, split=2, id="acc2-split2"),
    g(300, 1000, 4096, "mnmn", out="f32", acc=2, split=4, ldc_extra=2, id="acc2-split4"),
    g(64, 64, 8192, "mnmn", out="f32", acc=2, split=64, id="acc2-split64"),
    g(200, 130, 1000, out="f32", acc=2, split=4, bias=True, alpha=0.5, id="acc2-split4-bias"),
    g(128, 128, 320, "mnmn", out="f32", acc=2, split=4, id="acc2-split4-over-5-kblocks-runs-3"),
    g(100, 200, 100, "kmn", out="f32", acc=2, split=64, c_off=1, id="acc2-split64-over-2-kblocks-scalar"),
    # batched with padded operand strides and a gap between the batches of C
    g(300, 200, 300, batch=2, pad=8, gap=8, bias=True, id="batch2-tma-gap"),
    g(100, 130, 72, "kmn", batch=3, pad=8, c_off=1, gap=5, id="batch3-bf16-reg-gap"),
    g(64, 64, 100, "mnmn", batch=2, pad=16, out="f32", gap=3, id="batch2-f32-scalar-gap"),
    g(65, 257, 1000, batch=3, pad=8, out="f32", gap=2, acc=1, id="batch3-f32-acc1-gap"),
    # operand views: NaN in the row padding past K and in the rows past M / N
    g(130, 200, 1000, pad=8, id="nan-pad-kk"),
    g(100, 300, 72, "kmn", pad=16, out="f32", id="nan-pad-kmn"),
    g(129, 129, 1000, "mnmn", pad=8, id="nan-pad-mnmn"),
    # the cases of the former whole-tensor test, with the per-element criterion (bf16 out, and fp32 out with bias)
    *[g(M, N, K, lay, batch=bt, pad=8, alpha=0.5, out=o, bias=o == "f32", id=f"legacy-{lay}-{M}x{N}x{K}-b{bt}-{o}")
      for (M, N, K, lay, bt) in [(128, 256, 64, "kk", 1), (128, 256, 256, "kk", 1), (256, 512, 1024, "kk", 1),
                                 (300, 640, 1000, "kk", 1), (2048, 5460, 1024, "kk", 1), (2048, 1024, 2736, "kk", 1),
                                 (512, 128, 1024, "kk", 1), (512, 64, 512, "kk", 1), (128, 256, 64, "kmn", 1),
                                 (384, 1024, 5460, "kmn", 1), (300, 1000, 520, "kmn", 1), (128, 256, 64, "mnmn", 1),
                                 (1024, 512, 4096, "mnmn", 1), (5460, 1024, 2048, "mnmn", 1),
                                 (200, 328, 1000, "mnmn", 1), (384, 1025, 1024, "kk", 3)]
      for o in ("bf16", "f32")],
    # exact integers: bitwise
    g(129, 64, 1000, bias=True, exact=True, id="exact-kk-bn64-tma"),
    g(200, 300, 1024, out="f32", alpha=0.5, bias=True, exact=True, id="exact-kk-bn128-f32"),
    g(65, 1000, 520, alpha=0.5, c_off=1, exact=True, id="exact-kk-bn256-bf16-reg"),
    g(127, 63, 1024, "kmn", out="f32", exact=True, id="exact-kmn-bn64-f32"),
    g(128, 129, 72, "kmn", bias=True, exact=True, id="exact-kmn-bn256-tma"),
    g(300, 384, 1000, "kmn", out="f32", acc=1, exact=True, id="exact-kmn-bn128-acc1"),
    g(64, 128, 1024, "mnmn", out="f32", acc=2, split=4, exact=True, id="exact-mnmn-bn128-split4"),
    g(1, 255, 1000, "mnmn", acc=1, alpha=0.5, exact=True, id="exact-mnmn-bn256-acc1-bf16"),
    g(129, 8, 1024, "mnmn", out="f32", acc=2, split=64, exact=True, id="exact-mnmn-bn64-split64"),
    g(200, 1025, 1024, "mnmn", out="f32", acc=2, split=2, bias=True, pad=8, exact=True, id="exact-mnmn-split2-bias"),
    g(300, 200, 1000, batch=3, pad=8, gap=8, exact=True, id="exact-batch3-tma"),
    g(128, 65, 320, out="f32", acc=2, split=4, exact=True, id="exact-split4-over-5-kblocks"),
]


def operand(rows, K, mn, batch, gen, *, exact=False, pad=0):
    """one GEMM operand of logical shape [batch, rows, K] -> (its fp64 values on the GPU, the kernel's bf16 view).
    Stored K-major ([rows, K]) or MN-major ([K, rows]) in a NaN-filled buffer whose row pitch is the width rounded up
    to 8 elements plus `pad`, with `pad` more NaN rows at the end of every batch."""
    if exact:
        v = torch.randint(-2, 3, (batch, rows, K), generator=gen).float()
    else:
        e = torch.randint(-8, 9, (batch, rows, 1), generator=gen).float()
        v = torch.randn(batch, rows, K, generator=gen) * torch.exp2(e)
    v = v.to(bf16)
    st = v.transpose(1, 2) if mn else v
    r, w = st.shape[1], st.shape[2]
    buf = torch.full((batch, r + pad, -(-w // 8) * 8 + pad), math.nan, dtype=bf16)
    buf[:, :r, :w] = st
    view = buf.to(DEV)[:, :r, :w]
    return v.to(DEV, f64), (view if batch > 1 else view[0])


def out_buffer(c, dtype):
    """(flat sentinel-filled buffer, the C window [batch, M, N] in it, bool mask of the window over the buffer)"""
    ldc, pitch = out_geometry(c)
    n = c["c_off"] + c["batch"] * pitch
    flat = torch.empty(n, dtype=dtype, device=DEV)
    flat.view(INT[dtype]).fill_(SENT[dtype])
    geo = ((c["batch"], c["M"], c["N"]), (pitch, ldc, 1), c["c_off"])
    inside = torch.zeros(n, dtype=torch.bool, device=DEV)
    inside.as_strided(*geo).fill_(True)
    return flat, flat.as_strided(*geo), inside


@pytest.mark.gpu
@pytest.mark.parametrize("c", GEMM_CASES)
def test_gemm_matches_fp64(c, request):
    run_gemm_case(c, request.node.callspec.id)


@pytest.mark.gpu
def test_gemm_accumulate_and_splitk():
    """the wgrad shape of a long sequence (M = 640, N = 1024, K = 8192, both operands MN-major) accumulated into an
    fp32 C that holds prior values: read-modify-write (acc_mode 1), and fp32 atomics over 4 k splits (acc_mode 2)"""
    run_gemm_case(gemm_case(640, 1024, 8192, "mnmn", out="f32", acc=1), "accumulate-acc1")
    run_gemm_case(gemm_case(640, 1024, 8192, "mnmn", out="f32", acc=2, split=4), "accumulate-split4")


def run_gemm_case(c, tag):
    """one GEMM case against the fp64 reference: writes outside C, finiteness, reproducibility without split-K, then
    the per-element criterion (or bitwise equality for the integer family)"""
    from audiolm_pytorch_b200 import ops

    gen = torch.Generator().manual_seed(zlib.crc32(tag.encode()))
    a_mn, b_mn = LAYOUTS[c["lay"]]
    batch, M, N, exact = c["batch"], c["M"], c["N"], c["exact"]
    A, a = operand(M, c["K"], a_mn, batch, gen, exact=exact, pad=c["pad"])
    B, b = operand(N, c["K"], b_mn, batch, gen, exact=exact, pad=c["pad"])
    dtype = bf16 if c["out"] == "bf16" else f32
    bias = None
    if c["bias"]:
        bias = (torch.randint(-8, 9, (N,), generator=gen).float() if exact else torch.randn(N, generator=gen) * 4).to(DEV)
    flat, out, inside = out_buffer(c, dtype)
    c0 = None
    if c["acc"]:
        if exact:
            c0 = torch.randint(-8, 9, (batch, M, N), generator=gen).float()
        else:
            c0 = torch.randn(batch, M, N, generator=gen) * torch.exp2(torch.randint(-8, 9, (batch, M, 1), generator=gen))
        out.copy_(c0.to(DEV))
        c0 = out.to(f64)
    before = flat.clone()
    ldc, pitch = out_geometry(c)
    assert epilogue(dtype, c["acc"], out.data_ptr(), ldc, pitch, batch) == c["path"]
    kw = dict(a_mn=a_mn, b_mn=b_mn, alpha=c["alpha"], bias=bias, acc_mode=c["acc"], split_k=c["split"])
    ops.gemm(a, b, out=out if batch > 1 else out[0], **kw)
    torch.cuda.synchronize()
    it = INT[dtype]
    assert torch.equal(flat.view(it)[~inside], before.view(it)[~inside]), "a write outside C"
    assert torch.isfinite(out).all(), "NaN / inf in C: a read past an operand's logical extent"
    if c["split"] == 1:
        flat2 = before.clone()
        out2 = flat2.as_strided(out.shape, out.stride(), c["c_off"])
        ops.gemm(a, b, out=out2 if batch > 1 else out2[0], **kw)
        torch.cuda.synchronize()
        assert torch.equal(flat2.view(it), flat.view(it)), "two identical calls differ"
    ref, scale = gemm_ref(A, B, alpha=c["alpha"], bias=bias, c0=c0)
    if exact:
        want = ref.to(f32).to(dtype)
        bad = out != want
        print(f"[err] gemm-exact {tag} {int(bad.sum())} elements differ")
        assert not bad.any(), (f"{int(bad.sum())} of {bad.numel()} elements differ from the exact result, first at "
                               f"{bad.nonzero()[0].tolist()}")
    else:
        worst = report("gemm", tag, excess(out, ref, scale, dtype == bf16))
        assert worst <= BOUND["gemm"], (worst, BOUND["gemm"])


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["a-mn-without-b-mn", "lda-not-multiple-of-8", "operand-base-misaligned",
                                  "split-k-with-bf16-c"])
def test_gemm_refuses_without_launching(kind):
    from audiolm_pytorch_b200 import _lib, ops

    M = N = K = 128
    a = torch.ones(M, K, dtype=bf16, device=DEV)
    b = torch.ones(N, K, dtype=bf16, device=DEV)
    out = torch.zeros(M, N, dtype=bf16, device=DEV)
    kw = dict(out=out)
    if kind == "a-mn-without-b-mn":
        kw.update(a_mn=True)
    elif kind == "lda-not-multiple-of-8":
        a = torch.ones(M, K + 4, dtype=bf16, device=DEV)[:, :K]
    elif kind == "operand-base-misaligned":
        b = torch.ones(N, K + 8, dtype=bf16, device=DEV)[:, 1:K + 1]     # 2 B past a 16-B boundary, ldb = K + 8
    else:
        kw.update(acc_mode=2, split_k=2)
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    with pytest.raises(_lib.AlmError):
        ops.gemm(a, b, **kw)
    torch.cuda.synchronize()
    assert _lib.launch_count() == n0
    assert (out == 0).all()


# ---- GEMV -------------------------------------------------------------------------------------------------------------
def gv(rows, N, K, *, id, out="f32", bias=False, ldw_extra=0, ldx_extra=0):
    return pytest.param(dict(rows=rows, N=N, K=K, out=out, bias=bias, ldw_extra=ldw_extra, ldx_extra=ldx_extra), id=id)


GEMV_BIG_N = 2 * 4 * H100_SMS * 8 + 3   # more columns than 4 CTAs per SM x 8 warps: every warp loops over several


GEMV_CASES = [
    gv(1, 1, 8, id="r1-n1-k8"),
    gv(2, 7, 24, bias=True, id="r2-n7-k24-bias"),
    gv(3, 9, 1021, ldw_extra=16, id="r3-n9-k1021-nan-past-kp"),
    gv(4, GEMV_BIG_N, 1021, ldx_extra=5, id="r4-strided-n-loop-k1021"),
    gv(5, 300, 24, out="bf16", id="r5-k24-bf16"),
    gv(6, 1000, 8, bias=True, ldx_extra=3, id="r6-k8-bias-strided-x"),
    gv(7, 4100, 1021, out="bf16", bias=True, ldw_extra=8, id="r7-k1021-bf16-bias"),
    gv(8, 1024, 6144, id="r8-k6144-96kb"),
    gv(8, 9, 6144, bias=True, ldw_extra=8, ldx_extra=8, id="r8-n9-k6144-bias"),
    gv(8, GEMV_BIG_N, 1021, out="bf16", id="r8-strided-n-loop-bf16"),
    gv(1, GEMV_BIG_N, 6144, bias=True, id="r1-strided-n-loop-k6144"),
    gv(3, 7, 8, out="bf16", bias=True, id="r3-n7-k8-bf16-bias"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("c", GEMV_CASES)
def test_gemv_matches_fp64(c, request):
    from audiolm_pytorch_b200 import ops

    tag = request.node.callspec.id
    gen = torch.Generator().manual_seed(zlib.crc32(tag.encode()))
    rows, N, K = c["rows"], c["N"], c["K"]
    Kp = -(-K // 8) * 8
    X = (torch.randn(rows, K, generator=gen) * torch.exp2(torch.randint(-8, 9, (rows, 1), generator=gen))).to(bf16)
    W = (torch.randn(N, K, generator=gen) * torch.exp2(torch.randint(-8, 9, (N, 1), generator=gen))).to(bf16)
    xbuf = torch.full((rows, K + c["ldx_extra"]), math.nan, dtype=bf16)
    xbuf[:, :K] = X
    wbuf = torch.full((N, Kp + c["ldw_extra"]), math.nan, dtype=bf16)   # NaN in [Kp, ldw): never read
    wbuf[:, :Kp] = 0                                                      # zero padding up to Kp: the contract
    wbuf[:, :K] = W
    x = xbuf.to(DEV)[:, :K]
    w = wbuf.to(DEV)[:, :Kp]
    bias = (torch.randn(N, generator=gen) * 4).to(DEV) if c["bias"] else None
    dtype = bf16 if c["out"] == "bf16" else f32
    got = ops.gemv(x, w, out_dtype=dtype, bias=bias)
    again = ops.gemv(x, w, out_dtype=dtype, bias=bias)
    torch.cuda.synchronize()
    assert torch.equal(got, again), "two identical calls differ"
    assert torch.isfinite(got).all()
    ref, scale = gemm_ref(X.to(DEV, f64), W.to(DEV, f64), bias=bias)
    worst = report("gemv", tag, excess(got, ref, scale, dtype == bf16))
    assert worst <= BOUND["gemv"], (worst, BOUND["gemv"])


@pytest.mark.gpu
@pytest.mark.parametrize("rows,K", [(8, 6152), (5, 9832), (2, 24600)], ids=["r8-k6152", "r5-k9832", "r2-k24600"])
def test_gemv_refuses_past_96kb(rows, K):
    """x is staged in shared memory as [rows][Kp]: more than 96 KB is refused before any launch"""
    from audiolm_pytorch_b200 import _lib, ops

    assert rows * (-(-K // 8) * 8) * 2 > 96 * 1024
    x = torch.ones(rows, K, dtype=bf16, device=DEV)
    w = torch.zeros(16, -(-K // 8) * 8, dtype=bf16, device=DEV)
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    with pytest.raises(_lib.AlmError):
        ops.gemv(x, w)
    assert _lib.launch_count() == n0


# ---- fused head + cross entropy, and the materialised cross entropy ------------------------------------------------
def ce_case(M, V, *, id, K=256, bias=False, ignore=-1, all_ignored=False):
    return pytest.param(dict(M=M, V=V, K=K, bias=bias, ignore=ignore, all_ignored=all_ignored), id=id)


CE_CASES = [
    ce_case(1, 1, id="m1-v1"),
    ce_case(127, 63, bias=True, id="m127-v63-bias"),
    ce_case(129, 64, id="m129-v64"),
    ce_case(200, 65, bias=True, ignore=0, id="v65-ignore-class-0-bias"),
    ce_case(300, 128, id="v128"),
    ce_case(129, 129, bias=True, id="m129-v129-bias"),
    ce_case(127, 256, id="m127-v256"),
    ce_case(500, 257, bias=True, id="v257-one-column-in-last-tile-bias"),
    ce_case(600, 1025, id="v1025-one-column-in-last-tile"),
    ce_case(300, 1025, bias=True, ignore=0, id="v1025-ignore-class-0-bias"),
    ce_case(4096, 16385, K=1024, bias=True, id="v16385-many-tiles-bias"),
    ce_case(20000, 129, K=64, id="m20000-more-row-tiles-than-sms"),
    ce_case(256, 300, all_ignored=True, id="all-rows-ignored"),
]


def ce_operands(c, gen):
    """x [M, K], w [V, K] bf16 (fp64 copies on the GPU), bias, labels.  Rows cycle through five shapes: random logits
    (std ~2); flat (every logit 3 without bias: lse = 3 + ln V); peaked (one column 60 nats above the rest); max in the
    last, partial tile (30 nats up); a ramp over 120 nats across the columns, where most tiles' partials underflow.
    Labels hit 0, V - 1, the peak column and both sides of every tile edge; every 7th row is ignored."""
    M, V, K = c["M"], c["V"], c["K"]
    x = torch.randn(M, K, generator=gen) * 0.5
    w = torch.randn(V, K, generator=gen) * 0.25
    x[:, :4] = 0
    w[:, :4] = 0
    peak = V // 2
    w[:, 0] = 1.0
    w[peak, 1] = 1.0
    w[V - 1, 2] = 1.0
    w[:, 3] = torch.arange(V) / V
    kind = torch.arange(M) % 5
    x[kind == 1] = 0
    x[kind == 1, 0] = 3.0
    x[kind == 2, 1] = 60.0
    x[kind == 3, 2] = 30.0
    x[kind == 4, 3] = 120.0
    bn = gemm_block_n()(V)
    special = [0, V - 1, peak] + [t * bn + d for t in range(1, -(-V // bn)) for d in (-1, 0)]
    labels = torch.randint(0, V, (M,), generator=gen)
    perm = torch.randperm(M, generator=gen)[:len(special)]
    labels[perm] = torch.tensor(special[:len(perm)])
    labels[3::7] = c["ignore"]
    if c["all_ignored"]:
        labels[:] = c["ignore"]
    bias = (torch.randn(V, generator=gen) * 2).to(DEV) if c["bias"] else None
    x, w = x.to(bf16).to(DEV), w.to(bf16).to(DEV)
    return x, w, bias, labels.to(DEV)


def ce_check(tag, what, got_lse, got_loss, got_d, want, scale, ign):
    """per-row LSE / loss errors in nats and per-element dlogits errors -> worst of each"""
    lse, loss, d = want
    out = {}
    if got_lse is not None:
        out["lse"] = report(f"{what}-lse", tag, (got_lse.to(f64) - lse).abs())
    out["loss"] = report(f"{what}-loss", tag, (got_loss.to(f64) - loss).abs())
    out["dlogits"] = report(f"{what}-dlogits", tag, excess(got_d, d, scale, True))
    assert (got_loss[ign] == 0).all(), "an ignored row has a nonzero loss"
    assert (got_d[ign] == 0).all(), "an ignored row has a nonzero gradient"
    for q, w_ in out.items():
        bound = BOUND[q] if what == "fused" else BOUND[f"{q}_mat"]
        assert w_ <= bound, (what, q, w_, bound)


@pytest.mark.gpu
@pytest.mark.parametrize("c", CE_CASES)
def test_head_ce_matches_fp64(c, request):
    from audiolm_pytorch_b200 import ops

    tag = request.node.callspec.id
    gen = torch.Generator().manual_seed(zlib.crc32(tag.encode()))
    x, w, bias, labels = ce_operands(c, gen)
    M, V, ignore = c["M"], c["V"], c["ignore"]
    num = torch.tensor([0.75], device=DEV)
    den = torch.tensor([3.0], device=DEV)
    scale = 0.25
    ldd = V + 13

    def fused():
        lse, loss = ops.head_ce_fwd(x, w, bias, labels, ignore)
        dl = torch.empty(M, ldd, dtype=bf16, device=DEV)
        dl.view(torch.int16).fill_(SENT[bf16])
        ops.head_ce_bwd(x, w, bias, labels, ignore, lse, num, den, dl)
        return lse, loss, dl

    lse, loss, dl = fused()
    lse2, loss2, dl2 = fused()
    torch.cuda.synchronize()
    assert torch.equal(lse, lse2) and torch.equal(loss, loss2), "two identical forward calls differ"
    assert torch.equal(dl.view(torch.int16), dl2.view(torch.int16)), "two identical backward calls differ"
    assert (dl[:, V:].view(torch.int16) == SENT[bf16]).all(), "dlogits columns >= V were written"
    assert torch.isfinite(lse).all() and torch.isfinite(loss).all() and torch.isfinite(dl[:, :V]).all()
    logits = x.to(f64) @ w.to(f64).T
    if bias is not None:
        logits = logits + bias.to(f64)
    ign = labels == ignore
    ce_check(tag, "fused", lse, loss, dl[:, :V], ce_ref(logits, labels, ignore, scale), scale, ign)
    # the materialised path on the fp32 logits, in a buffer with NaN past V
    lbuf = torch.full((M, V + 5), math.nan, dtype=f32, device=DEV)
    lbuf[:, :V] = logits.to(f32)
    lg = lbuf[:, :V]
    loss_m, dl_m = ops.ce_fwd_bwd(lg, labels, ignore_index=ignore, scale_num=num, scale_den=den)
    torch.cuda.synchronize()
    assert (dl_m[:, V:] == 0).all(), "the materialised dlogits padding is not zero"
    ce_check(tag, "materialised", None, loss_m, dl_m[:, :V], ce_ref(lg, labels, ignore, scale), scale, ign)


@pytest.mark.gpu
def test_out_of_range_labels_give_nan_rows():
    """a label outside [0, V) that is not ignore_index: NaN row loss and NaN dlogits row on the fused and the
    materialised paths, every other row as usual.  V = 300 runs 3 tiles of 128; V + 1 lies in the last tile's padding,
    where a column index exists but no logit does."""
    from audiolm_pytorch_b200 import ops

    M, V, K, ignore = 300, 300, 128, -1
    gen = torch.Generator().manual_seed(300)
    x = (torch.randn(M, K, generator=gen) * 0.5).to(bf16).to(DEV)
    w = (torch.randn(V, K, generator=gen) * 0.25).to(bf16).to(DEV)
    bias = torch.randn(V, generator=gen).to(DEV)
    labels = torch.randint(0, V, (M,), generator=gen)
    labels[::9] = ignore
    bad_rows = [5, 77, 130, 298]
    labels[bad_rows] = torch.tensor([-5, V, V + 1000, V + 1])
    labels = labels.to(DEV)
    bad = torch.zeros(M, dtype=torch.bool, device=DEV)
    bad[bad_rows] = True
    num = torch.ones(1, device=DEV)
    den = torch.tensor([float(M)], device=DEV)
    lse, loss = ops.head_ce_fwd(x, w, bias, labels, ignore)
    dl = torch.empty(M, V + 8, dtype=bf16, device=DEV)
    dl.view(torch.int16).fill_(SENT[bf16])
    ops.head_ce_bwd(x, w, bias, labels, ignore, lse, num, den, dl)
    logits = x.to(f64) @ w.to(f64).T + bias.to(f64)
    lbuf = logits.to(f32)
    loss_m, dl_m = ops.ce_fwd_bwd(lbuf, labels, ignore_index=ignore, scale_num=num, scale_den=den)
    torch.cuda.synchronize()
    assert torch.isfinite(lse).all(), "the LSE of a row does not depend on its label"
    for what, ls, d in (("fused", loss, dl[:, :V]), ("materialised", loss_m, dl_m[:, :V])):
        assert torch.equal(torch.isnan(ls), bad), f"{what}: NaN loss rows are not exactly the out-of-range labels"
        assert torch.isnan(d[bad]).all() and torch.isfinite(d[~bad]).all(), f"{what}: dlogits NaN rows"
    assert (dl[:, V:].view(torch.int16) == SENT[bf16]).all() and (dl_m[:, V:] == 0).all()
    ok = ~bad
    good_labels = torch.where(bad, ignore, labels)
    ign = good_labels == ignore
    ce_check("out-of-range", "fused", lse[ok], loss[ok], dl[ok, :V],
             [t[ok] for t in ce_ref(logits, good_labels, ignore, 1.0 / M)], 1.0 / M, ign[ok])
    ce_check("out-of-range", "materialised", None, loss_m[ok], dl_m[ok, :V],
             [t[ok] for t in ce_ref(lbuf, good_labels, ignore, 1.0 / M)], 1.0 / M, ign[ok])


# ---- autograd: heads.cross_entropy against F.cross_entropy in fp64 -------------------------------------------------
def ag(kind, b, n, V, d, *, id, Q=1, bias=False, ignore=-1, ignored_group=None, all_ignored=False):
    return pytest.param(dict(kind=kind, b=b, n=n, V=V, d=d, Q=Q, bias=bias, ignore=ignore,
                             ignored_group=ignored_group, all_ignored=all_ignored), id=id)


AG_CASES = [
    ag("linear", 2, 150, 300, 64, bias=True, id="linear-bias"),
    ag("linear", 3, 50, 1025, 128, ignore=0, id="linear-v1025-ignore-0"),
    ag("grouped", 2, 7, 129, 64, Q=3, id="grouped-q3-n7"),
    ag("grouped", 3, 2, 65, 64, Q=3, id="grouped-q3-n2-fewer-positions-than-heads"),
    ag("grouped", 2, 9, 257, 64, Q=3, ignored_group=1, id="grouped-q3-group-1-all-ignored"),
    ag("linear", 2, 40, 300, 64, bias=True, all_ignored=True, id="linear-all-ignored"),
    ag("grouped", 2, 7, 129, 64, Q=3, all_ignored=True, id="grouped-all-ignored"),
]


def head_logits(t, w, b, grouped):
    """fp64 logits [b, n, V] of tokens t [b, n, d]: t w^T + b, or position p against w[p mod Q] when grouped"""
    if grouped:
        idx = torch.arange(t.shape[1], device=t.device) % w.shape[0]
        return torch.einsum("bnd,nvd->bnv", t, w[idx])
    out = t @ w.T
    return out + b if b is not None else out


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["fused", "materialised"])
@pytest.mark.parametrize("c", AG_CASES)
def test_cross_entropy_autograd_matches_fp64(c, path, request):
    from audiolm_pytorch_b200 import heads

    tag = request.node.callspec.id
    gen = torch.Generator().manual_seed(zlib.crc32(tag.encode()))
    b, n, V, d, Q, ignore = c["b"], c["n"], c["V"], c["d"], c["Q"], c["ignore"]
    grouped = c["kind"] == "grouped"
    tokens = (torch.randn(b, n, d, generator=gen) * 0.5).to(bf16).float().to(DEV).requires_grad_()
    wshape = (Q, V, d) if grouped else (V, d)
    weight = (torch.randn(*wshape, generator=gen) * 0.3).to(bf16).float().to(DEV).requires_grad_()
    bias = (torch.randn(V, generator=gen)).to(DEV).requires_grad_() if c["bias"] else None
    labels = torch.randint(0, V, (b, n), generator=gen)
    labels[torch.rand(b, n, generator=gen) < 0.1] = ignore
    if c["ignored_group"] is not None:
        labels[:, c["ignored_group"]::Q] = ignore
    if c["all_ignored"]:
        labels[:] = ignore
    labels = labels.to(DEV)
    lazy = heads.LazyLogits(heads.HeadCache(), tokens, weight, bias, "head", grouped)
    loss = heads.cross_entropy(lazy if path == "fused" else lazy.materialize(), labels, ignore_index=ignore)
    loss.backward()
    torch.cuda.synchronize()
    got = dict(dx=tokens.grad, dw=weight.grad, db=None if bias is None else bias.grad)
    for name, t in got.items():
        assert t is None or torch.isfinite(t).all(), name
    if c["all_ignored"]:
        assert loss.item() == 0.0
        for name, t in got.items():
            assert t is None or torch.count_nonzero(t) == 0, f"{name} is not exactly zero"
        return
    # fp64 reference: mean over the rows that are not ignored, as heads.cross_entropy defines it
    t64 = tokens.detach().to(f64).requires_grad_()
    w64 = weight.detach().to(f64).requires_grad_()
    b64 = None if bias is None else bias.detach().to(f64).requires_grad_()
    logits = head_logits(t64, w64, b64, grouped)
    logits.retain_grad()
    den = max(int((labels != ignore).sum()), 1)
    ref = F.cross_entropy(logits.reshape(-1, V), labels.reshape(-1), ignore_index=ignore, reduction="sum") / den
    ref.backward()
    want = dict(dx=t64.grad, dw=w64.grad, db=None if b64 is None else b64.grad)
    # error scales: the same contractions over |dlogits| and the operands' magnitudes
    ta = t64.detach().abs().requires_grad_()
    wa = w64.detach().abs().requires_grad_()
    ba = None if b64 is None else b64.detach().abs().requires_grad_()
    head_logits(ta, wa, ba, grouped).backward(logits.grad.abs())
    scales = dict(dx=ta.grad, dw=wa.grad, db=None if ba is None else ba.grad)
    worst = dict(ce_mean=report("autograd-loss", tag, (loss.detach().to(f64) - ref.detach()).abs().reshape(1)))
    for name in ("dx", "dw", "db"):
        if got[name] is not None:
            worst[name] = report(f"autograd-{name}", tag, excess(got[name], want[name], scales[name] + TINY, False))
    for q, w_ in worst.items():
        assert w_ <= BOUND[q], (q, w_, BOUND[q])


# ---- host: references, the criterion's sensitivity, coverage, the BLOCK_N copy -------------------------------------
def test_references_match_torch():
    """gemm_ref against a @ b.T and ce_ref against F.cross_entropy with autograd, on small CPU inputs"""
    gen = torch.Generator().manual_seed(1)
    a = torch.randn(2, 5, 9, generator=gen, dtype=f64)
    b = torch.randn(2, 7, 9, generator=gen, dtype=f64)
    bias = torch.randn(7, generator=gen, dtype=f64)
    c0 = torch.randn(2, 5, 7, generator=gen, dtype=f64)
    ref, scale = gemm_ref(a, b, alpha=-0.5, bias=bias, c0=c0)
    for i in range(2):
        assert torch.allclose(ref[i], -0.5 * a[i] @ b[i].T + bias + c0[i], rtol=1e-12, atol=1e-12)
        assert torch.allclose(scale[i], 0.5 * a[i].abs() @ b[i].abs().T + bias.abs() + c0[i].abs(), rtol=1e-12)
    assert (scale >= (ref - c0).abs() - 1e-12).all()
    for ignore in (-1, 0):
        logits = (torch.randn(11, 13, generator=gen, dtype=f64) * 3).requires_grad_()
        labels = torch.randint(0, 13, (11,), generator=gen)
        labels[::4] = ignore
        lse, loss, d = ce_ref(logits.detach(), labels, ignore, scale=0.3)
        want = F.cross_entropy(logits, labels, ignore_index=ignore, reduction="none")
        assert torch.allclose(loss, want.detach(), rtol=1e-12, atol=1e-12)
        assert torch.allclose(lse, torch.logsumexp(logits.detach(), -1), rtol=1e-12)
        (want.sum() * 0.3).backward()
        assert torch.allclose(d, logits.grad, rtol=1e-12, atol=1e-14)


def _fault_operands():
    gen = torch.Generator().manual_seed(7)
    M, N, K = 96, 80, 1000
    a = (torch.randn(1, M, K, generator=gen) * torch.exp2(torch.randint(-8, 9, (1, M, 1), generator=gen))).to(bf16)
    b = (torch.randn(1, N, K, generator=gen) * torch.exp2(torch.randint(-8, 9, (1, N, 1), generator=gen))).to(bf16)
    return a.to(f64), b.to(f64), torch.randn(N, generator=gen, dtype=f64) * 4


@pytest.mark.parametrize("fault", ["k-block-dropped", "k-tail-dropped", "columns-swapped"])
def test_criterion_sees_injected_faults(fault):
    """each fault, applied to the fp64 reference, exceeds the GEMM and GEMV bounds by at least 10x under the
    criterion, for fp32 and for bf16 outputs"""
    a, b, bias = _fault_operands()
    ref, scale = gemm_ref(a, b, alpha=0.5, bias=bias)
    if fault == "columns-swapped":
        got = ref.clone()
        got[..., [10, 11]] = ref[..., [11, 10]]
    else:
        a2 = a.clone()
        a2[..., slice(320, 384) if fault == "k-block-dropped" else slice(960, None)] = 0
        got = gemm_ref(a2, b, alpha=0.5, bias=bias)[0]
    for bf in (False, True):
        worst = excess(got, ref, scale, bf).max().item()
        assert worst >= 10 * max(BOUND["gemm"], BOUND["gemv"]), (fault, bf, worst)


def test_criterion_sees_an_lse_missing_a_tile():
    """an LSE that leaves out one 256-column tile of V = 1025 random logits misses the bound by at least 10x; so do
    the loss of a row whose label is in that tile, and its dlogits with the softmax renormalised over the rest"""
    gen = torch.Generator().manual_seed(8)
    logits = torch.randn(64, 1025, generator=gen, dtype=f64) * 2
    labels = torch.randint(512, 768, (64,), generator=gen)
    lse, loss, d = ce_ref(logits, labels, -1)
    keep = torch.ones(1025, dtype=torch.bool)
    keep[512:768] = False
    lse2 = torch.logsumexp(logits[:, keep], -1)
    assert (lse - lse2).abs().max().item() >= 10 * BOUND["lse"]
    assert ((loss - (lse2 - logits.gather(1, labels[:, None])[:, 0])).abs().max().item() >= 10 * BOUND["loss"])
    d2 = torch.softmax(logits.masked_fill(~keep, -math.inf), -1)
    d2[torch.arange(64), labels] -= 1
    assert excess(d2, d, torch.ones(()), True).max().item() >= 10 * max(BOUND["dlogits"], BOUND["dlogits_mat"])


def test_cases_cover_the_envelope():
    """the case lists hit every layout x BLOCK_N pair, every epilogue path, each acc_mode, the split-K rewrite, the M /
    N / K residues named in the module docstring, one persistent case per BLOCK_N, batched and padded operands and C
    windows; the GEMV, CE and autograd lists their own envelopes"""
    bn = gemm_block_n()
    cs = [p.values[0] for p in GEMM_CASES]
    assert {(lay, blk) for lay in LAYOUTS for blk in (64, 128, 256)} <= {(c["lay"], bn(c["N"])) for c in cs}
    assert {1, 63, 64, 65, 127, 128, 129} <= {c["M"] for c in cs}
    assert {1, 8, 63, 64, 65, 127, 128, 129, 255, 256, 257} <= {c["N"] for c in cs}
    assert {8, 16, 56, 64, 72, 1000, 5460} <= {c["K"] for c in cs} and max(c["K"] for c in cs) >= 16384
    assert {384: 128, 1000: 256, 1025: 256} == {N: bn(N) for N in (384, 1000, 1025)}
    paths = {c["path"] for c in cs}
    assert {"tma", "bf16-reg", "f32-vec", "f32-scalar"} <= paths
    tma = [c for c in cs if c["path"] == "tma"]
    assert {64, 128, 256} <= {bn(c["N"]) for c in tma}                     # NBUF 1 and 2
    assert {True, False} == {c["bias"] for c in tma} and any(c["alpha"] != 1 for c in tma)
    assert any(c["ldc_extra"] > 0 for c in tma) and all(c["rows_extra"] > 0 for c in cs)
    for path in ("bf16-reg", "f32-scalar"):
        assert any(c["path"] == path and c["c_off"] == 1 for c in cs)                          # base off by one
        assert any(c["path"] == path and (c["N"] + c["ldc_extra"]) % 2 == 1 for c in cs)      # odd ldc
    assert {(0, "bf16"), (0, "f32"), (1, "bf16"), (1, "f32"), (2, "f32")} <= {(c["acc"], c["out"]) for c in cs}
    assert {2, 4, 64} <= {c["split"] for c in cs if c["acc"] == 2}
    kb = lambda c: -(-c["K"] // BLOCK_K)  # noqa: E731
    assert any(c["split"] > kb(c) for c in cs)
    assert any(c["split"] <= kb(c) and split_after_rewrite(c["K"], c["split"]) < c["split"] for c in cs)
    assert split_after_rewrite(5 * 64, 4) == 3
    assert any(c["split"] > 1 and c["bias"] for c in cs)
    for blk in (64, 128, 256):
        assert any(bn(c["N"]) == blk and split_after_rewrite(c["K"], c["split"]) * c["batch"]
                   * -(-c["M"] // BLOCK_M) * -(-c["N"] // blk) > H100_SMS for c in cs), blk
    batched = [c for c in cs if c["batch"] > 1]
    assert {2, 3} <= {c["batch"] for c in batched} and {"tma", "bf16-reg"} <= {c["path"] for c in batched}
    assert any(c["gap"] > 0 for c in batched) and all(c["pad"] > 0 for c in batched)
    assert set(LAYOUTS) <= {c["lay"] for c in cs if c["pad"] > 0}
    ex = [c for c in cs if c["exact"]]
    assert set(LAYOUTS) <= {c["lay"] for c in ex} and {"tma", "bf16-reg", "f32-vec"} <= {c["path"] for c in ex}
    assert any(c["split"] > 1 for c in ex) and {0, 1, 2} == {c["acc"] for c in ex}
    assert all(c["K"] <= 1024 and c["alpha"] in (0.5, 1.0) for c in ex)
    # GEMV
    gs = [p.values[0] for p in GEMV_CASES]
    assert set(range(1, 9)) == {c["rows"] for c in gs}
    assert {8, 24, 1021, 6144} <= {c["K"] for c in gs} and any(c["rows"] == 8 and c["K"] == 6144 for c in gs)
    assert {1, 7, 9} <= {c["N"] for c in gs} and max(c["N"] for c in gs) > 4 * H100_SMS * 8
    assert any(c["ldw_extra"] for c in gs) and any(c["ldx_extra"] for c in gs)
    assert any(c["bias"] and c["out"] == "f32" for c in gs) and any(c["out"] == "bf16" for c in gs)
    # cross entropy
    ce = [p.values[0] for p in CE_CASES]
    Vs = {c["V"] for c in ce}
    assert {1, 63, 64, 65, 128, 129, 256, 257, 1025} <= Vs and max(Vs) >= 16385
    assert any((c["V"] - 1) % 256 == 0 and bn(c["V"]) == 256 and c["V"] > 256 for c in ce)   # V = 256 k + 1
    assert {1, 127, 129} <= {c["M"] for c in ce} and any(-(-c["M"] // BLOCK_M) > H100_SMS for c in ce)
    assert {-1, 0} <= {c["ignore"] for c in ce} and any(c["all_ignored"] for c in ce)
    assert {True, False} == {c["bias"] for c in ce}
    ags = [p.values[0] for p in AG_CASES]
    grp = [c for c in ags if c["kind"] == "grouped"]
    assert any(c["n"] < c["Q"] for c in grp) and any(c["n"] % c["Q"] for c in grp)
    assert any(c["ignored_group"] is not None for c in grp)
    assert any(c["all_ignored"] and c["kind"] == k for c in ags for k in ("linear", "grouped"))
    assert any(c["bias"] and c["kind"] == "linear" for c in ags)


def test_block_n_copy_matches_the_library():
    """transformer.gemm_block_n (which best_split_k uses) against the library's pick_block_n, through the tile count
    alm_gemm_head_ce_tiles(N) = ceil(N / pick_block_n(N)); the library loads without a GPU"""
    from audiolm_pytorch_b200 import _lib

    lib = _lib.load()
    bn = gemm_block_n()
    bad = [N for N in range(1, 5001) if lib.alm_gemm_head_ce_tiles(N) != -(-N // bn(N))]
    assert not bad, bad[:10]
