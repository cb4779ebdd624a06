#!/usr/bin/env python
"""Stand-alone timings of the HBM-bound row kernels, attention and every wgmma GEMM shape at C3 sizes (CUDA events,
L2 flushed between iterations).
usage: python tools/bench_kernels.py [geglu] [hc] [attn] [gemm] [dropout] ..."""
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from audiolm_pytorch_b200 import ops  # noqa: E402

dev = "cuda"
bf16, f32 = torch.bfloat16, torch.float32
torch.manual_seed(0)
M, d, H = 16 * 2048, 1024, 8
which = set(sys.argv[1:]) or {"geglu", "hc", "attn"}
flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)


def rnd(*s, dt=bf16, k=1.0):
    return (torch.randn(*s, device=dev) * k).to(dt)


def timeit(name, fn, nbytes=None, flops=None, iters=8):
    for _ in range(2):
        fn()
    ts = []
    for _ in range(iters):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ms = sorted(ts)[len(ts) // 2]
    extra = ""
    if nbytes:
        extra += f"  {nbytes / ms / 1e6:8.0f} GB/s"
    if flops:
        extra += f"  {flops / ms / 1e9:8.0f} TFLOP/s"
    print(f"{name:34s} {ms * 1e3:9.1f} us{extra}", flush=True)


if "geglu" in which:
    ip = 2736
    h = rnd(M, 2 * ip)
    g = rnd(2730, dt=f32)
    gn, st = ops.geglu_ln_fwd(h, g, inner=2730, inner_pad=ip)
    dgn = rnd(M, ip)
    gg = torch.zeros_like(g)
    timeit("geglu_ln_fwd", lambda: ops.geglu_ln_fwd(h, g, inner=2730, inner_pad=ip), nbytes=M * ip * 6)
    timeit("geglu_ln_bwd", lambda: ops.geglu_ln_bwd(h, g, st, dgn, gg, inner=2730, inner_pad=ip), nbytes=M * ip * 10)

if "hc" in which:
    hc = dict(gamma=rnd(d, dt=f32, k=0.1), dyn_alpha=rnd(d, 5, dt=f32, k=0.05), dyn_beta=rnd(d, dt=f32, k=0.05),
              static_alpha=rnd(4, 5, dt=f32), static_beta=rnd(4, dt=f32), alpha_scale=torch.tensor(0.3, device=dev),
              beta_scale=torch.tensor(0.3, device=dev))
    lng = rnd(d, dt=f32)
    R, Y, bp = rnd(M, 4, d), rnd(M, d), rnd(M, 4, dt=f32)
    timeit("hc_pre_fwd", lambda: ops.hc_pre_fwd(hc, lng, R_in=R, Y=Y, beta_prev=bp, M=M, d=d), nbytes=M * d * 22)
    timeit("hc_pre_fwd (no bin)", lambda: ops.hc_pre_fwd(hc, lng, R_in=R, Y=Y, beta_prev=bp, M=M, d=d, want_bin=False),
           nbytes=M * d * 20)
    R_out, bin_, xn, beta, aux = ops.hc_pre_fwd(hc, lng, R_in=R, Y=Y, beta_prev=bp, M=M, d=d)
    x = rnd(M, d, dt=f32)
    aux_x = ops.hc_pre_fwd(hc, lng, x_expand=x, M=M, d=d)[4]
    dR, dxn, dbe, dbin = rnd(M, 4, d), rnd(M, d), rnd(M, 4, dt=f32), rnd(M, d)
    grads = {k_: torch.zeros_like(v_) for k_, v_ in hc.items()}
    gl = torch.zeros_like(lng)

    def hcb(extra):
        return ops.hc_pre_bwd(hc, lng, grads, gl, aux, dR, dxn, dbe, dbin_extra=extra, R_in=R, Y=Y, beta_prev=bp, M=M,
                              d=d)

    timeit("hc_pre_bwd (dbin_extra)", lambda: hcb(dbin), nbytes=M * d * 32)
    timeit("hc_pre_bwd (no dbin_extra)", lambda: hcb(None), nbytes=M * d * 30)
    timeit("hc_pre_bwd (expand)", lambda: ops.hc_pre_bwd(hc, lng, grads, gl, aux_x, dR, dxn, dbe, dbin_extra=dbin,
                                                         x_expand=x, dx_scale=0.5, M=M, d=d), nbytes=M * d * 20)

if "attn" in which:
    q, k, v = rnd(16, 2048, 512), rnd(16, 2048, 64), rnd(16, 2048, 64)
    fl = 4.0 * 16 * 8 * 64 * (2048 * 2049 / 2)
    timeit("attn fwd", lambda: ops.mqa_attn_fwd(q, k, v, heads=8), flops=fl)
    o, lse = ops.mqa_attn_fwd(q, k, v, heads=8)
    do = rnd(16, 2048, 512)
    timeit("attn bwd (delta + fused + dq convert)", lambda: ops.mqa_attn_bwd(q, k, v, o, do, lse, heads=8), flops=2.5 * fl)
    # the trainer always passes a key mask: ~15 % of keys dropped
    km = ops.pack_key_mask(torch.rand(16, 2048, device=dev) > 0.15)
    o, lse = ops.mqa_attn_fwd(q, k, v, heads=8, key_mask=km)
    timeit("attn bwd, key mask", lambda: ops.mqa_attn_bwd(q, k, v, o, do, lse, heads=8, key_mask=km), flops=2.5 * fl)

if "gemm" in which:
    from audiolm_pytorch_b200.transformer import best_split_k

    # every distinct wgmma GEMM shape of one C3 layer (inner 2730, padded 2736): (name, M, N, K)
    fwd = [("fwd to_q", M, 512, d), ("fwd to_kv", M, 128, d), ("fwd to_out", M, d, 512), ("fwd w1", M, 5472, d),
           ("fwd w2", M, d, 2736)]
    dgrad = [("dgrad w2", M, 2736, d), ("dgrad w1", M, d, 5472), ("dgrad to_out", M, 512, d), ("dgrad to_q", M, d, 512),
             ("dgrad to_kv", M, d, 128)]
    wgrads = [("wgrad w2", d, 2730, M), ("wgrad w1 (half)", 2730, d, M), ("wgrad to_out", d, 512, M),
              ("wgrad to_q", 512, d, M), ("wgrad to_kv", 128, d, M)]
    for name, m, n, k in fwd:
        a, b = rnd(m, k), rnd(n, k)
        timeit(f"gemm {name} M{m} N{n} K{k}", lambda a=a, b=b: ops.gemm(a, b), flops=2.0 * m * n * k)
    for name, m, n, k in dgrad:
        a, b = rnd(m, k), rnd(k, n)  # b: the layer's weight read MN-major
        timeit(f"gemm {name} M{m} N{n} K{k}", lambda a=a, b=b: ops.gemm(a, b, b_mn=True), flops=2.0 * m * n * k)
    for name, m, n, k in wgrads:
        s = best_split_k(m, n, k)
        # 2730-wide operands are column slices of wider tensors in the step, which keeps their rows 16-B aligned
        a, b = rnd(k, -(-m // 8) * 8)[:, :m], rnd(k, -(-n // 8) * 8)[:, :n]
        out = torch.zeros(m, n, dtype=f32, device=dev)
        timeit(f"gemm {name} M{m} N{n} K{k} s{s}",
               lambda a=a, b=b, out=out, s=s: ops.gemm(a, b, a_mn=True, b_mn=True, out=out,
                                                        acc_mode=2 if s > 1 else 1, split_k=s),
               flops=2.0 * m * n * k)

if "dropout" in which:
    # every dropout site of a C3 layer with p = 0.1 against p = 0 (the dropout-free kernels), then a C3-shaped
    # training step of the Transformer stack (dim 1024, depth 6, 8 heads, 4 streams, batch 16 x 2048)
    from audiolm_pytorch_b200.transformer import Transformer

    q, k, v = rnd(16, 2048, 512), rnd(16, 2048, 64), rnd(16, 2048, 64)
    do = rnd(16, 2048, 512)
    ip = 2736
    h = rnd(M, 2 * ip)
    g = rnd(2730, dt=f32)
    dgn = rnd(M, ip)
    gg = torch.zeros_like(g)
    y = rnd(M, d)
    for p in (0.0, 0.1):
        drop = (p, 12345, 1) if p > 0 else None
        timeit(f"p={p} attn fwd", lambda: ops.mqa_attn_fwd(q, k, v, heads=8, dropout=drop))
        o, lse = ops.mqa_attn_fwd(q, k, v, heads=8, dropout=drop)
        timeit(f"p={p} attn bwd (delta + fused + dq)", lambda: ops.mqa_attn_bwd(q, k, v, o, do, lse, heads=8, dropout=drop))
        timeit(f"p={p} geglu_ln_fwd", lambda: ops.geglu_ln_fwd(h, g, inner=2730, inner_pad=ip, dropout=drop),
               nbytes=M * ip * 6)
        _, st = ops.geglu_ln_fwd(h, g, inner=2730, inner_pad=ip, dropout=drop)
        timeit(f"p={p} geglu_ln_bwd", lambda: ops.geglu_ln_bwd(h, g, st, dgn, gg, inner=2730, inner_pad=ip, dropout=drop),
               nbytes=M * ip * 10)
        if p > 0:
            timeit(f"p={p} output dropout [M, {d}] in place", lambda: ops.dropout_(y, p, 12345, 2), nbytes=M * d * 4)
    del q, k, v, do, h, dgn, y
    x = torch.randn(16, 2048, d, device=dev)
    steps = {}
    for p in (0.0, 0.1):
        torch.manual_seed(0)
        steps[p] = Transformer(dim=d, depth=6, heads=8, flash_attn=True, attn_dropout=p, ff_dropout=p).to(dev).train()

    def step(tr):
        for prm in tr.parameters():
            prm.grad = None
        tr(x).float().pow(2).mean().backward()

    for rep in range(3):   # alternate the two models
        for p, tr in steps.items():
            timeit(f"p={p} C3 stack fwd+bwd (run {rep})", lambda tr=tr: step(tr), iters=5)
