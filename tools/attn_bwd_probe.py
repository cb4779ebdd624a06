#!/usr/bin/env python
"""Attention backward at the C3 shape (b 16, 8 heads sharing one 64-wide k/v head, n 2048, causal): the whole
backward (delta + fused kernel + dq conversion) with and without a key mask (~15 % of keys dropped, as the trainer
always passes one), CUDA events with L2 flushed; the per-kernel split from torch.profiler; with `variants`, the
same masked backward through the score-bias, dropout and bias + dropout instantiations; and, when libalm_b200.so
was built with -DALM_ATTN_BWD_TRACE, the per-phase cycle table of CTA 0 (key block 0: 128 tiles, the 8 with query
block 0 on the causal diagonal).
    ALM_EXTRA_NVCC_FLAGS=-DALM_ATTN_BWD_TRACE python -m audiolm_pytorch_b200.build --force   # for the phase table
    python tools/attn_bwd_probe.py [variants]"""
import ctypes
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from audiolm_pytorch_b200 import _lib, ops  # noqa: E402

dev = "cuda"
bf16 = torch.bfloat16
B, H, N = 16, 8, 2048
ITERS, STAMPS = 128, 8   # AB_TRACE_ITERS, AB_TRACE_STAMPS of attn_bwd_wgmma.cu
# stamp i -> i + 1 (stamp 7 -> stamp 0 of the next tile)
PHASES = ["wait Q/dO/lse/delta", "issue S^T, dP^T", "wait S^T + exp", "dV issue, wait dP^T, dS -> smem",
          "dS^T barrier", "dK, dQ issue + wait", "dQ out", "loop"]

torch.manual_seed(0)
flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
q = torch.randn(B, N, H * 64, device=dev).to(bf16)
k = torch.randn(B, N, 64, device=dev).to(bf16)
v = torch.randn(B, N, 64, device=dev).to(bf16)
d_o = torch.randn(B, N, H * 64, device=dev).to(bf16)
key_mask = torch.rand(B, N, device=dev) > 0.15
key_mask[:, 0] = True
flops = 10.0 * B * H * 64 * (N * N - N * (N - 1) / 2)


def time_us(fn, iters=10):
    for _ in range(3):
        fn()
    ts = []
    for _ in range(iters):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) * 1e3)
    ts.sort()
    return ts[len(ts) // 2], ts[0], ts[-1]


print(torch.cuda.get_device_name(), flush=True)
for name, mask in (("unmasked", None), ("key mask", key_mask)):
    o, lse = ops.mqa_attn_fwd(q, k, v, heads=H, key_mask=mask)
    med, lo, hi = time_us(lambda: ops.mqa_attn_bwd(q, k, v, o, d_o, lse, heads=H, key_mask=mask))
    print(f"attn bwd {name:9s} (delta + fused + dq convert) {med:8.1f} us ({lo:.1f}-{hi:.1f})  "
          f"{flops / med / 1e6:6.1f} TFLOP/s", flush=True)

if "variants" in sys.argv[1:]:
    # the flash_attn=False path passes an fp32 [heads, n_q, n_k] score bias and accumulates its gradient
    bias = torch.randn(H, N, N, device=dev) * 0.5
    dbias = torch.zeros_like(bias)
    drop = (0.1, 12345, 1)
    for name, kw in (("score bias", dict(bias=bias, dbias=dbias)), ("dropout 0.1", dict(dropout=drop)),
                     ("bias + dropout", dict(bias=bias, dbias=dbias, dropout=drop))):
        fkw = {k_: v_ for k_, v_ in kw.items() if k_ != "dbias"}
        o, lse = ops.mqa_attn_fwd(q, k, v, heads=H, key_mask=key_mask, **fkw)
        med, lo, hi = time_us(lambda: ops.mqa_attn_bwd(q, k, v, o, d_o, lse, heads=H, key_mask=key_mask, **kw))
        print(f"attn bwd key mask, {name:14s} (delta + fused + dq convert) {med:8.1f} us ({lo:.1f}-{hi:.1f})",
              flush=True)
    del bias, dbias

o, lse = ops.mqa_attn_fwd(q, k, v, heads=H, key_mask=key_mask)
with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    for _ in range(5):
        ops.mqa_attn_bwd(q, k, v, o, d_o, lse, heads=H, key_mask=key_mask)
    torch.cuda.synchronize()
print("\nkey-masked backward, per kernel (torch.profiler, 5 calls, L2 warm):")
for ev in sorted(prof.key_averages(), key=lambda e: -e.device_time_total):
    if ev.device_time_total > 0:
        print(f"  {ev.key[:70]:70s} {ev.device_time_total / ev.count:8.1f} us x {ev.count}")

lib = _lib.load()
if not hasattr(lib, "alm_attn_bwd_trace_read"):
    print("\n(no phase table: build with ALM_EXTRA_NVCC_FLAGS=-DALM_ATTN_BWD_TRACE)")
    sys.exit(0)
ops.mqa_attn_bwd(q, k, v, o, d_o, lse, heads=H, key_mask=key_mask)
torch.cuda.synchronize()
buf = (ctypes.c_longlong * (2 * ITERS * STAMPS))()
assert lib.alm_attn_bwd_trace_read(buf) == 0
t = torch.tensor(list(buf), dtype=torch.int64).view(2, ITERS, STAMPS)
nxt = torch.cat((t[:, 1:, :1], t[:, -1:, -1:]), dim=1)     # stamp 0 of the next tile (last tile: its own end)
d = torch.cat((t[:, :, 1:] - t[:, :, :-1], nxt - t[:, :, -1:]), dim=2).double()
sel = slice(2, ITERS - 1)    # steady state: skip the pipeline fill and the last tile
print(f"\nCTA 0 phase table (SM clock cycles per tile, mean over tiles {sel.start}..{sel.stop - 1}; "
      "warp 0 of each warpgroup)")
print(f"  {'phase':34s} {'wg0':>8s} {'wg1':>8s}")
for i, name in enumerate(PHASES):
    print(f"  {name:34s} {d[0, sel, i].mean():8.0f} {d[1, sel, i].mean():8.0f}")
per_tile = (t[:, sel.start + 1:sel.stop + 1, 0] - t[:, sel, 0]).double().mean(1)
print(f"  {'tile total':34s} {per_tile[0]:8.0f} {per_tile[1]:8.0f}")
print(f"  whole CTA: {(t[0, -1, -1] - t[0, 0, 0]).item()} cycles for {ITERS} tiles; "
      f"wg1 - wg0 skew at 'issue S^T, dP^T': {(t[1, sel, 2] - t[0, sel, 2]).double().mean():.0f} cycles")
