"""Attention forward and backward alone at the C3 shape (b 16, n 2048, causal, key mask, no bias, no dropout) for
heads = 8 and dim_head = 32, 64, 128: the table of DESIGN.md section 6.

    python tools/bench_attn_dim_head.py [--reps 5] [--iters 20]

CUDA events around `iters` back-to-back calls, after a warm-up of every shape; between calls the operands rotate over
enough independent copies to exceed the 50 MB L2, so no call finds its inputs cached by the previous one.  Each row is
the median over `reps` repetitions with the min-max spread.  The card's name, power limit and clocks are printed with
the numbers.  Algorithmic work: 2 matmuls x 2 FLOP x h x D x n^2 / 2 per sequence forward (the causal half), 2.5x that
backward (5 matmuls); the backward time includes alm_attn_delta and the dq conversion, as ops.mqa_attn_bwd runs them.
There is no CPU path: without a GPU the script fails."""
import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from audiolm_pytorch_b200 import ops  # noqa: E402

B, N, H = 16, 2048, 8
L2_BYTES = 50 * 2 ** 20


def card():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # the numbers are still valid, but say that the card's state is unknown
        out = f"nvidia-smi unavailable ({e})"
    return out


def operands(D, copies):
    gen = torch.Generator(device="cuda").manual_seed(D)
    mk = lambda *s: torch.randn(*s, device="cuda", generator=gen).to(torch.bfloat16)  # noqa: E731
    sets = []
    for _ in range(copies):
        mask = torch.rand(B, N, device="cuda", generator=gen) > 0.1
        sets.append(dict(q=mk(B, N, H * D), k=mk(B, N, D), v=mk(B, N, D), d_o=mk(B, N, H * D),
                         mask=ops.pack_key_mask(mask)))
    return sets


def time_ms(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for i in range(iters):
        fn(i)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_attn_dim_head needs a GPU: there is no CPU timing to report")
    print(f"# {card()}  (name, power limit, max SM clock, SM clock before the run)")
    rows = []
    for D in (32, 64, 128):
        per_set = (2 * B * N * H * D + 2 * B * N * D) * 2          # q, d_o, k, v in bf16
        sets = operands(D, max(2, -(-2 * L2_BYTES // per_set)))
        saved = [ops.mqa_attn_fwd(s["q"], s["k"], s["v"], heads=H, key_mask=s["mask"]) for s in sets]

        def fwd(i):
            s = sets[i % len(sets)]
            ops.mqa_attn_fwd(s["q"], s["k"], s["v"], heads=H, key_mask=s["mask"])

        def bwd(i):
            s, (o, lse) = sets[i % len(sets)], saved[i % len(sets)]
            ops.mqa_attn_bwd(s["q"], s["k"], s["v"], o, s["d_o"], lse, heads=H, key_mask=s["mask"])

        flop_f = 2 * 2 * H * D * N * N / 2 * B
        for name, fn, flop in (("fwd", fwd, flop_f), ("bwd", bwd, 2.5 * flop_f)):
            time_ms(fn, args.iters)                                  # warm-up of this shape
            ts = [time_ms(fn, args.iters) for _ in range(args.reps)]
            med = statistics.median(ts)
            rows.append(dict(dim_head=D, heads=H, what=name, ms=round(med, 4), ms_min=round(min(ts), 4),
                             ms_max=round(max(ts), 4), tflops=round(flop / med / 1e9, 1)))
            print(f"dim_head {D:3d}  {name}  {med:7.3f} ms  [{min(ts):.3f}, {max(ts):.3f}]  "
                  f"{flop / med / 1e9:6.1f} TFLOP/s (algorithmic)")
    print(f"# {card()}  (after the run)")
    print(json.dumps(dict(shape=dict(b=B, n=N, heads=H, causal=True, key_mask=True), card=card(), rows=rows)))


if __name__ == "__main__":
    main()
