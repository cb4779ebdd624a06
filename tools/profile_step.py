#!/usr/bin/env python
"""Per-kernel-class / per-GEMM-shape device time of one C3 training step (CUDA events on the launching stream).
Writes a markdown table to stdout; run on the GPU:  python tools/profile_step.py > step_breakdown.md"""
import json
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import bench  # noqa: E402
from audiolm_pytorch_b200 import ops  # noqa: E402
from audiolm_pytorch_b200.audiolm import CoarseTransformer  # noqa: E402
from audiolm_pytorch_b200.heads import cross_entropy  # noqa: E402

dev = torch.device("cuda:0")
torch.manual_seed(1234)
model = CoarseTransformer(**bench.CFG).to(dev).train()
sem, coarse = (t.to(dev) for t in bench.synth_ids(bench.BATCH, 0))
eos = torch.full((bench.BATCH, 1), bench.CFG["codebook_size"], device=dev)


def step():
    for p in model.parameters():
        p.grad = None
    sl, cl = model(semantic_token_ids=sem, coarse_token_ids=coarse)
    loss = (cross_entropy(sl, sem) * sl.shape[1] + cross_entropy(cl, torch.cat((coarse, eos), 1)) * cl.shape[1]) / (
        sl.shape[1] + cl.shape[1])
    loss.backward()


for _ in range(3):
    step()
torch.cuda.synchronize()
a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
a.record()
for _ in range(3):
    step()
b.record()
torch.cuda.synchronize()
step_ms = a.elapsed_time(b) / 3
ops.PROFILE_SHAPES = True
ops.profile_start()
step()
prof = ops.profile_stop()
pk = bench.peaks()
print(f"# C3 step breakdown (batch 16 x 2048, d1024 L6) — step {step_ms:.2f} ms\n")
print("| kernel class | launches | ms | TFLOP/s | % of bf16 sustained peak |")
print("|---|---|---|---|---|")
tot = 0.0
for cls, (ms, work, n) in sorted(prof.items(), key=lambda kv: -kv[1][0]):
    rate = work / (ms * 1e-3) if ms else 0
    tot += ms
    if ops.CLASS_UNIT.get(cls) == "byte":  # HBM-bound classes: GB/s of algorithmic bytes vs the HBM peak
        print(f"| {cls} | {n} | {ms:.3f} | {rate / 1e9:.0f} GB/s | {100 * rate / 1e9 / pk['hbm']:.0f}% of HBM |")
    else:
        print(f"| {cls} | {n} | {ms:.3f} | {rate / 1e12:.0f} | {100 * rate / 1e12 / pk['tf_sustained']:.0f}% |")
print(f"\ntimed classes total {tot:.2f} ms of {step_ms:.2f} ms step; the rest is hyper-connection / GEGLU / CE / torch glue "
      "kernels (see the ncu launch list).")
