"""Decode-step latency: one-kernel stack step vs the multi-kernel step (both replayed from a CUDA graph), C5 shapes.
    python tools/decode_bench.py [cache_len]"""
import json
import sys
import time

import torch

sys.path.insert(0, ".")
from audiolm_pytorch_b200 import decode  # noqa: E402
from audiolm_pytorch_b200.transformer import Transformer  # noqa: E402

dev = "cuda"
n0 = int(sys.argv[1]) if len(sys.argv) > 1 else 600
torch.manual_seed(0)
tr = Transformer(dim=1024, depth=6, heads=8, flash_attn=True).to(dev).eval()
res = {}
default = decode.FUSED_STACK_STEP
for b in (1, 4):
    for fused in (False, True):
        decode.FUSED_STACK_STEP = fused
        dec = decode.StackDecoder(tr, b, 2048)
        dec.load_cache(torch.randn(6, 2, b, n0, 64, device=dev))
        x = torch.randn(b, 1024, device=dev)
        y = torch.zeros(b, 1024, device=dev, dtype=torch.bfloat16)

        def fn():
            y.copy_(dec.step(x))

        g = decode.GraphedStep(fn, [dec.len, y])
        for _ in range(20):
            g()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        iters = 200
        e0.record()
        for _ in range(iters):
            g()
        e1.record()
        torch.cuda.synchronize()
        res[f"b{b}_{'fused' if fused else 'multi'}_us_per_step"] = round(e0.elapsed_time(e1) * 1e3 / iters, 2)
        res[f"b{b}_{'fused' if fused else 'multi'}_timeouts"] = dec.barrier_timeouts()
        assert torch.isfinite(y.float()).all()
decode.FUSED_STACK_STEP = default
res["cache_len"] = n0
print(json.dumps(res))
