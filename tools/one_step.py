#!/usr/bin/env python
"""Exactly N C3 training steps exactly as bench.py times them (CoarseTransformerWrapper.forward with its key mask + FCM
mask, loss, backward) with no other GPU work - a clean target for a profiler."""
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import bench  # noqa: E402
from audiolm_pytorch_b200.audiolm import CoarseTransformer, CoarseTransformerWrapper  # noqa: E402
from audiolm_pytorch_b200.parallel import FlatGradBucket  # noqa: E402

n = int(sys.argv[1]) if len(sys.argv) > 1 else 1
flash = "--no-flash" not in sys.argv
dev = torch.device("cuda:0")
torch.manual_seed(1234)
model = CoarseTransformer(**{**bench.CFG, "flash_attn": flash}).to(dev).train()
wrapper = CoarseTransformerWrapper(transformer=model, codec=bench._CodecStub()).train()
bucket = FlatGradBucket(model.parameters()).attach(model)
sem, coarse = (t.to(dev) for t in bench.synth_wrapper_ids(bench.BATCH, 0))
for _ in range(n):
    bucket.zero_()
    model.transformer.invalidate_weight_cache()
    model._heads.clear()
    loss = wrapper(semantic_token_ids=sem, coarse_token_ids=coarse, return_loss=True)
    loss.backward()
torch.cuda.synchronize()
print("loss", loss.item())
