#!/usr/bin/env python
"""C5 (BASELINE.json configs[4]): autoregressive decode latency with the KV cache, batch 1, d1024 L6 h8 models.
Reports ms per generated token for Semantic / Coarse / Fine .generate() and the codec decode, plus the card name and
its power limit (both are part of the numbers).

    python tools/bench_decode.py [steps]                 flash_attn=True, 4 residual streams (C5 as configured)
    python tools/bench_decode.py [steps] --no-flash      flash_attn=False: relative-position / cross / fine 2-D bias
    python tools/bench_decode.py [steps] --streams 1     num_residual_streams=1 (plain residual)
"""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from audiolm_pytorch_b200 import _lib  # noqa: E402
from audiolm_pytorch_b200.audiolm import (CoarseTransformer, CoarseTransformerWrapper, FineTransformer,  # noqa: E402
                                          FineTransformerWrapper, SemanticTransformer, SemanticTransformerWrapper)
from audiolm_pytorch_b200.soundstream import SoundStream  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("steps", nargs="?", type=int, default=64, help="tokens per generate() window")
ap.add_argument("--no-flash", action="store_true", help="flash_attn=False (the reference's constructor default)")
ap.add_argument("--streams", type=int, default=4, choices=range(1, 9), help="num_residual_streams")
ap.add_argument("--skip-codec", action="store_true", help="do not time the codec decode")
args = ap.parse_args()


def card():
    """device name and enforced power limit (nvidia-smi query; 'unknown' when it is not available)"""
    limit = "unknown"
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        if r.returncode == 0 and r.stdout.strip():
            limit = r.stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pass
    return torch.cuda.get_device_name(), limit


dev = "cuda"
torch.manual_seed(0)
kw = dict(dim=1024, depth=6, heads=8, flash_attn=not args.no_flash, num_residual_streams=args.streams)
steps = args.steps
codec = SoundStream(codebook_size=1024, rq_num_quantizers=8, use_local_attn=False)
for l in codec.rq.rvqs[0].layers:
    l._codebook.embed.normal_(0, 0.3)
    l._codebook.initted.fill_(True)
codec = codec.to(dev).eval()
sem = SemanticTransformerWrapper(transformer=SemanticTransformer(num_semantic_tokens=500, **kw).to(dev),
                                 unique_consecutive=False)
coarse = CoarseTransformerWrapper(transformer=CoarseTransformer(num_semantic_tokens=500, codebook_size=1024,
                                                                num_coarse_quantizers=3, **kw).to(dev),
                                  codec=codec, unique_consecutive=False)
fine = FineTransformerWrapper(transformer=FineTransformer(num_coarse_quantizers=3, num_fine_quantizers=5,
                                                          codebook_size=1024, **kw).to(dev), codec=codec)
out = {}


def timed(name, fn, n_tokens, reps=3, count=None):
    fn()  # warm-up (packs weights, captures the decode graphs)
    torch.cuda.synchronize()
    times, r = [], None
    for _ in range(reps):
        _lib.reset_launch_count()
        t0 = time.perf_counter()
        r = fn()
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t0) * 1e3 / (count(r) if count else n_tokens))
    times.sort()
    out[name] = {"ms_per_token": times[len(times) // 2], "ms_per_token_min": times[0], "ms_per_token_max": times[-1],
                 "tokens": n_tokens, "alm_launches_per_token": _lib.launch_count() / n_tokens}
    return r


# random weights may emit EOS early: time per token actually generated in each repetition
timed("semantic", lambda: sem.generate(max_length=steps, batch_size=1), steps, count=lambda r: max(int(r.shape[1]), 1))
sem_ids = torch.randint(0, 500, (1, 500), device=dev)
c = timed("coarse", lambda: coarse.generate(semantic_token_ids=sem_ids, max_time_steps=steps // 3), steps // 3 * 3)
c = c.clamp(min=0)
timed("fine", lambda: fine.generate(coarse_token_ids=torch.randint(0, 1024, (1, steps // 5, 3), device=dev)), steps // 5 * 5)
if not args.skip_codec:
    idx = torch.randint(0, 1024, (1, 512, 8), device=dev)
    timed("codec_decode_512_frames", lambda: codec.decode_from_codebook_indices(idx), 512)
name, limit = card()
print(json.dumps({"config": f"C5 decode, batch 1, KV cache, d1024 L6 h8, flash_attn={not args.no_flash}, "
                            f"num_residual_streams={args.streams}",
                  "device": name, "power_limit": limit, "window_steps": steps, **out}))
