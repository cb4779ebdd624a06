"""SoundStream C1 residual VQ with Euclidean, cosine-similarity and projected (codebook_dim 64 / 128) codebooks,
interleaved in one process.

    python tools/bench_rvq_options.py [--batches 1 16 64] [--reps 7] [--iters 5]

C1 shapes: 32 channels, strides 2/4/5/8, 2 s at 24 kHz = 48 000 samples -> 150 frames per clip, codebook_dim 512,
1024 codes, 8 stages, no local attention; the four models share their conv weights.  Times, with CUDA events after a
warm-up, the median over repetitions of `iters` calls each, alternating the models:
- search only: `ss.rq(h)` on the encoder output (projections included where the model has them);
- tokenize: wave -> ids end to end.
Prints the card's name and power limit.  Needs a GPU.
"""
from __future__ import annotations

import argparse
import statistics
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
from bench_codec_se import card, timed  # noqa: E402

OPTIONS = {"euclid": {}, "cosine": dict(use_cosine_sim=True), "proj64": dict(codebook_dim=64),
           "proj128": dict(codebook_dim=128)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 16, 64])
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--iters", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    from audiolm_pytorch_b200.soundstream import SoundStream

    dev = torch.device("cuda")
    base = dict(codebook_size=1024, rq_num_quantizers=8, target_sample_hz=24000, use_local_attn=False)
    torch.manual_seed(0)
    models = {k: SoundStream(rq_kwargs=kw, **base) for k, kw in OPTIONS.items()}
    shared = {k: v for k, v in models["euclid"].state_dict().items() if not k.startswith("rq.")}
    for name, m in models.items():
        m.load_state_dict(shared, strict=False)
        rvq = m.rq.rvqs[0]
        for i, layer in enumerate(rvq.layers):
            g = torch.Generator().manual_seed(i)
            e = torch.randn(layer._codebook.embed.shape, generator=g)
            layer._codebook.embed.copy_(e / e.norm(dim=-1, keepdim=True) if name == "cosine" else e * 0.05)
            layer._codebook.initted.fill_(True)
    models = {k: m.to(dev).eval() for k, m in models.items()}
    print(f"card: {card()}")
    for B in args.batches:
        wave = torch.randn(B, 48000, generator=torch.Generator().manual_seed(1)).to(dev)
        with torch.inference_mode():
            h = models["euclid"].encode_frames(wave[:, None, :])
        work = {}
        for k, m in models.items():
            work[(k, "search")] = lambda m=m: m.rq(h)
            work[(k, "tokenize")] = lambda m=m: m.tokenize(wave)
        times = {k: [] for k in work}
        with torch.inference_mode():
            for fn in work.values():   # warm-up: module load, codebook and weight packing
                fn()
                fn()
            torch.cuda.synchronize()
            for _ in range(args.reps):
                for k, fn in work.items():
                    times[k].append(timed(fn, args.iters))
        print(f"C1 SoundStream, batch {B} x 48000 samples ({h.shape[0] * h.shape[1]} rows of {h.shape[2]}), median of "
              f"{args.reps} x {args.iters} calls")
        for k, v in times.items():
            print(f"  B={B} {k[0]} {k[1]}: {statistics.median(v):.3f} ms ({min(v):.3f}-{max(v):.3f})")


if __name__ == "__main__":
    main()
