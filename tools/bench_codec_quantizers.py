"""SoundStream C1 with the residual VQ, FSQ and LFQ quantizers, interleaved in one process.

    python tools/bench_codec_quantizers.py [--batch 64] [--reps 7] [--iters 3]

C1 shapes (32 channels, strides 2/4/5/8, 2 s at 24 kHz = 48 000 samples -> 150 frames, codebook_dim 512, 8 stages, no
local attention); FSQ levels [8, 5, 5, 5] (codebook 1000), LFQ codebook 1024; the three models share conv weights.
Times, with CUDA events and the median over repetitions of `iters` calls each, alternating the models:
- the FSQ / LFQ kernels alone (alm_sq_encode on the encoder output, alm_sq_decode on its indices) against their HBM
  floor: the bytes the shapes force (rows in and out, indices, projection weights) at 3.35 TB/s;
- encode (wave -> quantized + ids) and decode (ids -> wave) end to end for each quantizer.
Prints the card's name and power limit.  Needs a GPU.
"""
from __future__ import annotations

import argparse
import statistics
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from bench_codec_se import card, timed  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--iters", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    from audiolm_pytorch_b200.soundstream import SoundStream

    dev = torch.device("cuda")
    base = dict(rq_num_quantizers=8, target_sample_hz=24000, use_local_attn=False)
    torch.manual_seed(0)
    models = {"rvq": SoundStream(codebook_size=1024, **base),
              "fsq": SoundStream(finite_scalar_quantizer_levels=[8, 5, 5, 5], use_finite_scalar_quantizer=True, **base),
              "lfq": SoundStream(codebook_size=1024, use_lookup_free_quantizer=True, **base)}
    shared = {k: v for k, v in models["rvq"].state_dict().items() if not k.startswith("rq.")}
    for i, layer in enumerate(models["rvq"].rq.rvqs[0].layers):
        layer._codebook.embed.copy_(torch.randn(1, 1024, 512, generator=torch.Generator().manual_seed(i)) * 0.05)
        layer._codebook.initted.fill_(True)
    for name in ("fsq", "lfq"):
        models[name].load_state_dict(shared, strict=False)
    models = {k: m.to(dev).eval() for k, m in models.items()}
    wave = torch.randn(args.batch, 48000, generator=torch.Generator().manual_seed(1)).to(dev)
    with torch.inference_mode():
        h = models["fsq"].encode_frames(wave[:, None, :])
        ids = {k: m(wave, return_encoded=True)[1] for k, m in models.items()}
        codes = {k: models[k].rq(h)[1] for k in ("fsq", "lfq")}
    N, D = h.shape[0] * h.shape[1], h.shape[2]
    work, floor = {}, {}
    for k in ("fsq", "lfq"):
        rq, c = models[k].rq, codes[k]
        w_bytes = 4 * (2 * rq.codebook_dim * D + rq.codebook_dim + D)
        work[(k, "kernel encode")] = lambda rq=rq: rq(h)
        work[(k, "kernel decode")] = lambda rq=rq, c=c: rq.get_output_from_indices(c)
        floor[(k, "kernel encode")] = (2 * N * D * 4 + c.numel() * c.element_size() + w_bytes) / HBM_BYTES_PER_S * 1e3
        floor[(k, "kernel decode")] = (N * D * 4 + c.numel() * c.element_size() + w_bytes) / HBM_BYTES_PER_S * 1e3
    for k, m in models.items():
        work[(k, "encode")] = lambda m=m: m(wave, return_encoded=True)
        work[(k, "decode")] = lambda m=m, i=ids[k]: m.decode_from_codebook_indices(i)
    times = {k: [] for k in work}
    with torch.inference_mode():
        for fn in work.values():   # warm-up: module load, weight packing
            fn()
            fn()
        torch.cuda.synchronize()
        for _ in range(args.reps):
            for k, fn in work.items():
                times[k].append(timed(fn, args.iters))
    print(f"card: {card()}")
    print(f"C1 SoundStream, batch {args.batch} x 48000 samples (150 frames, {N} rows of {D}), median of "
          f"{args.reps} x {args.iters} calls")
    for k, v in times.items():
        med = statistics.median(v)
        extra = f", HBM floor {floor[k] * 1e3:.1f} us ({100 * floor[k] / med:.0f} % of it)" if k in floor else ""
        print(f"  {k[0]} {k[1]}: {med:.3f} ms ({min(v):.3f}-{max(v):.3f}){extra}")


if __name__ == "__main__":
    main()
