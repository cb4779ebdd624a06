"""SoundStream C1 encode / decode with and without squeeze_excite, interleaved in one process.

    python tools/bench_codec_se.py [--batch 64] [--reps 7] [--iters 3]

C1 shapes (32 channels, strides 2/4/5/8, 2 s at 24 kHz = 48 000 samples -> 150 frames, 8-stage RVQ, no local attention).
Both models have the same conv weights; the SE model adds the units' SqueezeExcite.  Each repetition times `iters`
calls of each (model, direction) with CUDA events, alternating the models; the median over repetitions is printed with
the card's name and power limit.  Needs a GPU.
"""
from __future__ import annotations

import argparse
import statistics
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))


def card():
    name = torch.cuda.get_device_name()
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        q = "power limit unknown"
    return f"{name} ({q})"


def timed(fn, iters):
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    stop.record()
    torch.cuda.synchronize()
    return start.elapsed_time(stop) / iters


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
    kw = dict(codebook_size=1024, rq_num_quantizers=8, target_sample_hz=24000, use_local_attn=False)
    torch.manual_seed(0)
    plain = SoundStream(**kw)
    se = SoundStream(**kw, squeeze_excite=True)
    se.load_state_dict(plain.state_dict(), strict=False)   # same convs and codebooks; SE weights from their init
    g = torch.Generator().manual_seed(1)
    for m in (plain, se):
        for i, layer in enumerate(m.rq.rvqs[0].layers):
            layer._codebook.embed.copy_(torch.randn(1, 1024, 512, generator=torch.Generator().manual_seed(i)) * 0.05)
            layer._codebook.initted.fill_(True)
    plain, se = plain.to(dev).eval(), se.to(dev).eval()
    assert plain._tc_plan() is not None and se._tc_plan() is not None
    assert plain._tc_plan_dec() is not None and se._tc_plan_dec() is not None
    wave = torch.randn(args.batch, 48000, generator=g).to(dev)
    frames = torch.randn(args.batch, 150, 512, generator=g).to(dev) * 0.5
    work = {(name, d): fn for name, m in (("off", plain), ("on", se))
            for d, fn in (("encode", lambda m=m: m(wave, return_encoded=True)),
                          ("decode", lambda m=m: m.decode(frames)))}
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
    print(f"C1 SoundStream, batch {args.batch} x 48000 samples (150 frames), median of {args.reps} x {args.iters} calls")
    for d in ("encode", "decode"):
        off, on = statistics.median(times[("off", d)]), statistics.median(times[("on", d)])
        spread = {k: (min(v), max(v)) for k, v in times.items() if k[1] == d}
        print(f"  {d}: squeeze_excite off {off:.3f} ms ({spread[('off', d)][0]:.3f}-{spread[('off', d)][1]:.3f}), "
              f"on {on:.3f} ms ({spread[('on', d)][0]:.3f}-{spread[('on', d)][1]:.3f}), +{100 * (on / off - 1):.1f} %")


if __name__ == "__main__":
    main()
