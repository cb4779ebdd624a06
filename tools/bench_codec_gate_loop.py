"""SoundStream C1 encode / decode with and without use_gate_loop_layers, interleaved in one process, and each gate-loop
layer's launch time against its HBM floor.

    python tools/bench_codec_gate_loop.py [--batch 64] [--reps 7] [--iters 3]

C1 shapes (32 channels, strides 2/4/5/8, 2 s at 24 kHz = 48 000 samples -> 150 frames, 8-stage RVQ, no local attention).
Both models have the same conv weights; the gate-loop model adds a Residual(ChannelTranspose(GateLoop(C))) after every
encoder and decoder block.  Each repetition times `iters` calls of each (model, direction) with CUDA events, alternating
the models; the median and range over repetitions are printed with the card's name and power limit.  The per-layer
table times ops.codec_gate_loop_tc (projection + scan) alone at each layer's shape; its floor is the bytes the shapes
force (read x and write y in C8S, 4 B per value each) at 3.35 TB/s.  Needs a GPU.
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
    gated = SoundStream(**kw, use_gate_loop_layers=True)
    # same convs and codebooks (the gate loops shift the Sequential indices); gate-loop weights from their init
    shifted = {0: 0, 1: 1, 2: 3, 3: 5, 4: 7, 5: 9}
    sd = {}
    for k, v in plain.state_dict().items():
        part, i, *rest = k.split(".")
        if part in ("encoder", "decoder"):
            k = ".".join((part, str(shifted[int(i)]), *rest))
        sd[k] = v
    gated.load_state_dict(sd, strict=False)
    g = torch.Generator().manual_seed(1)
    for m in (plain, gated):
        for i, layer in enumerate(m.rq.rvqs[0].layers):
            layer._codebook.embed.copy_(torch.randn(1, 1024, 512, generator=torch.Generator().manual_seed(i)) * 0.05)
            layer._codebook.initted.fill_(True)
    plain, gated = plain.to(dev).eval(), gated.to(dev).eval()
    assert plain._tc_plan() is not None and gated._tc_plan() is not None
    assert plain._tc_plan_dec() is not None and gated._tc_plan_dec() is not None
    wave = torch.randn(args.batch, 48000, generator=g).to(dev)
    frames = torch.randn(args.batch, 150, 512, generator=g).to(dev) * 0.5
    work = {(name, d): fn for name, m in (("off", plain), ("on", gated))
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
    from audiolm_pytorch_b200 import ops

    layers = []   # (side, C, T, launch) of every gate-loop layer at its C1 shape
    T = 48000
    for rus, down, gl in gated._tc_plan()[1]:
        T //= down.stride
        layers.append(("encoder", gl, T))
    for up, rus, gl in gated._tc_plan_dec()[1]:
        T *= up.upsample_factor
        layers.append(("decoder", gl, T))
    layers = [(side, gl.norm.gamma.numel(), T, gl) for side, gl, T in layers]
    inputs = {(side, C, T): ops.c8s_pack(torch.randn(args.batch, C, T, generator=g).to(dev) * 0.3)
              for side, C, T, _ in layers}
    layer_ms = {}
    with torch.inference_mode():
        for side, C, T, gl in layers:
            fn = lambda gl=gl, h=inputs[(side, C, T)]: gl.block_tc(h)   # noqa: E731
            fn()
            torch.cuda.synchronize()
            layer_ms[(side, C, T)] = statistics.median(timed(fn, args.iters * 3) for _ in range(args.reps))
    print(f"card: {card()}")
    print(f"C1 SoundStream, batch {args.batch} x 48000 samples (150 frames), median of {args.reps} x {args.iters} calls")
    for d in ("encode", "decode"):
        off, on = statistics.median(times[("off", d)]), statistics.median(times[("on", d)])
        spread = {k: (min(v), max(v)) for k, v in times.items() if k[1] == d}
        print(f"  {d}: gate loops off {off:.3f} ms ({spread[('off', d)][0]:.3f}-{spread[('off', d)][1]:.3f}), "
              f"on {on:.3f} ms ({spread[('on', d)][0]:.3f}-{spread[('on', d)][1]:.3f}), +{100 * (on / off - 1):.1f} %")
    print("  gate-loop launches (projection + scan), median:")
    for (side, C, T), ms in layer_ms.items():
        floor_ms = 8.0 * args.batch * C * T / 3.35e12 * 1e3
        print(f"    {side} C={C:3d} T={T:5d}: {ms:.3f} ms, HBM floor {floor_ms:.3f} ms ({ms / floor_ms:.1f}x)")


if __name__ == "__main__":
    main()
