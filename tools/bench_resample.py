"""Time ops.resample against torchaudio.functional.resample on the same CUDA tensors (CUDA events after warm-up).

For each rate pair, batch (1, 8, 32) and clip length (10 s, 30 s of the input rate) it prints the time per call, the
bytes/s achieved against the HBM floor rows (L + count) 4 bytes (read the input once, write the output once) and the
ratio torchaudio / ops.resample.  The card's name and power limit are printed in the same run, since both are part of
every number.  Writes a JSON copy of the table to --out if given.

    python tools/bench_resample.py [--iters 20] [--out results.json]
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from audiolm_pytorch_b200 import ops  # noqa: E402

PAIRS = [(44100, 16000), (44100, 24000), (22050, 16000), (48000, 16000), (48000, 24000), (24000, 16000),
         (16000, 24000)]
BATCHES = (1, 8, 32)
SECONDS = (10, 30)


def _time(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_resample needs a GPU"
    from torchaudio.functional import resample as ta_resample

    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    card = smi[torch.cuda.current_device()] if smi else torch.cuda.get_device_name()
    print(f"card: {card}")
    print(f"{'orig->new':>13} {'B':>3} {'s':>3} {'ops ms':>9} {'TB/s':>6} {'torchaudio ms':>14} {'ratio':>7}")
    rows = []
    g = torch.Generator(device="cuda").manual_seed(0)
    for orig, new in PAIRS:
        for B in BATCHES:
            for s in SECONDS:
                L = orig * s
                x = torch.randn(B, L, device="cuda", generator=g)
                count = ops.resample_length(L, orig, new)
                t_ops = _time(lambda: ops.resample(x, orig, new), args.iters)
                t_ta = _time(lambda: ta_resample(x, orig, new), args.iters)
                tbs = B * (L + count) * 4 / (t_ops * 1e-3) / 1e12
                rows.append(dict(orig=orig, new=new, batch=B, seconds=s, ops_ms=t_ops, torchaudio_ms=t_ta,
                                 tb_per_s=tbs, ratio=t_ta / t_ops))
                print(f"{orig:>6}->{new:<6} {B:>3} {s:>3} {t_ops:9.3f} {tbs:6.2f} {t_ta:14.3f} {t_ta / t_ops:7.2f}",
                      flush=True)
    if args.out:
        Path(args.out).write_text(json.dumps(dict(card=card, rows=rows), indent=1))


if __name__ == "__main__":
    main()
