"""FairseqVQWav2Vec (the published vq-wav2vec k-means shape: eight 512-wide convs, 2 groups of 320 codewords, 10 s
clips at 24 kHz) on the sm_90a path against the same network in stock fp32 PyTorch (oracle/vq_wav2vec.py on the GPU,
TF32 off), alternated in one process.

    python tools/bench_vq_wav2vec.py [--batches 1 8 32] [--reps 7]

Weights are seeded random in the fairseq layout (the published checkpoint is not needed for timing).  Each repetition
times one call of each path with CUDA events after a warm-up; the median and [min, max] over repetitions are printed.
A separate profiled pass gives the native path's per-stage time (ops profiler: conv extractor, projection,
assignment).  FLOPs are computed from shapes below; the split-bf16 GEMMs execute 3x their algorithmic FLOPs on the
tensor cores (conv 0 runs on fp32 CUDA cores), so two rates are printed: algorithmic FLOPs / time, and executed FLOPs
/ time with its share of the 989 TFLOP/s dense-bf16 data-sheet figure.  The card's name and power limit are read in
the same run.  Needs a GPU.
"""
from __future__ import annotations

import argparse
import json
import statistics
import sys
import tempfile
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

from tools.bench_hubert import card  # noqa: E402

SR, SECONDS = 24000, 10
STAGE_CLASS = {"conv extractor": "w2v_conv_extractor", "projection": "w2v_projection",
               "assignment": "w2v_assignment"}


def stage_flops(arch, B, T, num_vars):
    """{stage: (algorithmic FLOPs, executed FLOPs)} of one forward; executed counts split-bf16 GEMMs 3x"""
    from oracle.vq_wav2vec import conv_layers

    conv0, rest, cin = 0.0, 0.0, 1
    for i, (c, k, s) in enumerate(conv_layers(arch)):
        T = (T - k) // s + 1
        f = 2.0 * B * T * c * cin * k
        conv0, rest = (conv0 + f, rest) if i == 0 else (conv0, rest + f)
        cin = c
    G = arch["vq_groups"]
    proj = 2.0 * B * T * cin * cin / G    # the block-diagonal GEMM executes G x this
    assign = 2.0 * B * T * num_vars * cin
    return {"conv extractor": (conv0 + rest, conv0 + 3 * rest), "projection": (proj, 3 * G * proj),
            "assignment": (assign, 3 * assign)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 8, 32])
    ap.add_argument("--reps", type=int, default=7)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    from audiolm_pytorch_b200 import ops
    from audiolm_pytorch_b200.vq_wav2vec import FairseqVQWav2Vec
    from oracle import vq_wav2vec as ov

    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    dev = torch.device("cuda")
    arch = ov.PUBLISHED
    st = ov.random_state(arch, seed=0, groups=arch["vq_groups"], num_vars=arch["vq_vars"],
                         combine_groups=arch["combine_groups"])
    with tempfile.TemporaryDirectory() as d:
        ov.write_checkpoint(Path(d) / "vq.pt", st, arch)
        q = FairseqVQWav2Vec(Path(d) / "vq.pt").to(dev)
    st_dev = {k: v.to(dev) for k, v in st.items()}
    e = ov.codewords(st_dev, arch["vq_groups"])

    def stock(w):
        with torch.inference_mode():
            return ov.ids(ov.project(st_dev, ov.features(st_dev, arch, w)), e)

    print(f"card: {card()}")
    rows = []
    for B in args.batches:
        wave = torch.randn(B, SR * SECONDS, generator=torch.Generator().manual_seed(B)).to(dev)
        ids_n, ids_s = q(wave, flatten=False), stock(wave)   # warm-up (and a sanity check of agreement)
        agree = (ids_n == ids_s).float().mean().item()
        times = {"native": [], "stock fp32": []}
        for _ in range(args.reps):
            for name, fn in (("native", lambda: q(wave)), ("stock fp32", lambda: stock(wave))):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                fn()
                b.record()
                torch.cuda.synchronize()
                times[name].append(a.elapsed_time(b))
        ops.profile_start()
        q(wave)
        prof = ops.profile_stop()
        flops = stage_flops(arch, B, SR * SECONDS, arch["vq_vars"])
        stages = {}
        for stage, cls in STAGE_CLASS.items():
            ms = prof[cls][0]
            alg, exe = flops[stage]
            stages[stage] = dict(ms=round(ms, 3), alg_tflops=round(alg / ms / 1e9, 1),
                                 exec_tflops=round(exe / ms / 1e9, 1), exec_share_of_989=round(exe / ms / 1e9 / 989, 3))
        res = dict(batch=B, seconds=SECONDS, ids_agree_with_stock=round(agree, 4),
                   **{f"{k}_ms": dict(median=round(statistics.median(v), 2), min=round(min(v), 2),
                                      max=round(max(v), 2)) for k, v in times.items()},
                   stages=stages)
        rows.append(res)
        print(json.dumps(res))
    print("\n| batch | native ms median [min, max] | stock fp32 ms median [min, max] | speed-up |")
    print("|---|---|---|---|")
    for r in rows:
        n, s = r["native_ms"], r["stock fp32_ms"]
        print(f"| {r['batch']} | {n['median']} [{n['min']}, {n['max']}] | {s['median']} [{s['min']}, {s['max']}] | "
              f"{s['median'] / n['median']:.2f}x |")
    print("\n| batch | stage | ms | algorithmic TFLOP/s | executed TFLOP/s (split x3) | share of 989 |")
    print("|---|---|---|---|---|---|")
    for r in rows:
        for stage, v in r["stages"].items():
            print(f"| {r['batch']} | {stage} | {v['ms']} | {v['alg_tflops']} | {v['exec_tflops']} | "
                  f"{v['exec_share_of_989']} |")


if __name__ == "__main__":
    main()
