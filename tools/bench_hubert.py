"""HubertWithKmeans (HuBERT-base shapes, output_layer 9, 500 clusters, 10 s clips at 16 kHz) on the sm_90a path against
the same network in stock fp32 PyTorch (oracle/hubert.py on the GPU, TF32 off), alternated in one process.

    python tools/bench_hubert.py [--batches 1 8 32] [--reps 7]

Weights are seeded random in the fairseq layout (the published checkpoint is not needed for timing).  Each repetition
times one call of each path with CUDA events after a warm-up; the median and [min, max] over repetitions are printed.
A separate profiled pass gives the native path's per-stage kernel time (ops profiler: conv extractor, positional conv,
encoder layers, assignment).  FLOPs are computed from shapes below; the split-bf16 GEMMs execute 3x their algorithmic
FLOPs on the tensor cores, so two rates are printed: algorithmic FLOPs / time, and executed FLOPs / time with its share
of the 989 TFLOP/s dense-bf16 data-sheet figure.  The card's name and power limit are read in the same run.  Needs a GPU.
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
import tempfile
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

PEAK_BF16 = 989e12
SR, SECONDS, LAYER, CLUSTERS = 16000, 10, 9, 500


def card():
    name = torch.cuda.get_device_name()
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        q = "power limit unknown"
    return f"{name} ({q})"


def stage_flops(arch, B, T):
    """{stage: (algorithmic FLOPs, executed FLOPs)} of one forward; executed counts split-bf16 GEMMs 3x"""
    from oracle.hubert import parse_conv_layers

    conv0, conv_rest, cin = 0.0, 0.0, 1
    for i, (c, k, s) in enumerate(parse_conv_layers(arch["conv_feature_layers"])):
        T = (T - k) // s + 1
        f = 2.0 * B * T * c * cin * k
        conv0, conv_rest = (conv0 + f, conv_rest) if i == 0 else (conv0, conv_rest + f)
        cin = c
    D, Fi, G, K = arch["encoder_embed_dim"], arch["encoder_ffn_embed_dim"], arch["conv_pos_groups"], arch["conv_pos"]
    proj = 2.0 * B * T * cin * D
    pos = 2.0 * B * T * D * (D // G) * K
    gemm = LAYER * 2.0 * B * T * D * (4 * D + 2 * Fi)
    attn = LAYER * 4.0 * B * T * T * D
    assign = 2.0 * B * T * CLUSTERS * D
    return {"conv extractor": (conv0 + conv_rest + proj, conv0 + 3 * (conv_rest + proj)),
            "positional conv": (pos, 3 * pos),
            "encoder layers": (gemm + attn, 3 * gemm + attn),
            "assignment": (assign, 3 * assign)}


STAGE_CLASS = {"conv extractor": "hubert_conv_extractor", "positional conv": "hubert_pos_conv",
               "encoder layers": "hubert_layers", "assignment": "hubert_assignment"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 8, 32])
    ap.add_argument("--reps", type=int, default=7)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    from audiolm_pytorch_b200 import ops
    from audiolm_pytorch_b200.hubert import HubertWithKmeans
    from oracle import hubert as oh

    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    dev = torch.device("cuda")
    arch = oh.BASE
    st = oh.random_state(arch, seed=0)
    centers = torch.randn(CLUSTERS, arch["encoder_embed_dim"], generator=torch.Generator().manual_seed(1))
    with tempfile.TemporaryDirectory() as d:
        oh.write_checkpoint(Path(d) / "ck.pt", st, arch)
        oh.write_kmeans(Path(d) / "km.bin", centers)
        h = HubertWithKmeans(Path(d) / "ck.pt", Path(d) / "km.bin", output_layer=LAYER).to(dev)
    st_dev = {k: v.to(dev) for k, v in st.items()}
    c_dev = centers.to(dev)

    def stock(w):
        with torch.inference_mode():
            return oh.assign(oh.extract_features(st_dev, arch, w, LAYER), c_dev)

    print(f"card: {card()}")
    rows = []
    for B in args.batches:
        wave = torch.randn(B, SR * SECONDS, generator=torch.Generator().manual_seed(B)).to(dev)
        ids_n, ids_s = h(wave), stock(wave)   # warm-up (and a sanity check of agreement)
        agree = (ids_n == ids_s).float().mean().item()
        times = {"native": [], "stock fp32": []}
        for _ in range(args.reps):
            for name, fn in (("native", lambda: h(wave)), ("stock fp32", lambda: stock(wave))):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                fn()
                b.record()
                torch.cuda.synchronize()
                times[name].append(a.elapsed_time(b))
        ops.profile_start()
        h(wave)
        prof = ops.profile_stop()
        flops = stage_flops(arch, B, SR * SECONDS)
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
    print("\n| batch | stage | kernel ms | algorithmic TFLOP/s | executed TFLOP/s (split x3) | share of 989 |")
    print("|---|---|---|---|---|---|")
    for r in rows:
        for stage, v in r["stages"].items():
            print(f"| {r['batch']} | {stage} | {v['ms']} | {v['alg_tflops']} | {v['exec_tflops']} | "
                  f"{v['exec_share_of_989']} |")


if __name__ == "__main__":
    main()
