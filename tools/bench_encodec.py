"""EncodecWrapper encode (wave -> codes) and decode (codes -> wave) on 10 s clips at batch 1, 8 and 32: this package's
kernels against the same network in stock fp32 PyTorch (oracle/encodec.py run in fp32 on the GPU: cuDNN convs, the
LSTM as torch.nn.LSTM on cuDNN, TF32 off), alternated in one process.  CUDA events; median [min, max] of REPS runs
after warm-up.  Also a per-stage split of the native path (convs + resnet blocks, LSTM, RVQ) and the share of codes
equal to stock fp32.  Seeded random weights: the published checkpoint is not needed for timing.

    python tools/bench_encodec.py [--reps 7] [--batches 1 8 32]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import tempfile
from pathlib import Path

import torch
import torch.nn.functional as F

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from audiolm_pytorch_b200 import EncodecWrapper, ops  # noqa: E402
from oracle import encodec as oe  # noqa: E402

T = 240000  # 10 s at 24 kHz


class Stock(torch.nn.Module):
    """the oracle's network in fp32 with nn.LSTM (cuDNN) for the LSTM blocks"""

    def __init__(self, st, n_q):
        super().__init__()
        self.st = {k: v.cuda() for k, v in st.items()}
        self.w = {}
        for p, kind, *_ in oe.conv_specs():
            self.w[p] = oe.fold_weight_norm(self.st[f"{p}.weight_g"], self.st[f"{p}.weight_v"]).float()
        self.lstm = {}
        for side, idx in (("encoder", oe.ENC_LSTM), ("decoder", oe.DEC_LSTM)):
            m = torch.nn.LSTM(512, 512, 2).cuda()
            m.load_state_dict({k.split(".lstm.")[1]: v for k, v in self.st.items()
                               if k.startswith(f"{side}.model.{idx}.lstm.")})
            self.lstm[side] = m
        self.cbs = oe.codebooks(self.st, n_q).float()

    def conv(self, p, x, stride=1):
        w = self.w[p]
        return F.conv1d(oe.pad1d(x, w.shape[-1] - stride, -x.shape[-1] % stride), w, self.st[f"{p}.bias"],
                        stride=stride)

    def convtr(self, p, x, s):
        y = F.conv_transpose1d(x, self.w[p], self.st[f"{p}.bias"], stride=s)
        return y[..., : y.shape[-1] - s]

    def res(self, p, x):
        h = self.conv(f"{p}.block.3.conv.conv", F.elu(self.conv(f"{p}.block.1.conv.conv", F.elu(x))))
        return self.conv(f"{p}.shortcut.conv.conv", x) + h

    def lstm_block(self, side, x):
        return self.lstm[side](x.permute(2, 0, 1))[0].permute(1, 2, 0) + x

    def encode(self, wave):
        x = self.conv("encoder.model.0.conv.conv", wave[:, None])
        for i, s in enumerate(oe.RATIOS):
            x = self.res(f"encoder.model.{oe.ENC_RES[i]}", x)
            x = self.conv(f"encoder.model.{oe.ENC_DOWN[i]}.conv.conv", F.elu(x), stride=s)
        x = self.lstm_block("encoder", x)
        e = self.conv(f"encoder.model.{oe.ENC_LAST}.conv.conv", F.elu(x)).transpose(1, 2).reshape(-1, 128)
        r, codes = e, []
        for cb in self.cbs:
            idx = ((r * r).sum(-1, keepdim=True) - 2 * r @ cb.T + (cb * cb).sum(-1)).argmin(-1)
            codes.append(idx)
            r = r - cb[idx]
        return torch.stack(codes, -1).reshape(wave.shape[0], -1, len(self.cbs))

    def decode(self, codes):
        b, n, q = codes.shape
        emb = sum(self.cbs[i][codes[..., i]] for i in range(q)).transpose(1, 2)
        x = self.lstm_block("decoder", self.conv(f"decoder.model.{oe.DEC_FIRST}.conv.conv", emb))
        for i, s in enumerate(reversed(oe.RATIOS)):
            x = self.convtr(f"decoder.model.{oe.DEC_UP[i]}.convtr.convtr", F.elu(x), s)
            x = self.res(f"decoder.model.{oe.DEC_RES[i]}", x)
        return self.conv(f"decoder.model.{oe.DEC_LAST}.conv.conv", F.elu(x))


def timed(fn, reps):
    for _ in range(2):
        fn()
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        out.append(a.elapsed_time(b))
    out.sort()
    return out[len(out) // 2], out[0], out[-1]


def fmt(t):
    return f"{t[0]:.2f} [{t[1]:.2f}, {t[2]:.2f}]"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 8, 32])
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_encodec.py measures on the GPU"
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    print(f"card: {torch.cuda.get_device_name()} | nvidia-smi: {smi[0] if smi else 'n/a'}")
    st = oe.random_state(0, noise_clips=1, noise_samples=24000)
    with tempfile.TemporaryDirectory() as d:
        p = Path(d) / "encodec.th"
        torch.save(st, p)
        w = EncodecWrapper(checkpoint_path=p).cuda()
    stock = Stock(st, w.num_quantizers)
    rows = []
    print("| batch | encode native (ms) | encode stock fp32 | decode native (ms) | decode stock fp32 | codes equal |")
    print("|---|---|---|---|---|---|")
    for B in args.batches:
        wave = 0.3 * torch.randn(B, T, device="cuda", generator=torch.Generator(device="cuda").manual_seed(B))
        with torch.no_grad():
            _, codes, _ = w(wave)
            codes_stock = stock.encode(wave)
            eq = (codes == codes_stock).float().mean().item()
            en, es, dn, ds = [], [], [], []
            for _ in range(args.reps):  # alternate the two paths
                en.append(timed(lambda: w(wave), 1)[0])
                es.append(timed(lambda: stock.encode(wave), 1)[0])
                dn.append(timed(lambda: w.decode_from_codebook_indices(codes), 1)[0])
                ds.append(timed(lambda: stock.decode(codes), 1)[0])
            med = lambda v: (sorted(v)[len(v) // 2], min(v), max(v))  # noqa: E731
            r = dict(batch=B, encode_native=med(en), encode_stock=med(es), decode_native=med(dn),
                     decode_stock=med(ds), codes_equal=eq)
            # per-stage split of the native encode
            h = w.encode_frames(wave)
            Wt = w._weights()
            x_lstm = torch.randn(B, 512, h.shape[1], device="cuda")
            r["lstm_ms"] = timed(lambda: ops.encodec_lstm(x_lstm, Wt["enc_lstm"], elu_out=True), args.reps)
            r["rvq_ms"] = timed(lambda: w.rq(h), args.reps)
            r["encoder_ms"] = timed(lambda: w.encode_frames(wave), args.reps)
        rows.append(r)
        print(f"| {B} | {fmt(r['encode_native'])} | {fmt(r['encode_stock'])} | {fmt(r['decode_native'])} | "
              f"{fmt(r['decode_stock'])} | {eq:.4f} |")
    print("| batch | encoder convs + blocks (ms) | encoder LSTM (ms) | RVQ 8 stages (ms) |")
    print("|---|---|---|---|")
    for r in rows:
        conv = r["encoder_ms"][0] - r["lstm_ms"][0]
        print(f"| {r['batch']} | {conv:.2f} | {fmt(r['lstm_ms'])} | {fmt(r['rvq_ms'])} |")
    print(json.dumps(dict(card=torch.cuda.get_device_name(), smi=smi, rows=rows)))


if __name__ == "__main__":
    main()
