"""fp64 restatement of torchaudio.functional.resample(x, orig, new) with its defaults (sinc_interp_hann,
lowpass_filter_width = 6, rolloff = 0.99), the call at soundstream.py:788, hubert_kmeans.py:102, vq_wav2vec.py:70 and
encodec.py:105 of the reference.  It builds torchaudio's dense filter with the same fp64 operations and applies it as
the polyphase sum

    y[k n + p] = sum_{m < 2 width + o} K[p, m] x[k o + m - width]     (x = 0 outside [0, L)),  len(y) = ceil(n L / o)

with o -> n the rates reduced by their gcd.  The filter is built a block of phases at a time, so coprime rates whose
dense filter would not fit in memory at once (44100 -> 16001 has 16001 x 44134 taps) still run.  Works on any device.
"""
from __future__ import annotations

import math

import torch

ZEROS = 6
ROLLOFF = 0.99
f64 = torch.float64


def rates(orig, new):
    """(o, n, base, width) of the reduced rates"""
    if orig <= 0 or new <= 0 or int(orig) != orig or int(new) != new:
        raise ValueError(f"sample rates must be positive integers, got {orig} -> {new}")
    g = math.gcd(int(orig), int(new))
    o, n = int(orig) // g, int(new) // g
    base = min(o, n) * ROLLOFF
    return o, n, base, math.ceil(ZEROS * o / base)


def dense_kernel(orig, new, phases=None, device="cpu"):
    """torchaudio's dense fp64 filter K [len(phases), 2 width + o] (all n phases by default), op for op as
    torchaudio's _get_sinc_resample_kernel builds it"""
    o, n, base, width = rates(orig, new)
    idx = torch.arange(-width, width + o, dtype=f64, device=device)[None] / o
    a = torch.arange(0, -n, -1, dtype=f64, device=device)
    if phases is not None:
        a = a[phases]
    t = a[:, None] / n + idx
    t *= base
    t = t.clamp_(-ZEROS, ZEROS)
    window = torch.cos(t * math.pi / ZEROS / 2) ** 2
    t *= math.pi
    scale = base / o
    kernels = torch.where(t == 0, torch.tensor(1.0).to(t), t.sin() / t)
    kernels *= window * scale
    return kernels


def resample(x, orig, new, *, with_magnitude=False, block_taps=1 << 22):
    """x [..., L] -> fp64 [..., ceil(n L / o)] (and, if with_magnitude, sum_m |K[p, m] x[k o + m - width]| of every
    output: the scale of its rounding error).  orig == new returns x as fp64."""
    o, n, base, width = rates(orig, new)
    x = x.to(f64)
    if o == n:
        return (x, x.abs()) if with_magnitude else x
    lead, L = x.shape[:-1], x.shape[-1]
    total = -(-n * L // o)
    xs = x.reshape(-1, L)
    frames = L // o + 1
    xp = torch.nn.functional.pad(xs, (width, width + o))
    win = xp.unfold(1, 2 * width + o, o)[:, :frames]           # [rows, frames, 2 width + o]
    y = torch.empty(xs.shape[0], frames, n, dtype=f64, device=x.device)
    mag = torch.empty_like(y) if with_magnitude else None
    step = max(1, block_taps // (2 * width + o))
    for p0 in range(0, n, step):
        ph = torch.arange(p0, min(n, p0 + step), device=x.device)
        K = dense_kernel(orig, new, ph, device=x.device)
        y[:, :, p0:p0 + len(ph)] = torch.einsum("rfm,pm->rfp", win, K)
        if with_magnitude:
            mag[:, :, p0:p0 + len(ph)] = torch.einsum("rfm,pm->rfp", win.abs(), K.abs())
    y = y.reshape(xs.shape[0], -1)[:, :total].reshape(*lead, total)
    if with_magnitude:
        return y, mag.reshape(xs.shape[0], -1)[:, :total].reshape(*lead, total)
    return y
