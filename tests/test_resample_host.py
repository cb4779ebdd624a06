"""Resampling without a GPU: the fp64 oracle (oracle/resample.py) against torchaudio.functional.resample, the compact
polyphase table (ops.resample_table) against torchaudio's dense fp64 filter, the output-length and window arithmetic
of the callers, and rate validation."""
import math

import pytest
import torch

from audiolm_pytorch_b200 import ops
from audiolm_pytorch_b200.soundstream import curtail_window
from oracle import resample as orr

PAIRS = [(44100, 16000), (44100, 24000), (22050, 16000), (48000, 16000), (48000, 24000), (24000, 16000),
         (16000, 24000), (96000, 8000), (8000, 96000)]
# reduced rates coprime and large; torchaudio's dense filter for 44100 -> 16001 (16001 x 44134 taps in fp64) is too big
# for a unit test, so the oracle comparison uses 4410 -> 1601 and the table test covers 44100 -> 16001 by blocks
COPRIME = (4410, 1601)


def _lengths(orig, new):
    o, n = ops.resample_rates(orig, new)
    return sorted({L for L in (1, o - 1, o, o + 1, orig + 17) if L >= 1})


@pytest.mark.parametrize("orig, new", PAIRS + [COPRIME])
def test_oracle_matches_torchaudio(orig, new):
    from torchaudio.functional import resample

    g = torch.Generator().manual_seed(orig + new)
    for L in _lengths(orig, new):
        x = torch.randn(2, L, generator=g, dtype=torch.float64)
        ref = resample(x, orig, new)
        got = orr.resample(x, orig, new)
        assert got.shape == ref.shape == (2, ops.resample_length(L, orig, new))
        assert (got - ref).abs().max() <= 1e-12 * x.abs().max()


@pytest.mark.parametrize("orig, new", PAIRS + [COPRIME])
def test_oracle_filter_is_torchaudios(orig, new):
    from torchaudio.functional.functional import _get_sinc_resample_kernel

    dense, width = _get_sinc_resample_kernel(orig, new, math.gcd(orig, new), dtype=torch.float64)
    assert width == orr.rates(orig, new)[3]
    assert torch.equal(orr.dense_kernel(orig, new), dense[:, 0])


def _check_table(orig, new, dense_of):
    o, n, _, width = orr.rates(orig, new)
    taps, first, counts = ops.resample_table(o, n)
    assert taps.shape == (n, int(counts.max())) and first.shape == counts.shape == (n,)
    for p0 in range(0, n, 512):
        ph = torch.arange(p0, min(n, p0 + 512))
        dense = dense_of(ph).clone()
        for r, p in enumerate(ph.tolist()):
            m0, c = int(first[p]) + width, int(counts[p])
            assert m0 >= 0 and m0 + c <= dense.shape[1]
            kept = dense[r, m0:m0 + c]
            assert (taps[p, :c] - kept).abs().max() <= 1e-15 * kept.abs().max()
            assert not taps[p, c:].any()
            dense[r, m0:m0 + c] = 0
        assert dense.abs().max() <= 1e-40


@pytest.mark.parametrize("orig, new", PAIRS + [COPRIME])
def test_table_is_torchaudios_filter(orig, new):
    from torchaudio.functional.functional import _get_sinc_resample_kernel

    dense = _get_sinc_resample_kernel(orig, new, math.gcd(orig, new), dtype=torch.float64)[0][:, 0]
    _check_table(orig, new, lambda ph: dense[ph])


def test_table_coprime_large():
    """44100 -> 16001: a 16001 x 34 table; the dense filter (the oracle's, equal to torchaudio's above) by blocks"""
    _check_table(44100, 16001, lambda ph: orr.dense_kernel(44100, 16001, ph))
    taps, _, _ = ops.resample_table(44100, 16001)
    assert taps.numel() > 48 * 1024  # larger than a block's default shared memory: the kernel reads it from L2


@pytest.mark.parametrize("orig, new, taps", [(44100, 16000, 34), (22050, 16000, 17), (44100, 24000, 23),
                                             (48000, 16000, 37), (24000, 16000, 19), (16000, 24000, 13)])
def test_kept_taps(orig, new, taps):
    assert ops.resample_table(*ops.resample_rates(orig, new))[0].shape[1] == taps


@pytest.mark.parametrize("orig, new", PAIRS + [COPRIME, (44100, 16001), (3, 2)])
def test_output_length(orig, new):
    o, n = ops.resample_rates(orig, new)
    for L in list(range(1, 40)) + _lengths(orig, new):
        assert ops.resample_length(L, orig, new) == math.ceil(n * L / o) == -(-new * L // orig)


def test_curtail_windows_match_slicing():
    """SoundStream (both directions) and HuBERT / vq-wav2vec curtailing, as windows into the resampled output"""
    from audiolm_pytorch_b200.hubert import curtail_to_multiple

    for total in range(0, 700):
        t = torch.arange(total)
        for mult in (1, 7, 320):
            keep = total // mult * mult
            for from_left, ref in ((False, t[..., :keep]), (True, t[..., -keep:])):
                s, c = curtail_window(total, mult, from_left)
                assert torch.equal(t[s:s + c], ref)
            assert torch.equal(curtail_to_multiple(t, mult), t[:keep])


@pytest.mark.parametrize("orig, new", [(0, 16000), (16000, 0), (-8000, 16000), (44100.5, 16000), (16000, 22050.25),
                                       (float("nan"), 16000)])
def test_bad_rates(orig, new):
    x = torch.randn(1, 100)
    with pytest.raises(ValueError):
        ops.resample(x, orig, new)
    with pytest.raises(ValueError):
        ops.resample_length(100, orig, new)


def test_same_rate_returns_input():
    x = torch.randn(2, 3, 101, dtype=torch.float64)
    assert ops.resample(x, 16000, 16000) is x
    assert ops.resample(x, 16000.0, 16000) is x
    assert torch.equal(ops.resample(x, 24000, 24000, count=100), x[..., :100])


def test_cpu_tensor_raises():
    from audiolm_pytorch_b200._lib import AlmError

    with pytest.raises(AlmError):
        ops.resample(torch.randn(1, 100), 44100, 16000)


def test_window_bounds():
    x = torch.randn(1, 441)
    for start, count in ((-1, None), (0, 161), (161, None), (100, 61)):
        with pytest.raises(ValueError):
            ops.resample(x, 44100, 16000, start=start, count=count)
