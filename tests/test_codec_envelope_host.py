"""Host check of the tensor-core codec plan: for a grid of SoundStream configurations, whenever `_tc_plan()` or
`_tc_plan_dec()` accepts one, every layer's launch arguments satisfy a restatement of the ALM_REQUIRE guards of the
entry points in csrc/codec_tc.cu, at the shortest input `encode_frames` / `decode_frames` route to the tensor cores
and at a long one.  A plan that sends a kernel something it refuses fails here without a GPU."""

import itertools
import math

import pytest

PADS = {"reflect": 0, "constant": 1, "replicate": 2}


# ---- restated guards (alm_codec_* in csrc/codec_tc.cu) ---------------------------------------------------------
def first_conv_ok(B, T, Cout, K, pad_mode):
    return B > 0 and T > 0 and 1 <= K <= 8 and pad_mode in PADS and T > K - 1 and Cout in (32, 64)


def ru_ok(B, C, T, d, pad_mode, P, se_ci=None):
    ok = (B > 0 and T > 0 and d >= 1 and 6 * d <= 54 and pad_mode in PADS and T > 6 * d and P >= 1 and T % P == 0
          and C in (32, 64, 128, 256))
    return ok and (se_ci is None or 1 <= se_ci <= max(32, C // 4))


def conv_tc_ok(B, Cin, Cout, Tin, K, s, pad_mode, P, fp32, up):
    if not (B > 0 and Tin > 0 and Cin % 16 == 0 and K >= s >= 1 and Tin % s == 0 and pad_mode in PADS and Tin > K):
        return False
    bn = 256 if Cout % 256 == 0 else (128 if Cout % 128 == 0 else 64)
    if Cout % bn or not (up >= 1 and Cout % up == 0 and (up == 1 or ((Cout // up) % 16 == 0 and not fp32))):
        return False
    return bool(fp32) or (P >= 1 and (Tin // s) % P == 0)


def last_conv_ok(B, T, Cin, K, pad_mode):
    return B > 0 and T > 0 and 1 <= K <= 8 and pad_mode in PADS and T > K - 1 and Cin in (32, 64)


# ---- the launches _encode_tc / _decode_tc make --------------------------------------------------------------------
def _se_ci(ru):
    from audiolm_pytorch_b200.soundstream import _se_of

    se = _se_of(ru)
    return None if se is None else se.net[0].out_channels


def encoder_launches(ss, plan, T, B=2):
    first, blocks, last = plan
    yield "first", first_conv_ok(B, T, first.conv.out_channels, first.conv.kernel_size[0], first.pad_mode)
    for rus, down, _ in blocks:
        for i, ru in enumerate(rus):
            c7 = getattr(ru.fn, "0")
            P = down.stride if i == len(rus) - 1 else 1
            yield "ru", ru_ok(B, c7.conv.in_channels, T, c7.dilation, c7.pad_mode, P, _se_ci(ru))
        yield "down", conv_tc_ok(B, down.conv.in_channels, down.conv.out_channels, T, down.conv.kernel_size[0],
                                 down.stride, down.pad_mode, 1, 0, 1)
        T //= down.stride
    yield "last", conv_tc_ok(B, last.conv.in_channels, last.conv.out_channels, T, last.conv.kernel_size[0], 1,
                             last.pad_mode, 1, 1, 1)


def decoder_launches(ss, plan, n, B=2):
    first, blocks, last = plan
    yield "first", conv_tc_ok(B, first.conv.in_channels, first.conv.out_channels, n, first.conv.kernel_size[0], 1,
                              first.pad_mode, 1, 0, 1)
    for up, rus, _ in blocks:
        s = up.upsample_factor
        yield "up", conv_tc_ok(B, up.conv.in_channels, s * up.conv.out_channels, n, 2, 1, "constant", 1, 0, s)
        n *= s
        for ru in rus:
            c7 = getattr(ru.fn, "0")
            yield "ru", ru_ok(B, c7.conv.in_channels, n, c7.dilation, c7.pad_mode, 1, _se_ci(ru))
    yield "last", last_conv_ok(B, n, last.conv.in_channels, last.conv.kernel_size[0], last.pad_mode)


def shortest_encode_frames(ss):
    """the fewest frames encode_frames sends to the tensor cores (its guard: frames >= 4, frames * strides[-1] > 54)"""
    return next(f for f in itertools.count(4) if f * ss.strides[-1] > 54)


def shortest_decode_frames(ss, plan):
    return next(n for n in itertools.count(8) if n * plan[1][0][0].upsample_factor > 54)


# ---- the configuration grid ----------------------------------------------------------------------------------------
AXES = dict(
    strides=[(2, 4, 5, 8), (3, 6), (2, 7), (3, 4, 5, 8), (1, 2), (8, 8)],
    channels=[16, 32, 48, 64],
    channel_mults=[(2, 4, 8, 16), (1, 2), (3, 4), (2, 4), (1, 1)],
    codebook_dim=[64, 192, 512, 96],
    dilations=[((1, 3, 9), (1, 3, 9)), ((1, 2, 5), (2, 4, 8)), ((4, 6, 7), (1, 1, 1)), ((10, 1, 1), (1, 3, 9))],
    pad_mode=["reflect", "constant", "replicate"],
    squeeze_excite=[False, True],
)


def _grid():
    """every value of every axis, crossed pairwise by a deterministic cycle (not the full product)"""
    names = list(AXES)
    n = max(len(v) for v in AXES.values())
    rows = []
    for shift in range(4 * n):
        for i in range(n):
            rows.append({k: AXES[k][(i + shift * j) % len(AXES[k])] for j, k in enumerate(names)})
    seen, out = set(), []
    for r in rows:
        key = repr(sorted(r.items()))
        if key not in seen and len(r["strides"]) <= len(r["channel_mults"]):
            seen.add(key)
            out.append(r)
    return out


GRID = _grid()


def _build(cfg):
    from audiolm_pytorch_b200.soundstream import SoundStream

    enc_d, dec_d = cfg["dilations"]
    mults = cfg["channel_mults"][:len(cfg["strides"])]
    return SoundStream(channels=cfg["channels"], strides=cfg["strides"], channel_mults=mults,
                       codebook_dim=cfg["codebook_dim"], codebook_size=16, rq_num_quantizers=1, use_local_attn=False,
                       enc_cycle_dilations=enc_d, dec_cycle_dilations=dec_d, pad_mode=cfg["pad_mode"],
                       squeeze_excite=cfg["squeeze_excite"])


@pytest.mark.parametrize("cfg", GRID, ids=[f"g{i}" for i in range(len(GRID))])
def test_plan_launches_satisfy_kernel_guards(cfg):
    ss = _build(cfg)
    plan = ss._tc_plan()
    if plan is not None:
        f0 = shortest_encode_frames(ss)
        for frames in (f0, f0 + 37):
            T = frames * math.prod(ss.strides)
            bad = [k for k, ok in encoder_launches(ss, plan, T) if not ok]
            assert not bad, f"encoder plan sends {bad} launches arguments their kernels refuse (T = {T})"
    plan = ss._tc_plan_dec()
    if plan is not None:
        n0 = shortest_decode_frames(ss, plan)
        for n in (n0, n0 + 37):
            bad = [k for k, ok in decoder_launches(ss, plan, n) if not ok]
            assert not bad, f"decoder plan sends {bad} launches arguments their kernels refuse (n = {n})"


def test_grid_covers_both_plan_outcomes():
    """the grid reaches the tensor-core plans and their refusals on both sides, so the check above is not vacuous"""
    enc = [_build(c)._tc_plan() is not None for c in GRID]
    dec = [_build(c)._tc_plan_dec() is not None for c in GRID]
    assert sum(enc) >= 5 and sum(dec) >= 5 and not all(enc) and not all(dec)
    for name, values in AXES.items():
        assert {repr(c[name]) for c in GRID} == {repr(v) for v in values}, name


def test_guard_restatement_refuses_known_bad_launches():
    assert not ru_ok(1, 32, 54, 9, "reflect", 1)          # T must exceed the 6 d halo
    assert not ru_ok(1, 48, 100, 1, "reflect", 1)
    assert not ru_ok(1, 32, 100, 10, "reflect", 1)
    assert not ru_ok(1, 64, 100, 1, "reflect", 1, se_ci=33)
    assert not conv_tc_ok(1, 48, 96, 100, 4, 2, "reflect", 1, 0, 1)   # Cout not a multiple of 64
    assert not conv_tc_ok(1, 24, 64, 100, 4, 2, "reflect", 1, 0, 1)   # Cin not a multiple of 16
    assert not conv_tc_ok(1, 64, 64, 2, 2, 1, "constant", 1, 0, 2)    # Tin must exceed K
    assert not conv_tc_ok(1, 64, 96, 30, 2, 1, "constant", 1, 0, 2)   # Cout / up not a multiple of 16
    assert not first_conv_ok(1, 100, 48, 7, "reflect") and not last_conv_ok(1, 100, 48, 7, "reflect")
    assert first_conv_ok(65536, 8, 32, 8, "replicate") and last_conv_ok(65536, 8, 64, 8, "constant")
