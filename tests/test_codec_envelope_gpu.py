"""H100: every kernel of the SoundStream tensor-core codec (csrc/codec_tc.cu) against an fp64 restatement
(oracle/codec.py, oracle/codec_se.py) across the shapes, modes and edges its C entry points accept, each output element
held to a bound derived from the split-bf16 error model; then SoundStream.encode_frames / decode_frames on small
configurations, on both sides of the plan's guards, with the path that ran asserted."""

import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"
f64 = torch.float64
bf16 = torch.bfloat16
MODES = ("reflect", "constant", "replicate")
WRONG_MODE = {"reflect": "replicate", "replicate": "constant", "constant": "reflect"}

# Error model of one conv  y = b + sum W x  (per output element, S = b + sum |W| |x|, the same conv on magnitudes):
# - split-bf16 products (alm_codec_ru_tc / _ru_se_tc / _conv_tc): a C8S input is exactly x_hi + x_lo; W is carried as
#   w_hi + w_lo to 2^-16 relative and the x_lo w_lo product is dropped (2^-16): EPS_SPLIT = 2^-15 of S covers both;
# - fp32 accumulation: 2^-24 of S per product that is not zero (EPS_ACC), K Cin for a dense weight row;
# - an fp32 activation the kernel re-splits into hi + lo for the next GEMM (E1, E2, E3): EPS_A = 2^-16 relative;
# - the output: hi + lo carries y to 2^-16 relative (EPS_C8S); an fp32 output is one rounding (EPS_F32 = 2^-23);
# - ELU(v) = __expf(v) - 1 below zero: 2^-21 absolute (ELU is 1-Lipschitz, so input errors pass through);
# - SiLU(v) = v / (1 + __expf(-v)) and sigmoid: (3 + 1.16 |v|) 2^-23 relative (__expf is good to 2 + 1.16 |v| ulp),
#   as in test_codec_gate_loop_gpu.py; the derivatives (<= 1.1 and gate (1 - gate)) carry the input errors.
# The CUDA-core first and last convs (alm_codec_first_conv / _last_conv) are plain fp32 FMAs: EPS_ACC per product.
# Each case also evaluates, in fp64, two plausible wrong kernels and requires each to break the bound by >= 10x:
#   x and W rounded to plain bf16 (the lo halves dropped), and the halo filled with another pad mode.
# For a wide conv, a bf16 kernel's rounding errors of random sign grow as sqrt(K Cin) while the bound grows as K Cin,
# so every conv case carries a "coherent window": output channel 0 reads 16 input channels only, and in one time
# window those inputs and weights are positive with their lo half +1.5 2^-10 of the hi half.  There the dropped lo
# halves add up to ~2^-9 of S while the bound stays ~2^-14: the same data then also tells a right kernel from one
# that loses the lo halves.
EPS_SPLIT = 2.0 ** -15
EPS_ACC = 2.0 ** -24
EPS_A = 2.0 ** -16
EPS_C8S = 2.0 ** -16
EPS_F32 = 2.0 ** -23
EPS_ELU = 2.0 ** -21


def _ops():
    from audiolm_pytorch_b200 import ops

    return ops


def _oc():
    from oracle import codec as oc

    return oc


def bf(t):
    return t.to(bf16).to(t.dtype)


def c8s_value(x, phases=1):
    """the C8S tensor a kernel reads for fp32 x [B, C, T], and its exact value in fp64"""
    ops = _ops()
    xc = ops.c8s_pack(x, phases)
    return xc, ops.c8s_unpack(xc).to(f64)


def nnz_rows(w):
    """[1, Cout, 1]: products per output element that are not zero (w [Cout, Cin, K])"""
    return (w != 0).flatten(1).sum(1).to(f64)[None, :, None]


def conv64(x, w, b, **kw):
    return _oc().causal_conv1d(x, w, b, **kw)


def conv_bound(x, w, b, *, split, eps_out, **kw):
    """fp64 reference and per-element bound of one conv (x, w, b fp64)"""
    y = conv64(x, w, b, **kw)
    S = conv64(x.abs(), w.abs(), b.abs(), **kw)
    return y, ((EPS_SPLIT if split else 0.0) + nnz_rows(w) * EPS_ACC) * S + eps_out * y.abs()


def check(label, got, y, bound, wrong):
    """err / bound <= 1 everywhere; every wrong-kernel emulation exceeds the bound by >= 10x somewhere"""
    got = got.to(f64)
    assert got.shape == y.shape, (got.shape, y.shape)
    assert torch.isfinite(got).all(), f"{label}: non-finite output"
    ratio = ((got - y).abs() / bound).max().item()
    teeth = {k: ((v - y).abs() / bound).max().item() for k, v in wrong.items() if v is not None}
    print(f"{label}: max err/bound {ratio:.3f}; wrong kernels " + ", ".join(f"{k} {v:.0f}x" for k, v in teeth.items()))
    assert ratio <= 1.0, f"{label}: error {ratio:.2f}x the split-bf16 error model"
    for k, v in teeth.items():
        assert v >= 10.0, f"{label}: the bound cannot tell the {k} kernel apart ({v:.1f}x)"
    return ratio


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _biased(t):
    """positive values whose lo half is +1.5 2^-10 of the hi half (below half a bf16 ulp: bf16(v) = hi)"""
    return bf(t.abs().clamp_min(1e-30)) * (1 + 1.5 * 2.0 ** -10)


def plant_window(x, w, t0, t1):
    """coherent window: output channel 0 reads input channels 0..15 only, positive and lo-biased; so are those inputs on
    [t0, t1).  x [B, Cin, T], w [Cout, Cin, K]"""
    x[:, :16, t0:t1] = _biased(x[:, :16, t0:t1])
    w0 = _biased(w[0, :16].abs() + 0.5 * w.abs().mean())
    w[0] = 0
    w[0, :16] = w0
    return x, w


# ---- alm_codec_first_conv -------------------------------------------------------------------------------------
FIRST_CASES = [(32 if K % 2 else 64, K, T, 1 if (K + i) % 2 else 3, MODES[(K + i) % 3])
               for K in range(1, 9) for i, T in enumerate((K, 127, 128, 129, 20000))]


def _first_conv_case(cout, K, T, B, mode, scale, seed):
    ops = _ops()
    g = _gen(seed)
    w = torch.randn(cout, 1, K, generator=g, device=DEV) * 0.4
    b = torch.randn(cout, generator=g, device=DEV) * 0.1 * scale
    x = torch.randn(B, T, generator=g, device=DEV) * scale
    got = ops.c8s_unpack(ops.codec_first_conv(x, w, b, pad_mode=mode))
    x64, w64, b64 = x[:, None].to(f64), w.to(f64), b.to(f64)
    y, bound = conv_bound(x64, w64, b64, split=False, eps_out=EPS_C8S, pad_mode=mode)
    wrong = {"plain-bf16": bf(conv64(bf(x64), bf(w64), b64, pad_mode=mode)),
             "pad-mode": conv64(x64, w64, b64, pad_mode=WRONG_MODE[mode]) if K > 1 else None}
    return got, y, bound, wrong


@pytest.mark.parametrize("cout,K,T,B,mode", FIRST_CASES)
def test_first_conv(cout, K, T, B, mode):
    got, y, bound, wrong = _first_conv_case(cout, K, T, B, mode, 1.0, K * 1000 + T)
    check(f"first_conv Cout={cout} K={K} T={T} B={B} {mode}", got, y, bound, wrong)


# ---- alm_codec_pack_c8s and the torch c8s_pack / c8s_unpack ------------------------------------------------------
@pytest.mark.parametrize("C", [8, 24, 512])
@pytest.mark.parametrize("n", [1, 37, 5000])
def test_pack_c8s_round_trip(C, n):
    ops = _ops()
    x = torch.randn(2, n, C, generator=_gen(C + n), device=DEV) * torch.logspace(-3, 3, C, device=DEV)
    packed = ops.codec_pack_c8s(x)
    assert packed.shape == (2, 2 * C // 8, 1, n, 8)
    # both round to nearest: the kernel's split is the torch split, bit for bit
    assert torch.equal(packed, ops.c8s_pack(x.transpose(1, 2).contiguous()))
    back = ops.c8s_unpack(packed).to(f64)
    ref = x.transpose(1, 2).to(f64)
    assert ((back - ref).abs() <= 2.0 ** -17 * ref.abs()).all()
    assert ((bf(ref) - ref).abs() > 2.0 ** -17 * ref.abs()).any()   # a lost lo half would fail the bound
    for P in (2, 5):   # the phase-split layout holds the same values
        if n % P == 0:
            assert torch.equal(ops.c8s_unpack(ops.c8s_pack(ref.float(), P)).to(f64), back)


# ---- alm_codec_ru_tc / alm_codec_ru_se_tc -----------------------------------------------------------------------
def _ru_state(C, seed, se_ci=None, gate_bias=0.0, scale=1.0):
    """unit weights; channel 0 is quiet (its 1x1-conv row and bias are zero, so the unit passes x through there): the
    bound on that channel is the output split alone, which a kernel that drops the lo half of x breaks"""
    g = _gen(seed)
    st = {"fn.0.conv.weight": torch.randn(C, C, 7, generator=g, device=DEV) * (0.7 / (7 * C) ** 0.5),
          "fn.0.conv.bias": torch.randn(C, generator=g, device=DEV) * 0.1 * scale,
          "fn.2.conv.weight": torch.randn(C, C, 1, generator=g, device=DEV) * (0.7 / C ** 0.5),
          "fn.2.conv.bias": torch.randn(C, generator=g, device=DEV) * 0.1 * scale}
    st["fn.2.conv.weight"][0] = 0
    st["fn.2.conv.bias"][0] = 0
    if se_ci is not None:
        st["fn.4.net.0.weight"] = torch.randn(se_ci, C, 1, generator=g, device=DEV) * (1.0 / C ** 0.5)
        st["fn.4.net.0.bias"] = torch.randn(se_ci, generator=g, device=DEV) * 0.1
        st["fn.4.net.2.weight"] = torch.randn(C, se_ci, 1, generator=g, device=DEV) * (1.0 / se_ci ** 0.5)
        st["fn.4.net.2.bias"] = torch.randn(C, generator=g, device=DEV) * 0.1 + gate_bias
    return st


def _elu(v, ev):
    """ELU and its error bound; __expf only runs where the kernel's input can be negative"""
    a = F.elu(v)
    return a, ev + EPS_ELU * (v < ev) * (1 + a.abs())


def ru_reference(st, x, d, mode):
    """fp64 reference (oracle/codec_se.residual_unit) and the per-element bound of the fused unit, SE or not"""
    from oracle import codec_se as ose

    y = ose.residual_unit(st, x, d, mode)
    w7, b7, w1, b1 = (st[k] for k in ("fn.0.conv.weight", "fn.0.conv.bias", "fn.2.conv.weight", "fn.2.conv.bias"))
    h1, e1 = conv_bound(x, w7, b7, split=True, eps_out=0.0, dilation=d, pad_mode=mode)
    a1, ea1 = _elu(h1, e1)
    ea1 = ea1 + EPS_A * a1.abs()                                         # E1: split into the A operand of the 1x1 conv
    h2, e2 = conv_bound(a1, w1, b1, split=True, eps_out=0.0)
    a2, ea2 = _elu(h2, e2 + torch.einsum("oc,bct->bot", w1[..., 0].abs(), ea1))
    if "fn.4.net.0.weight" not in st:
        return y, ea2 + (EPS_C8S + EPS_F32) * y.abs()
    C = w7.shape[0]
    ea2 = ea2 + EPS_A * a2.abs()                                         # E2: y split for D3 and re-read by E4
    w_s1 = st["fn.4.net.0.weight"][..., 0]
    w_fold = (w_s1 / torch.arange(1, C + 1, device=x.device, dtype=f64)).flip(-1).cumsum(-1).flip(-1)
    z = torch.einsum("ic,bct->bit", w_fold, a2) + st["fn.4.net.0.bias"][:, None]
    Sz = torch.einsum("ic,bct->bit", w_fold.abs(), a2.abs()) + st["fn.4.net.0.bias"].abs()[:, None]
    ez = (EPS_SPLIT + C * EPS_ACC) * Sz + torch.einsum("ic,bct->bit", w_fold.abs(), ea2)
    s, sig = F.silu(z), torch.sigmoid(z)
    # E3: SiLU (its __expf error enters through sigmoid'), then the split into register A fragments
    es = 1.1 * ez + z.abs() * sig * (1 - sig) * (3 + 1.16 * z.abs()) * EPS_F32 + (2 * EPS_F32 + EPS_A) * s.abs()
    w_s2, b_s2 = st["fn.4.net.2.weight"][..., 0], st["fn.4.net.2.bias"][:, None]
    gpre = torch.einsum("ci,bit->bct", w_s2, s) + b_s2
    Sg = torch.einsum("ci,bit->bct", w_s2.abs(), s.abs()) + b_s2.abs()
    eg = (EPS_SPLIT + max(32, C // 4) * EPS_ACC) * Sg + torch.einsum("ci,bit->bct", w_s2.abs(), es)
    gate = torch.sigmoid(gpre)
    egate = gate * (1 - gate) * (eg + (3 + 1.16 * gpre.abs()) * EPS_F32) + 2 * EPS_F32 * gate
    return y, gate * ea2 + a2.abs() * egate + (EPS_C8S + 2 * EPS_F32) * y.abs()


def _ru_run(st, x, d, mode, P):
    """run the fused unit on fp32 x [B, C, T]; returns (kernel output, reference, bound, wrong kernels)"""
    from oracle import codec_se as ose

    ops = _ops()
    xc, x64 = c8s_value(x)
    if "fn.4.net.0.weight" in st:
        wu = ops.pack_ru_se_weights(st["fn.0.conv.weight"], st["fn.2.conv.weight"], st["fn.4.net.0.weight"],
                                    st["fn.4.net.2.weight"])
        y = ops.codec_ru_se_tc(xc, wu, st["fn.0.conv.bias"], st["fn.2.conv.bias"], st["fn.4.net.0.bias"],
                               st["fn.4.net.2.bias"], dilation=d, pad_mode=mode, out_phases=P)
    else:
        wu = ops.pack_ru_weights(st["fn.0.conv.weight"], st["fn.2.conv.weight"])
        y = ops.codec_ru_tc(xc, wu, st["fn.0.conv.bias"], st["fn.2.conv.bias"], dilation=d, pad_mode=mode,
                            out_phases=P)
    B, C, T = x.shape
    assert y.shape == (B, C // 4, P, T // P, 8)
    st64 = {k: v.to(f64) for k, v in st.items()}
    ref, bound = ru_reference(st64, x64, d, mode)
    st_bf = {k: bf(v) if "weight" in k else v for k, v in st64.items()}
    wrong = {"plain-bf16": ose.residual_unit(st_bf, bf(x64), d, mode),
             "pad-mode": ose.residual_unit(st64, x64, d, WRONG_MODE[mode])}
    return ops.c8s_unpack(y), ref, bound, wrong


def _ru_cases():
    cases = []
    for ci, C in enumerate((32, 64, 128, 256)):
        for d in range(1, 10):
            Ts = [T for T in (6 * d + 1, 63, 64, 65, 127, 129, 5040) if T > 6 * d]
            T = Ts[(d + ci) % len(Ts)]
            Ps = [P for P in range(1, 9) if T % P == 0]
            P = Ps[(d + 2 * ci) % len(Ps)]
            cases.append((C, d, T, P, 2, MODES[(d + ci) % 3]))
        cases += [(C, 1 + (2 * P + ci) % 9, 5040, P, 1, MODES[(P + ci) % 3]) for P in range(1, 9)]
    cases += [(32, d, 6 * d + 1, 1, 3, MODES[d % 3]) for d in range(1, 10)]        # the shortest clip at every dilation
    cases += [(256, 9, 55, 5, 2, "replicate"), (128, 9, 55, 1, 1, "reflect")]
    return sorted(set(cases))


@pytest.mark.parametrize("C,d,T,P,B,mode", _ru_cases())
def test_ru_tc(C, d, T, P, B, mode):
    st = _ru_state(C, 10 * C + d)
    x = torch.randn(B, C, T, generator=_gen(T + d), device=DEV)
    check(f"ru_tc C={C} d={d} T={T} P={P} B={B} {mode}", *_ru_run(st, x, d, mode, P))


def _grid(C):
    """CTAs of launch_ru: RuCfg<C, SE>::CTAS_PER_SM per SM (two for the resident C = 32 unit, one otherwise)"""
    return _ops().num_sms() * (2 if C == 32 else 1)


TILE_COUNTS = ("1", "odd", "grid-1", "grid+1", "3grid")


def _tiles(label, grid):
    return {"1": 1, "odd": 7, "grid-1": grid - 1, "grid+1": grid + 1, "3grid": 3 * grid}[label]


@pytest.mark.parametrize("C", [32, 64, 128])
@pytest.mark.parametrize("tiles", TILE_COUNTS)
def test_ru_tc_tile_counts(C, tiles):
    """one 64-step tile per clip, B clips: the even/odd split of the two producers of the resident-weight units
    (C <= 64) with an odd tile count, fewer tiles than CTAs, and several tiles per CTA"""
    if C == 128 and tiles in ("odd", "grid-1"):
        pytest.skip("one producer: the tile count only matters around the grid size")
    B = _tiles(tiles, _grid(C))
    st = _ru_state(C, 500 + C)
    x = torch.randn(B, C, 64, generator=_gen(B), device=DEV)
    check(f"ru_tc tiles C={C} B={B} ({tiles})", *_ru_run(st, x, 3, MODES[B % 3], 2))


SE_CASES = ([(C, ci, d, T, P, MODES[i % 3], gb)
             for i, (C, ci, d, T, P, gb) in enumerate([
                 (32, 1, 1, 7, 1, 0.0), (32, 8, 9, 129, 3, 0.0), (32, 32, 4, 5040, 8, -12.0),
                 (64, 1, 2, 65, 5, 12.0), (64, 16, 7, 127, 1, 0.0), (64, 32, 3, 5040, 6, 0.0),
                 (128, 1, 5, 31, 1, 0.0), (128, 32, 9, 5040, 4, 12.0), (128, 32, 6, 64, 2, -12.0),
                 (256, 64, 8, 129, 3, 0.0), (256, 1, 1, 5040, 7, -12.0), (256, 64, 9, 55, 5, 12.0)])])


@pytest.mark.parametrize("C,se_ci,d,T,P,mode,gate_bias", SE_CASES)
def test_ru_se_tc(C, se_ci, d, T, P, mode, gate_bias):
    """se_ci at 1, C / 4 and the padded inner width NS = max(32, C / 4); gate_bias +-12 drives the gates into
    saturation near 1 and 0"""
    st = _ru_state(C, 30 * C + d, se_ci=se_ci, gate_bias=gate_bias)
    x = torch.randn(2, C, T, generator=_gen(T + C), device=DEV)
    check(f"ru_se_tc C={C} ci={se_ci} d={d} T={T} P={P} {mode} gate_bias={gate_bias}", *_ru_run(st, x, d, mode, P))


# ---- alm_codec_conv_tc ------------------------------------------------------------------------------------------
def _conv_cases():
    cins, couts = (16, 48, 256, 512), (64, 192, 128, 256, 512)
    cases, i = [], 0
    for s in range(1, 9):
        for K in sorted({s, 2 * s, 16} | ({3, 7} if s == 1 else set())):
            for long_ in (False, True):
                cin, cout = cins[i % 4], couts[i % 5]
                Tin = s * 1000 if long_ else (K // s + 1) * s      # minimal: the least multiple of s above K
                n_out = Tin // s
                P = [p for p in (4, 3, 2, 5, 1) if n_out % p == 0][0] if long_ and i % 2 else 1
                fp32 = P == 1 and i % 3 == 0
                cases.append((cin, cout, K, s, Tin, P, fp32, MODES[i % 3]))
                i += 1
    cases += [(256, 512, 16, 8, 8 * 150, 1, True, "replicate"), (512, 512, 3, 1, 150, 1, True, "reflect"),
              (48, 192, 8, 4, 4 * 517, 1, False, "replicate")]
    return cases


def _conv_run(cin, cout, K, s, Tin, P, fp32, mode, B=2, scale=1.0, seed=0):
    ops = _ops()
    g = _gen(seed + cin + cout + K + s + Tin)
    w = torch.randn(cout, cin, K, generator=g, device=DEV) * (0.7 / (cin * K) ** 0.5)
    b = torch.randn(cout, generator=g, device=DEV) * 0.1 * scale
    x = torch.randn(B, cin, Tin, generator=g, device=DEV) * scale
    t1 = min(Tin, 3 * s * 128 + 40)
    x, w = plant_window(x, w, max(0, t1 - 200), t1)
    xc, x64 = c8s_value(x, s)
    wu = ops.pack_conv_weights(w)
    y = ops.codec_conv_tc(xc, wu, b, cout=cout, kernel_size=K, stride=s, pad_mode=mode, out_phases=P, out_fp32=fp32)
    got = y.transpose(1, 2) if fp32 else ops.c8s_unpack(y)
    w64, b64 = w.to(f64), b.to(f64)
    ref, bound = conv_bound(x64, w64, b64, split=True, eps_out=EPS_F32 if fp32 else EPS_C8S, stride=s, pad_mode=mode)
    wrong = {"plain-bf16": conv64(bf(x64), bf(w64), b64, stride=s, pad_mode=mode),
             "pad-mode": conv64(x64, w64, b64, stride=s, pad_mode=WRONG_MODE[mode]) if K > s else None}
    return got, ref, bound, wrong


@pytest.mark.parametrize("cin,cout,K,s,Tin,P,fp32,mode", _conv_cases())
def test_conv_tc(cin, cout, K, s, Tin, P, fp32, mode):
    check(f"conv_tc {cin}->{cout} K={K} s={s} Tin={Tin} P={P} fp32={fp32} {mode}",
          *_conv_run(cin, cout, K, s, Tin, P, fp32, mode))


def _convT_run(cin, c, s, n, B=2, scale=1.0):
    """CausalConvTranspose1d(cin, c, 2s, s) as the 2-tap conv with s * c columns (ops.pack_convT_weights)"""
    ops, oc = _ops(), _oc()
    g = _gen(cin + c + s + n)
    w = torch.randn(cin, c, 2 * s, generator=g, device=DEV) * (0.7 / (2 * cin) ** 0.5)
    b = torch.randn(c, generator=g, device=DEV) * 0.1 * scale
    x = torch.randn(B, cin, n, generator=g, device=DEV) * scale
    # coherent window for output channel 0 (every phase r): input channels 0..15 only
    x[:, :16, n // 2:] = _biased(x[:, :16, n // 2:])
    w0 = _biased(torch.randn(16, 2 * s, generator=g, device=DEV).abs() + 0.5) * w.abs().mean()
    w[:, 0] = 0
    w[:16, 0] = w0
    xc, x64 = c8s_value(x)
    y = ops.codec_conv_tc(xc, ops.pack_convT_weights(w, s), b.repeat(s).contiguous(), cout=s * c, kernel_size=2,
                          stride=1, pad_mode="constant", upsample=s)
    w64, b64 = w.to(f64), b.to(f64)
    ref = oc.causal_conv_transpose1d(x64, w64, b64, s)
    S = oc.causal_conv_transpose1d(x64.abs(), w64.abs(), b64.abs(), s)
    nz = (w64 != 0).to(f64)
    n_or = (nz[..., :s] .sum(0) + nz[..., s:].sum(0)).repeat(1, n)[None]     # [1, c, n s]: products of output (o, r)
    bound = (EPS_SPLIT + n_or * EPS_ACC) * S + EPS_C8S * ref.abs()
    wrong_pad = ref.clone()   # reflect instead of zeros: x[-1] read as x[1]
    if n > 1:
        wrong_pad[..., :s] += torch.einsum("cor,bc->bor", w64[..., s:], x64[..., 1])
    wrong = {"plain-bf16": oc.causal_conv_transpose1d(bf(x64), bf(w64), b64, s),
             "pad-mode": wrong_pad if n > 1 else None}
    return ops.c8s_unpack(y), ref, bound, wrong


CONVT_CASES = [(cin, c, s, n) for i, (s, c) in enumerate([(2, 32), (3, 64), (4, 16), (5, 64), (6, 32), (7, 64),
                                                            (8, 16), (8, 32), (2, 256), (4, 128)])
               for cin, n in [((16, 64, 512, 128, 32)[i % 5], 3), ((256, 16, 64)[i % 3], 1000)]]


@pytest.mark.parametrize("cin,c,s,n", CONVT_CASES)
def test_conv_transpose_tc(cin, c, s, n):
    check(f"convT_tc {cin}->{c} s={s} n={n}", *_convT_run(cin, c, s, n))


@pytest.mark.parametrize("n", [1, 2])
def test_conv_transpose_tc_declines_short_input(n):
    """the 2-tap form needs Tin > K = 2: shorter inputs are refused before any launch (the decoder's plan needs n >= 8)"""
    from audiolm_pytorch_b200 import _lib

    ops = _ops()
    x = torch.randn(1, 64, n, device=DEV)
    w = torch.randn(64, 32, 4, device=DEV)
    xc, wu, b = ops.c8s_pack(x), ops.pack_convT_weights(w, 2), torch.zeros(64, device=DEV)
    before = _lib.launch_count()
    with pytest.raises(_lib.AlmError):
        ops.codec_conv_tc(xc, wu, b, cout=64, kernel_size=2, stride=1, pad_mode="constant", upsample=2)
    assert _lib.launch_count() == before


# ---- alm_codec_last_conv ----------------------------------------------------------------------------------------
LAST_CASES = [(32 if K % 2 else 64, K, T, MODES[(K + j) % 3]) for K in range(1, 9) for j, T in enumerate((K, 9000))]


def _last_run(cin, K, T, mode, B=2, scale=1.0, seed=0):
    ops = _ops()
    g = _gen(seed + cin + K + T)
    w = torch.randn(1, cin, K, generator=g, device=DEV) * (0.7 / (cin * K) ** 0.5)
    b = torch.randn(1, generator=g, device=DEV) * 0.1 * scale
    x = torch.randn(B, cin, T, generator=g, device=DEV) * scale
    x[..., T // 2:] = _biased(x[..., T // 2:])            # coherent window: every product positive, lo-biased
    w = _biased(w)
    xc, x64 = c8s_value(x)
    got = ops.codec_last_conv(xc, w, b, pad_mode=mode)
    w64, b64 = w.to(f64), b.to(f64)
    ref = conv64(x64, w64, b64, pad_mode=mode)
    S = conv64(x64.abs(), w64.abs(), b64.abs(), pad_mode=mode)
    bound = (cin * K + 1) * EPS_ACC * S + EPS_F32 * ref.abs()     # + 1: hi + lo summed in fp32
    wrong = {"plain-bf16": conv64(bf(x64), bf(w64), b64, pad_mode=mode),
             "pad-mode": conv64(x64, w64, b64, pad_mode=WRONG_MODE[mode]) if K > 1 else None}
    return got, ref, bound, wrong


@pytest.mark.parametrize("cin,K,T,mode", LAST_CASES)
def test_last_conv(cin, K, T, mode):
    check(f"last_conv Cin={cin} K={K} T={T} {mode}", *_last_run(cin, K, T, mode))


# ---- input scales: the bound is relative --------------------------------------------------------------------------
@pytest.mark.parametrize("scale", [1e-3, 1e3])
def test_input_scales(scale):
    """the conv bounds are relative; the residual unit's carries the ELU's absolute 2^-21 (__expf(v) - 1 near v = 0)"""
    check(f"first_conv x{scale:g}", *_first_conv_case(64, 7, 3000, 2, "reflect", scale, 1))
    st = _ru_state(64, 77, scale=scale)
    x = torch.randn(2, 64, 1000, generator=_gen(3), device=DEV) * scale
    check(f"ru_tc x{scale:g}", *_ru_run(st, x, 9, "replicate", 4))
    st = _ru_state(128, 78, se_ci=32, scale=scale)
    check(f"ru_se_tc x{scale:g}", *_ru_run(st, x.repeat(1, 2, 1), 3, "constant", 1))
    check(f"conv_tc x{scale:g}", *_conv_run(256, 192, 10, 5, 5 * 300, 3, False, "replicate", scale=scale))
    check(f"conv_tc fp32 x{scale:g}", *_conv_run(512, 256, 3, 1, 300, 1, True, "constant", scale=scale))
    check(f"convT_tc x{scale:g}", *_convT_run(128, 64, 5, 300, scale=scale))
    check(f"last_conv x{scale:g}", *_last_run(64, 7, 3000, "replicate", scale=scale))


# ---- size limits ------------------------------------------------------------------------------------------------
def _free():
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def test_batch_past_grid_y_limit():
    """65 536 clips: more than grid.y can hold (65 535); the first and last convs stride over the batch"""
    ops = _ops()
    B, T = 65536, 40
    g = _gen(11)
    w, b = torch.randn(32, 1, 7, generator=g, device=DEV) * 0.4, torch.randn(32, generator=g, device=DEV) * 0.1
    x = torch.randn(B, T, generator=g, device=DEV)
    y = ops.codec_first_conv(x, w, b, pad_mode="replicate")
    wl, bl = torch.randn(1, 32, 7, generator=g, device=DEV) * 0.1, torch.randn(1, generator=g, device=DEV)
    z = ops.codec_last_conv(y, wl, bl, pad_mode="reflect")
    for lo, hi in ((0, 4), (B - 4, B)):
        x64 = x[lo:hi, None].to(f64)
        ref, bound = conv_bound(x64, w.to(f64), b.to(f64), split=False, eps_out=EPS_C8S, pad_mode="replicate")
        check(f"first_conv clips {lo}..{hi - 1} of {B}", ops.c8s_unpack(y[lo:hi]), ref, bound, {})
        h64 = ops.c8s_unpack(y[lo:hi]).to(f64)
        ref = conv64(h64, wl.to(f64), bl.to(f64), pad_mode="reflect")
        S = conv64(h64.abs(), wl.to(f64).abs(), bl.to(f64).abs(), pad_mode="reflect")
        check(f"last_conv clips {lo}..{hi - 1} of {B}", z[lo:hi], ref, (33 * 7 * EPS_ACC) * S + EPS_F32 * ref.abs(), {})
    del x, y, z
    _free()


def _huge_c8s(B, T, P, seed):
    """a random C = 32 C8S tensor [B, 8, P, T / P, 8] (hi chunks, then lo chunks 2^-10 of their size)"""
    x = torch.empty(B, 8, P, T // P, 8, device=DEV, dtype=bf16)
    x.normal_(generator=_gen(seed))
    x[:, 4:] *= 2.0 ** -10
    return x


def _window(x, r0, r1):
    """fp64 value of rows [r0, r1) of every phase plane: times [r0 P, r1 P)"""
    return _ops().c8s_unpack(x[:, :, :, r0:r1]).to(f64)


def test_c8s_past_2_31_elements():
    """C8S tensors of more than 2^31 elements (C = 32, two clips of 2^24 + 64 steps: 4.3 GB each) through the fused
    residual unit and a stride-4 conv; compared on windows at the start, the middle and the end of both clips (the
    second clip's chunks lie past element 2^31)"""
    ops = _ops()
    B, T, d = 2, 2 ** 24 + 64, 9
    assert B * T * 64 > 2 ** 31
    st = _ru_state(32, 91)
    x = _huge_c8s(B, T, 1, 5)
    y = ops.codec_ru_tc(x, ops.pack_ru_weights(st["fn.0.conv.weight"], st["fn.2.conv.weight"]), st["fn.0.conv.bias"],
                        st["fn.2.conv.bias"], dilation=d, pad_mode="replicate", out_phases=4)
    st64 = {k: v.to(f64) for k, v in st.items()}
    halo = 6 * d
    for t0 in (0, T // 2 - 64, T - 256):
        xw = _window(x, max(0, t0 - halo), t0 + 256)
        ref, bound = ru_reference(st64, xw, d, "replicate")
        k = t0 - max(0, t0 - halo)
        got = _window(y, t0 // 4, t0 // 4 + 64)
        check(f"ru_tc 2^31+ window t={t0}", got, ref[..., k:], bound[..., k:], {})
    del x
    _free()
    # the unit's 4-plane output feeds a 32 -> 64, K = 8, stride-4 conv
    g = _gen(6)
    w = torch.randn(64, 32, 8, generator=g, device=DEV) * (0.7 / 256 ** 0.5)
    b = torch.randn(64, generator=g, device=DEV) * 0.1
    z = ops.codec_conv_tc(y, ops.pack_conv_weights(w), b, cout=64, kernel_size=8, stride=4, pad_mode="reflect")
    n = T // 4
    for t0 in (0, n // 2 - 64, n - 128):
        r0 = max(0, t0 - 1)                                    # pad = K - s = 4: one row of each plane before t0
        xw = _window(y, r0, t0 + 128)
        ref, bound = conv_bound(xw, w.to(f64), b.to(f64), split=True, eps_out=EPS_C8S, stride=4, pad_mode="reflect")
        check(f"conv_tc 2^31+ window t={t0}", _window(z, t0, t0 + 128), ref[..., t0 - r0:], bound[..., t0 - r0:], {})
    del y, z
    _free()


# ---- model level: SoundStream.encode_frames / decode_frames ------------------------------------------------------
def _model(**kw):
    from audiolm_pytorch_b200.soundstream import SoundStream

    torch.manual_seed(0)
    cfg = dict(channels=32, strides=(2, 4), channel_mults=(2, 4), codebook_dim=64, codebook_size=64,
               rq_num_quantizers=2, use_local_attn=False)
    cfg.update(kw)
    return SoundStream(**cfg).to(DEV).eval(), cfg


def _count_calls(monkeypatch, name):
    ops = _ops()
    real, calls = getattr(ops, name), []

    def spy(*a, **k):
        calls.append(1)
        return real(*a, **k)

    monkeypatch.setattr(ops, name, spy)
    return calls


def _layer_coef(convs):
    """sum over the layers of their relative bound coefficient: the coarse bound of a stack of unit-gain layers"""
    from audiolm_pytorch_b200.soundstream import CausalConvTranspose1d

    def products(m):
        w = m.conv.weight
        return 2 * w.shape[0] if isinstance(m, CausalConvTranspose1d) else w[0].numel()

    return sum(EPS_SPLIT + EPS_C8S + 2 * EPS_ELU + products(m) * EPS_ACC for m in convs)


def _convs(seq):
    from audiolm_pytorch_b200.soundstream import CausalConv1d, CausalConvTranspose1d

    return [m for m in seq.modules() if isinstance(m, (CausalConv1d, CausalConvTranspose1d))]


def _model_check(label, got, ref, convs, path):
    e = (got.to(f64) - ref).abs().max().item()
    bound = _layer_coef(convs) * ref.abs().max().item()
    print(f"{label} [{path}]: {len(convs)} layers, max err {e:.2e}, err / (sum of per-layer bounds x max|y|) "
          f"{e / bound:.3f}")
    assert e <= bound, f"{label}: {e / bound:.2f}x the coarse per-layer bound"


ENC_CONFIGS = [
    ("replicate", dict(pad_mode="replicate"), 16, True),
    ("strides 3,6 C64", dict(channels=64, strides=(3, 6), channel_mults=(1, 2), codebook_dim=128), 10, True),
    ("strides 2,7 C64", dict(channels=64, strides=(2, 7), channel_mults=(1, 2), codebook_dim=128), 8, True),
    ("dilations 1,2,5", dict(enc_cycle_dilations=(1, 2, 5), dec_cycle_dilations=(2, 4, 8)), 16, True),
    ("codebook_dim 192", dict(codebook_dim=192, pad_mode="constant"), 16, True),
    ("squeeze-excite", dict(squeeze_excite=True, pad_mode="replicate"), 16, True),
    # at 54 samples the d = 9 units' reflect halo does not fit on either path: the fp32 fallback runs with zero padding
    ("guard 54", dict(channels=64, strides=(3, 6), channel_mults=(1, 2), codebook_dim=128, pad_mode="constant"), 9,
     False),
    ("guard 55", dict(strides=(2, 5)), 11, True),
    ("channels 48", dict(channels=48, codebook_dim=64), 16, False),
    ("96-wide down conv", dict(channel_mults=(3, 4)), 16, False),
]


@pytest.mark.parametrize("label,kw,frames,tc", ENC_CONFIGS, ids=[c[0] for c in ENC_CONFIGS])
def test_encode_frames(monkeypatch, label, kw, frames, tc):
    from oracle import codec_se as ose
    from oracle.transformer import sub

    ss, cfg = _model(**kw)
    assert (ss._tc_plan() is not None) == (tc or frames * cfg["strides"][-1] <= 54)
    calls = _count_calls(monkeypatch, "codec_first_conv")
    T = frames * math.prod(cfg["strides"])
    wave = torch.randn(2, 1, T, generator=_gen(T), device=DEV)
    with torch.no_grad():
        got = ss.encode_frames(wave)
    assert bool(calls) == tc, f"{label}: expected the {'tensor-core' if tc else 'fp32'} path"
    st = {k: v.to(f64) for k, v in ss.state_dict().items() if v.is_floating_point()}
    ref = ose.encoder(sub(st, "encoder"), wave.to(f64), cfg["strides"], cfg.get("enc_cycle_dilations", (1, 3, 9)),
                      cfg.get("pad_mode", "reflect")).transpose(1, 2)
    _model_check(f"encode {label}", got, ref, _convs(ss.encoder), "tensor cores" if tc else "fp32 fallback")


DEC_CONFIGS = [
    ("replicate", dict(pad_mode="replicate"), 16, True),
    ("strides 3,6 C64", dict(channels=64, strides=(3, 6), channel_mults=(1, 2), codebook_dim=128), 10, True),
    ("dilations 2,4,8", dict(enc_cycle_dilations=(1, 2, 5), dec_cycle_dilations=(2, 4, 8)), 16, True),
    ("codebook_dim 192", dict(codebook_dim=192), 16, True),
    ("squeeze-excite", dict(squeeze_excite=True, pad_mode="constant"), 16, True),
    ("guard n=7", dict(channels=64, strides=(2, 7), channel_mults=(1, 2), codebook_dim=128, pad_mode="constant"), 7,
     False),
    ("guard n=8", dict(channels=64, strides=(2, 7), channel_mults=(1, 2), codebook_dim=128), 8, True),
    ("channels 48", dict(channels=48, codebook_dim=64), 16, False),
]


@pytest.mark.parametrize("label,kw,n,tc", DEC_CONFIGS, ids=[c[0] for c in DEC_CONFIGS])
def test_decode_frames(monkeypatch, label, kw, n, tc):
    from oracle import codec_se as ose
    from oracle.transformer import sub

    ss, cfg = _model(**kw)
    calls = _count_calls(monkeypatch, "codec_pack_c8s")
    q = torch.randn(2, n, cfg["codebook_dim"], generator=_gen(n), device=DEV) * 0.5
    with torch.no_grad():
        got = ss.decode_frames(q)
    assert bool(calls) == tc, f"{label}: expected the {'tensor-core' if tc else 'fp32'} path"
    st = {k: v.to(f64) for k, v in ss.state_dict().items() if v.is_floating_point()}
    ref = ose.decoder(sub(st, "decoder"), q.to(f64).transpose(1, 2), cfg["strides"],
                      cfg.get("dec_cycle_dilations", (1, 3, 9)), cfg.get("pad_mode", "reflect"))
    _model_check(f"decode {label}", got, ref, _convs(ss.decoder), "tensor cores" if tc else "fp32 fallback")
