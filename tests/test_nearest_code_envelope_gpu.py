"""H100: the nearest-code search kernels against exact and fp64 references across their envelope.

Kernels: the tensor-core search (ops.rvq_encode_tc / nearest_centroid: split-bf16 score GEMM, candidate window,
fp32 re-rank; csrc/rvq_tc.cu), the fp32 CUDA-core search in both generations (ops.rvq_encode: v2 for D % 32 == 0 and
a 16-byte aligned codebook, v1 otherwise; csrc/codec.cu) and ops.rvq_decode.  References and the error band are in
oracle/nearest_code.py:

* integer lattices, where the fp32 expansion is exact in any order: every kernel must return the exact argmin
  (lowest index on ties) on every row, and quantized must match bit for bit;
* continuous inputs (Gaussian, clustered k-means-like codebooks, a large common offset, many shrinking stages) at
  the consumers' shapes: the chosen code lies within the fp32 band of the fp64 minimum, quantized equals the fp32
  replay bit for bit, and rvq_decode of the ids equals quantized bit for bit.

The split-bf16 score error is measured against fp64 per width and must leave 4x headroom under the candidate
window of select_kernel.
"""

import pytest
import torch

from oracle import nearest_code as nc

pytestmark = pytest.mark.gpu
DEV = "cuda"
f32 = torch.float32


def _bits(t):
    return t.contiguous().view(torch.int32)


def _tc(x, cb):
    from audiolm_pytorch_b200 import ops

    return ops.rvq_encode_tc(x, ops.rvq_pack_codebooks(cb))


def _misaligned(cb):
    """a copy of cb 4 bytes past a 16-byte boundary: alm_rvq_encode takes its v1 kernel for it"""
    buf = torch.empty(cb.numel() + 1, device=cb.device, dtype=f32)
    out = buf[1:].view(cb.shape)
    out.copy_(cb)
    return out


def _strided(x, pad=16):
    """x as a column slice of a wider matrix (row pitch D + pad), as vq-wav2vec's per-group search sees it"""
    wide = torch.full((x.shape[0], x.shape[1] + pad), float("nan"), device=x.device, dtype=f32)
    wide[:, 8:8 + x.shape[1]] = x
    return wide[:, 8:8 + x.shape[1]]


def _searches(x, cb):
    """{name: (quantized, ids)} of every search kernel that takes (x, cb); the fp32 search must refuse exactly the
    widths its restated guards refuse"""
    from audiolm_pytorch_b200 import ops
    from audiolm_pytorch_b200._lib import AlmError

    out = {"tensor_cores": _tc(x, cb)}
    D = x.shape[1]
    if nc.rvq_encode_path(D) is None:
        with pytest.raises(AlmError):
            ops.rvq_encode(x, cb)
    else:
        out[f"fp32_{nc.rvq_encode_path(D)}"] = ops.rvq_encode(x, cb)
    if nc.rvq_encode_path(D) == "v2":
        out["fp32_v1"] = ops.rvq_encode(x, _misaligned(cb))
    return out


# ---- (a) integer lattices: zero tolerance ---------------------------------------------------------------------------
@pytest.mark.parametrize("D, C, N, Q", nc.LATTICE_GRID)
def test_lattice_exact(D, C, N, Q):
    from audiolm_pytorch_b200 import ops

    x, cb = nc.lattice(D, C, N, Q, seed=D + C + Q)
    x, cb = x.to(DEV), cb.to(DEV)
    q_ref, i_ref = nc.exact_search(x, cb)
    runs = _searches(x, cb)
    xs = _strided(x)
    runs.update({f"{k} strided": v for k, v in _searches(xs, cb).items()})
    for name, (q, i) in runs.items():
        bad = (i != i_ref).any(1).nonzero()[:, 0]
        assert bad.numel() == 0, (f"{name}: {bad.numel()} of {N} rows differ from the exact argmin; row {bad[0]}: "
                                  f"{i[bad[0]].tolist()} vs {i_ref[bad[0]].tolist()}")
        assert torch.equal(_bits(q), _bits(q_ref)), f"{name}: quantized"
    assert torch.equal(_bits(ops.rvq_decode(i_ref, cb)), _bits(q_ref))


# ---- (b) continuous inputs against fp64 -----------------------------------------------------------------------------
# label: (generator, generator kwargs, N, C, D, Q, groups, largest share of (row, stage) pairs in the fp32 band)
CONTINUOUS = {
    # SoundStream's default quantizer, Gaussian codebooks (8 x 1024 x 512, N = 600, x ~ 3 N(0, 1))
    "soundstream_gaussian_1024": ("gaussian", dict(x_scale=3.0), 600, 1024, 512, 8, 1, 0.1),
    "soundstream_shrinking_1024": ("shrinking", dict(ratio=0.7), 2000, 1024, 512, 8, 1, 0.1),
    "soundstream_shrinking_4096": ("shrinking", dict(ratio=0.7), 1000, 4096, 512, 8, 1, 0.1),
    # HuBERT-base k-means assignment, 500 x 768 (Gaussian centers: test_codec_gpu.py)
    "hubert_base_clustered_1e-1": ("clustered", dict(spread=1e-1), 3000, 500, 768, 1, 1, 1.0),
    "hubert_base_clustered_1e-3": ("clustered", dict(spread=1e-3), 3000, 500, 768, 1, 1, 1.0),
    "hubert_base_clustered_1e-5": ("clustered", dict(spread=1e-5), 3000, 500, 768, 1, 1, 1.0),
    "hubert_base_offset": ("offset", dict(level=30.0), 3000, 500, 768, 1, 1, 1.0),
    "hubert_large_offset": ("offset", dict(level=30.0), 3000, 500, 1024, 1, 1, 1.0),
    "hubert_large_clustered_1e-4": ("clustered", dict(spread=1e-4), 3000, 500, 1024, 1, 1, 1.0),
    "hubert_30s_batch": ("clustered", dict(spread=1e-2), 48000, 500, 768, 1, 1, 1.0),
    # vq-wav2vec: G = 2 groups of 320 x 256, per group on a column slice of [N, 512], or combine_groups
    "vq_wav2vec_per_group": ("clustered", dict(spread=1e-2), 2000, 320, 256, 1, 2, 1.0),
    "vq_wav2vec_combined": ("clustered", dict(spread=1e-2), 4000, 320, 256, 1, 1, 1.0),
    # EnCodec 24 kHz at 24 kbps: 32 stages of 1024 x 128
    "encodec_32_stages": ("shrinking", dict(ratio=0.7), 2000, 1024, 128, 32, 1, 0.1),
    "shrinking_32_stages_ragged": ("shrinking", dict(ratio=0.6), 777, 33, 64, 32, 1, 1.0),
    # widths the fp32 search refuses; the tensor-core search pads them to a multiple of 8
    "width_50": ("gaussian", dict(), 1000, 256, 50, 4, 1, 0.1),
    "width_796": ("clustered", dict(spread=1e-2), 1000, 256, 796, 4, 1, 1.0),
    "width_1020_offset": ("offset", dict(level=10.0), 500, 64, 1020, 2, 1, 1.0),
    "ragged_small": ("gaussian", dict(), 37, 31, 24, 2, 1, 1.0),
    "one_code": ("gaussian", dict(), 7, 1, 8, 1, 1, 1.0),
}


# here the kernels must also pick the fp64 argmin wherever the best code is (distance, not squared) `margin` clear
# of the next one, on at least the given share of (row, stage) pairs
MARGIN = {"soundstream_gaussian_1024": (1e-3, 0.9)}


@pytest.mark.parametrize("label", list(CONTINUOUS))
def test_fp64_band(label):
    from audiolm_pytorch_b200 import ops

    gen, kw, N, C, D, Q, G, max_band = CONTINUOUS[label]
    margin, min_safe = MARGIN.get(label, (None, 0.0))
    g = torch.Generator().manual_seed(sum(map(ord, label)))
    shares = []
    for grp in range(G):
        x, cb = nc.GENERATORS[gen](N, C, D, Q, g=g, **kw)
        x, cb = x.to(DEV), cb.to(DEV)
        runs = {}
        if G > 1:   # the group's columns of the [N, G * D] features
            wide = torch.randn(N, G * D, device=DEV)
            wide[:, grp * D:(grp + 1) * D] = x
            x = wide[:, grp * D:(grp + 1) * D]
            runs["nearest_centroid"] = (None, ops.nearest_centroid(x, ops.rvq_pack_codebooks(cb))[:, None])
        runs.update(_searches(x, cb))
        for name, (q, i) in runs.items():
            share, safe = nc.check_fp64(x, cb, i, quant=q, margin=margin, label=f"{label} {name}")
            assert torch.equal(_bits(ops.rvq_decode(i, cb)), _bits(nc.replay(x, cb, i)[0])), f"{name}: decode"
            assert safe >= min_safe
            shares.append(share)
            print(f"{label} {name}: {share:.3%} of (row, stage) pairs in the fp32 band")
    assert max(shares) <= max_band


# ---- the candidate window of select_kernel --------------------------------------------------------------------------
@pytest.mark.parametrize("D", [8, 24, 64, 128, 256, 512, 768, 1024])
def test_score_window_headroom(D):
    """the split-bf16 scores S ~ r.e of the score GEMM, with the operands built as rvq_encode_tc builds them: the
    relative error max |S - r.e| / (|r|^2 + |e|^2) must stay under CAND_TOL / 4 for every generator"""
    from audiolm_pytorch_b200 import ops

    N, C = 2048, 1024
    g = torch.Generator().manual_seed(D)
    worst = {}
    cases = {"gaussian": {}, "clustered_1e-1": dict(spread=1e-1), "clustered_1e-5": dict(spread=1e-5),
             "offset": dict(level=30.0), "shrinking": dict(ratio=0.6)}
    for name, kw in cases.items():
        gen = nc.GENERATORS[name.split("_")[0]]
        x, cb = gen(N, C, D, 1, g=g, **kw)
        x, cb = x.to(DEV), cb.to(DEV)
        _, packed, _ = ops.rvq_pack_codebooks(cb)
        _, px, _ = ops.rvq_pack_codebooks(x[None])     # [hi | hi | lo] of x -> R' = [hi | lo | hi]
        rp = torch.cat([px[0, :, :D], px[0, :, 2 * D:], px[0, :, :D]], 1).contiguous()
        S = ops.gemm(rp, packed[0], out=torch.empty(N, C, device=DEV, dtype=f32))
        x64, e64 = x.double(), cb[0].double()
        den = (x64 * x64).sum(1, keepdim=True) + (e64 * e64).sum(1)[None]
        worst[name] = ((S.double() - x64 @ e64.T).abs() / den).max().item()
    x, cb = nc.lattice(D, C, N, 1, seed=D)
    _, packed, _ = ops.rvq_pack_codebooks(cb.to(DEV))
    _, px, _ = ops.rvq_pack_codebooks(x.to(DEV)[None])
    rp = torch.cat([px[0, :, :D], px[0, :, 2 * D:], px[0, :, :D]], 1).contiguous()
    S = ops.gemm(rp, packed[0], out=torch.empty(N, C, device=DEV, dtype=f32)).double()
    x64, e64 = x.to(DEV).double(), cb[0].to(DEV).double()
    den = (x64 * x64).sum(1, keepdim=True) + (e64 * e64).sum(1)[None]
    worst["lattice"] = ((S - x64 @ e64.T).abs() / den.clamp_min(1)).max().item()
    print(f"score error / (|r|^2 + |e|^2) at D = {D} on {torch.cuda.get_device_name()}: "
          + ", ".join(f"{k} {v:.2e}" for k, v in worst.items())
          + f"; CAND_TOL / max = {nc.CAND_TOL / max(worst.values()):.0f}x")
    assert max(worst.values()) <= nc.CAND_TOL / 4


# ---- the two fp32 kernels ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D, C, Q, N", [(32, 33, 2, 77), (64, 1024, 8, 600), (256, 320, 4, 1000),
                                        (512, 1024, 8, 600), (768, 500, 1, 2000)])
def test_rvq_encode_v1_equals_v2(D, C, Q, N):
    """alm_rvq_encode's kernels accumulate in the same order, so their ids and quantized agree bit for bit: v2 on
    an aligned codebook, v1 on the same values 4 bytes off a 16-byte boundary"""
    from audiolm_pytorch_b200 import ops

    assert nc.rvq_encode_path(D, True) == "v2" and nc.rvq_encode_path(D, False) == "v1"
    g = torch.Generator().manual_seed(D + C)
    x, cb = nc.shrinking(N, C, D, Q, g=g, ratio=0.8)
    x, cb = _strided(x.to(DEV)), cb.to(DEV)
    q2, i2 = ops.rvq_encode(x, cb)
    q1, i1 = ops.rvq_encode(x, _misaligned(cb))
    assert torch.equal(i1, i2) and torch.equal(_bits(q1), _bits(q2))
    nc.check_fp64(x, cb, i2, quant=q2, label="v2")


# ---- decode -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D, C, Q, Qi", [(8, 1, 1, 1), (50, 33, 4, 4), (200, 1024, 8, 3), (1024, 500, 2, 1),
                                         (128, 1024, 32, 32), (796, 64, 4, 2)])
def test_rvq_decode_bit_exact(D, C, Q, Qi):
    """sum of the selected codes of the first Qi <= Q codebooks in stage order, -1 skipped (a dropped quantizer),
    D above the kernel's 128 threads included: bit for bit the fp32 replay"""
    from audiolm_pytorch_b200 import ops

    g = torch.Generator().manual_seed(D + Q)
    N = 333
    cb = torch.randn(Q, C, D, generator=g).to(DEV)
    ids = torch.randint(0, C, (N, Qi), generator=g)
    ids[torch.rand(N, Qi, generator=g) < 0.2] = -1
    ids[0] = -1
    ids = ids.to(DEV)
    ref = torch.zeros(N, D, device=DEV)
    for s in range(Qi):
        keep = ids[:, s] >= 0
        ref[keep] = ref[keep] + cb[s][ids[keep, s]]
    out = ops.rvq_decode(ids, cb)
    assert out.shape == (N, D) and torch.equal(_bits(out), _bits(ref)) and not out[0].any()


# ---- refusals and consumers -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", [50, 796, 1020, 1024])
def test_rvq_encode_refusals_raise(D):
    """widths the fp32 search cannot hold raise AlmError (no launch, no fault); the device stays usable"""
    from audiolm_pytorch_b200 import ops
    from audiolm_pytorch_b200._lib import AlmError

    assert nc.rvq_encode_path(D) is None
    x, cb = torch.randn(64, D, device=DEV), torch.randn(2, 32, D, device=DEV)
    with pytest.raises(AlmError):
        ops.rvq_encode(x, cb)
    torch.cuda.synchronize()
    q, i = _tc(x, cb)
    nc.check_fp64(x, cb, i, quant=q, label=f"tensor cores D={D}")


@pytest.mark.parametrize("codebook_dim", [50, 796])
def test_soundstream_tokenizes_any_codebook_dim(codebook_dim):
    """SoundStream accepts any codebook_dim; with initialised codebooks tokenize meets the fp64 band on its own
    encoder output"""
    from audiolm_pytorch_b200.soundstream import SoundStream

    torch.manual_seed(codebook_dim)
    ss = SoundStream(codebook_dim=codebook_dim, codebook_size=256, rq_num_quantizers=4, use_local_attn=False)
    ss = ss.to(DEV).eval()
    wave = torch.randn(2, 320 * 16, device=DEV)
    with torch.no_grad():
        h = ss.encode_frames(wave[:, None]).reshape(-1, codebook_dim)
        scale = h.std().item()
        for s, layer in enumerate(ss.rq.rvqs[0].layers):
            layer._codebook.embed.copy_(torch.randn_like(layer._codebook.embed) * scale * 0.7 ** s)
            layer._codebook.initted.fill_(1)
        codes = ss.tokenize(wave)
    cb = ss.rq.rvqs[0].codebooks()
    share, _ = nc.check_fp64(h, cb, codes.reshape(-1, 4), label=f"SoundStream(codebook_dim={codebook_dim})")
    print(f"codebook_dim {codebook_dim}: {share:.3%} of (row, stage) pairs in the fp32 band")
