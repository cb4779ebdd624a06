"""Host checks of the nearest-code search envelope.

* Every search launch a consumer makes, for every configuration its constructor accepts (SoundStream over
  codebook_dim x rq_groups, EncodecWrapper's bandwidths, HuBERT and vq-wav2vec geometries), satisfies a restatement
  of the ALM_REQUIRE guards and shared-memory caps of the entry point it reaches.  The consumers' own forward code
  runs on CPU tensors with the C entry points replaced by a recorder, so a route that sends a width to a kernel
  which refuses it fails here without a GPU.
* The integer lattices the GPU suite compares against (oracle/nearest_code.py) stay exact and keep stressing the
  kernels: the split-bf16 argmin differs from the exact one on a large share of rows, exact ties occur, and the
  exact winner lies inside the candidate window of rvq_tc.cu.
"""

import pytest
import torch

from oracle import nearest_code as nc


# ---- restated guards (csrc/rvq_tc.cu, csrc/codec.cu, csrc/gemm_wgmma.cu) ---------------------------------------------
def _aligned16(t):
    return (t.storage_offset() * t.element_size()) % 16 == 0


def _launch_ok(name, a):
    """a: the arguments ops passes to _lib.call (tensors unconverted)"""
    if name == "alm_rvq_pack_codebooks":
        cb, packed, e2, rows, D = a
        return rows > 0 and D > 0 and packed.shape[-1] == 3 * D and cb.shape[-1] == D
    if name == "alm_rvq_prepare":
        x, ldx, r, quant, ldq, rp, N, *widths = a   # x's width, then the (padded) search width
        Dx, D = widths[0], widths[-1]
        return N > 0 and Dx > 0 and D >= Dx and ldx >= Dx and ldq >= D and rp.shape[-1] == 3 * D
    if name == "alm_gemm_bf16":
        A, a_mn, lda, sA, B, b_mn, ldb, sB, C, c_fp32, ldc, sC, M, N, K, nb = a[:16]
        # lda / ldb: 16-byte row pitch; the tensor maps also need 16-byte aligned base addresses
        return (M > 0 and N > 0 and K > 0 and lda % 8 == 0 and ldb % 8 == 0 and sA % 8 == 0 and sB % 8 == 0
                and _aligned16(A) and _aligned16(B))
    if name == "alm_rvq_select":
        S, lds, e2, cb, r, quant, ldq, rp, idx, ldi, N, D, C, write_rp = a
        return N > 0 and D > 0 and C > 0 and cb.shape[-1] == D and lds >= C and ldq >= D
    if name == "alm_rvq_encode":
        x, ldx, cb, ws, quant, ldq, idx, ldi, N, D, C, Q = a
        return N > 0 and C > 0 and Q > 0 and nc.rvq_encode_path(D, _aligned16(cb)) is not None
    if name == "alm_rvq_decode":
        idx, ldi, cb, out, ldo, N, D, C, Q = a
        return N > 0 and D > 0 and C > 0 and Q > 0
    raise AssertionError(f"unexpected launch {name}")


@pytest.fixture
def launches(monkeypatch):
    """replace the C entry points by a recorder of (name, accepted) and let ops run on CPU tensors"""
    from audiolm_pytorch_b200 import _lib, ops

    seen = []
    monkeypatch.setattr(_lib, "call", lambda name, *a: seen.append((name, _launch_ok(name, a))))
    monkeypatch.setattr(ops, "_check_cuda", lambda *ts: None)
    return seen


def _refused(seen):
    assert seen, "no search launch recorded"
    return [name for name, ok in seen if not ok]


def _initialise(rvq):
    for layer in rvq.layers:
        layer._codebook.initted.fill_(1)
        layer._codebook.embed.normal_()


# ---- consumers ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("codebook_dim", [8, 12, 50, 64, 100, 128, 256, 500, 512, 796, 800, 1020, 1024])
@pytest.mark.parametrize("rq_groups", [1, 2, 4])
def test_soundstream_searches_accepted(launches, codebook_dim, rq_groups):
    """SoundStream accepts any codebook_dim divisible by rq_groups; tokenize and decode of every one must reach only
    launches the kernels take (widths 50, 796 and 1020 once went to alm_rvq_encode, which refuses them)"""
    from audiolm_pytorch_b200.soundstream import SoundStream

    if codebook_dim % rq_groups:
        with pytest.raises(AssertionError):
            SoundStream(codebook_dim=codebook_dim, codebook_size=64, rq_groups=rq_groups, use_local_attn=False)
        return
    ss = SoundStream(codebook_dim=codebook_dim, codebook_size=64, rq_num_quantizers=3, rq_groups=rq_groups,
                     use_local_attn=False).eval()
    for rvq in ss.rq.rvqs:
        _initialise(rvq)
    with torch.no_grad():
        _, idx, _ = ss.rq(torch.randn(2, 5, codebook_dim))
        ss.rq.get_output_from_indices(torch.zeros(rq_groups, 2, 5, 3, dtype=torch.long))
    assert not _refused(launches), f"codebook_dim {codebook_dim} / {rq_groups} groups: refused {_refused(launches)}"


@pytest.mark.parametrize("bandwidth", [1.5, 3.0, 6.0, 12.0, 24.0])
def test_encodec_searches_accepted(launches, bandwidth):
    """EncodecWrapper's quantizer: ResidualVQ(dim=128, codebook_size=1024, num_quantizers=n_q of the bandwidth)"""
    from audiolm_pytorch_b200.encodec import BANDWIDTH_QUANTIZERS, CODEBOOK_SIZE, DIM
    from audiolm_pytorch_b200.soundstream import ResidualVQ

    rvq = ResidualVQ(dim=DIM, codebook_size=CODEBOOK_SIZE, num_quantizers=BANDWIDTH_QUANTIZERS[bandwidth]).eval()
    _initialise(rvq)
    rvq(torch.randn(1, 75, DIM))
    assert not _refused(launches)


@pytest.mark.parametrize("D, heads, clusters", [(768, 12, 500), (1024, 16, 500), (1024, 16, 1000), (512, 8, 2000),
                                                (1280, 20, 500), (384, 6, 100)])
def test_hubert_searches_accepted(launches, D, heads, clusters):
    """HubertWithKmeans: widths its envelope accepts, centers packed and searched as hubert.py does"""
    from audiolm_pytorch_b200 import ops
    from audiolm_pytorch_b200.hubert import check_envelope
    from oracle import hubert as oh

    check_envelope(dict(oh.BASE, encoder_embed_dim=D, encoder_ffn_embed_dim=4 * D, encoder_attention_heads=heads,
                        conv_pos_groups=16, activation_fn="gelu"))
    centers = torch.randn(clusters, D)
    ids = ops.nearest_centroid(torch.randn(2 * 49, D), ops.rvq_pack_codebooks(centers.float()[None]))
    assert ids.shape == (98,) and not _refused(launches)


@pytest.mark.parametrize("groups, var_dim", [(2, 256), (2, 8), (4, 128), (1, 512), (8, 64), (3, 24)])
@pytest.mark.parametrize("combine_groups", [False, True])
def test_vq_wav2vec_searches_accepted(launches, groups, var_dim, combine_groups):
    """FairseqVQWav2Vec.assign: one search over all groups with combine_groups, else one per group on a column slice
    of the [rows, G * var_dim] features (row pitch G * var_dim)"""
    from types import SimpleNamespace

    from audiolm_pytorch_b200 import ops
    from audiolm_pytorch_b200.vq_wav2vec import FairseqVQWav2Vec

    num_vars = 320
    e = torch.randn(num_vars, 1 if combine_groups else groups, var_dim)   # the k-means embedding, as _pack reads it
    if combine_groups:
        codes = ops.rvq_pack_codebooks(e[:, 0][None])
    else:
        cb, packed, e2 = ops.rvq_pack_codebooks(e.permute(1, 0, 2))
        codes = [(cb[g:g + 1], packed[g:g + 1], e2[g:g + 1]) for g in range(groups)]
    stub = SimpleNamespace(_packed=lambda: {"codes": codes}, geo={"combine_groups": combine_groups},
                           codebook_size=num_vars)
    ids = FairseqVQWav2Vec.assign(stub, torch.randn(2, 30, groups, var_dim))
    assert ids.shape == (2, 30, groups) and not _refused(launches)


@pytest.mark.parametrize("D, aligned, path", [(8, True, "v1"), (50, True, None), (96, True, "v2"), (96, False, "v1"),
                                              (768, True, "v2"), (792, True, "v1"), (796, True, None),
                                              (992, True, "v2"), (1020, True, None), (1024, True, None)])
def test_rvq_encode_path_restatement(D, aligned, path):
    """the restated dispatch of alm_rvq_encode at its edges: v2 up to D = 992, v1 up to D = 792, errors beyond"""
    assert nc.rvq_encode_path(D, aligned) == path


# ---- lattice self-checks --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D, C, N, Q", nc.LATTICE_GRID)
def test_lattice_stresses_the_kernels(D, C, N, Q):
    x, cb = nc.lattice(D, C, N, Q, seed=D + C + Q)
    assert x.shape == (N, D) and cb.shape == (Q, C, D)
    if N > 1:
        assert x[1:, 0].any() and x[1:, -1].any(), "the first and last columns carry data"
    _, ids = nc.exact_search(x, cb)
    assert not nc.exactness_violations(x, cb, ids)
    hi, lo = nc.bf16_split(cb)
    assert torch.equal(hi + lo, cb), "the split must represent every code exactly"
    hi, lo = nc.bf16_split(x)
    assert torch.equal(hi + lo, x)
    rows = slice(0, 1000)
    r = x[rows].double()
    differs = ties = total = 0
    for s in range(Q):
        e = cb[s].double()
        r2, e2 = (r * r).sum(1, keepdim=True), (e * e).sum(1)[None]
        approx = e2 - 2 * nc.split_scores(r, e)
        best = ids[rows, s:s + 1]
        inside = approx.gather(1, best) <= approx.min(1, keepdim=True).values + nc.CAND_TOL * (r2 + e2.expand_as(
            approx).gather(1, best))
        assert inside.all(), "the exact winner must lie inside the candidate window"
        dist = torch.sqrt(nc._d2(r, e).float())
        differs += int((approx.argmin(1, keepdim=True) != best).sum())
        ties += int(((dist == dist.min(1, keepdim=True).values).sum(1) > 1).sum())
        total += r.shape[0]
        r = r - e[best[:, 0]]
    if C >= 31 and total >= 100:
        assert differs / total > 0.15, f"split argmin differs from the exact one on only {differs / total:.1%}"
        assert ties / total > 0.01, f"exact ties on only {ties / total:.1%} of rows"


def test_lattice_special_rows():
    """x = 0, rows equal to codewords, and the duplicated dead code at 1, 129 and C - 1 picked at its lowest index"""
    x, cb = nc.lattice(64, 320, 37, 1, seed=3)
    assert not x[0].any()
    assert torch.equal(cb[0, 1], cb[0, 129]) and torch.equal(cb[0, 1], cb[0, 319])
    _, ids = nc.exact_search(x, cb)
    assert ids[4, 0] == 1 and ids[3, 0] == 1   # row 3 equals code C - 1, row 4 the dead code
    assert ids[1, 0] == 0
