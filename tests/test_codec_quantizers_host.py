"""Host checks of SoundStream's residual FSQ / LFQ quantizers: state-dict surface against the reference
(tests/golden/quantizers.pt), the constructor asserts, the envelope, the host-side stage constants and the quantizer
restatement against the reference."""

import pytest
import torch

from oracle import golden

MODELS = ("fsq", "fsq_groups", "lfq", "lfq_groups")


@pytest.fixture(scope="module")
def g():
    return golden.load("quantizers.pt")


@pytest.mark.parametrize("name", MODELS)
def test_state_dict_matches_reference(g, name):
    from audiolm_pytorch_b200 import SoundStream

    case = g[name]
    ss = SoundStream(**case["kwargs"])
    ours = [(k, tuple(v.shape)) for k, v in ss.state_dict().items()]
    assert ours == case["keys"]
    assert not any(".layers." in k for k, _ in ours if k.startswith("rq."))   # levels, scales, masks: not persistent
    ss.load_state_dict(case["state"], strict=True)
    assert ss.codebook_size == case["codebook_size"]
    assert ss.use_finite_scalar_quantizer == name.startswith("fsq")
    assert ss.use_lookup_free_quantizer == name.startswith("lfq")


def test_vq_codec_unchanged():
    from audiolm_pytorch_b200 import SoundStream
    from audiolm_pytorch_b200.soundstream import GroupedResidualVQ

    ss = SoundStream(codebook_size=64, channels=4, codebook_dim=32, use_local_attn=False, rq_num_quantizers=3)
    assert isinstance(ss.rq, GroupedResidualVQ) and ss.codebook_size == 64
    assert not ss.use_finite_scalar_quantizer and not ss.use_lookup_free_quantizer
    assert [k for k in ss.state_dict() if k.startswith("rq.")] == [
        f"rq.rvqs.0.layers.{q}._codebook.{b}" for q in range(3) for b in ("initted", "cluster_size", "embed_avg", "embed")]


def test_constructor_asserts_match_reference():
    from audiolm_pytorch_b200 import SoundStream

    kw = dict(channels=4, codebook_dim=32, use_local_attn=False)
    with pytest.raises(AssertionError):
        SoundStream(codebook_size=1024, use_lookup_free_quantizer=True, use_finite_scalar_quantizer=True, **kw)
    with pytest.raises(AssertionError, match="`codebook_size` must be set"):
        SoundStream(use_lookup_free_quantizer=True, **kw)
    with pytest.raises(AssertionError, match="`codebook_size` must be set"):
        SoundStream(codebook_size=1024, finite_scalar_quantizer_levels=[8, 5], use_lookup_free_quantizer=True, **kw)
    with pytest.raises(AssertionError, match="`finite_scalar_quantizer_levels` must be set"):
        SoundStream(codebook_size=1024, finite_scalar_quantizer_levels=[8, 5], use_finite_scalar_quantizer=True, **kw)
    with pytest.raises(AssertionError, match="`finite_scalar_quantizer_levels` must be set"):
        SoundStream(use_finite_scalar_quantizer=True, **kw)
    with pytest.raises(AssertionError, match="`codebook_size` must be set"):
        SoundStream(**kw)
    ss = SoundStream(finite_scalar_quantizer_levels=[8, 5, 5, 5], use_finite_scalar_quantizer=True, **kw)
    assert ss.codebook_size == 1000 and ss.rq.codebook_size == 1000


@pytest.mark.parametrize("kw, bad", [
    (dict(use_finite_scalar_quantizer=True, finite_scalar_quantizer_levels=[5] * 17), "[5, 5"),
    (dict(use_finite_scalar_quantizer=True, finite_scalar_quantizer_levels=[8, 1, 5]), "[8, 1, 5]"),
    (dict(use_finite_scalar_quantizer=True, finite_scalar_quantizer_levels=[2 ** 16, 2 ** 15]), "65536"),
    (dict(use_lookup_free_quantizer=True, codebook_size=1000), "1000"),
    (dict(use_lookup_free_quantizer=True, codebook_size=2 ** 17), "131072"),
    (dict(use_lookup_free_quantizer=True, codebook_size=1024, rq_num_quantizers=33), "33"),
    (dict(use_lookup_free_quantizer=True, codebook_size=1024, rq_groups=3, codebook_dim=48), "groups=3"),
    (dict(use_lookup_free_quantizer=True, codebook_size=1024, rq_groups=8, codebook_dim=64), "groups=8"),
    (dict(use_lookup_free_quantizer=True, codebook_size=1024, codebook_dim=2048), "2048"),
    (dict(use_lookup_free_quantizer=True, codebook_size=1024, codebook_dim=30), "30"),
    (dict(use_finite_scalar_quantizer=True, finite_scalar_quantizer_levels=[8, 5], rq_kwargs=dict(preserve_symmetry=True)),
     "preserve_symmetry"),
    (dict(use_lookup_free_quantizer=True, codebook_size=1024, rq_kwargs=dict(spherical=True)), "spherical"),
    (dict(use_lookup_free_quantizer=True, codebook_size=1024, rq_kwargs=dict(soft_clamp_input_value=10.0)),
     "soft_clamp_input_value"),
])
def test_outside_envelope_raises_with_value(kw, bad):
    from audiolm_pytorch_b200 import SoundStream

    base = dict(channels=4, codebook_dim=32, use_local_attn=False)
    with pytest.raises(NotImplementedError, match=bad.replace("[", r"\[")):
        SoundStream(**{**base, **kw})


def test_envelope_edges_construct():
    from audiolm_pytorch_b200 import SoundStream

    base = dict(channels=4, use_local_attn=False)
    SoundStream(codebook_dim=16, use_finite_scalar_quantizer=True, finite_scalar_quantizer_levels=[2] * 16,
                rq_num_quantizers=32, **base)
    SoundStream(codebook_dim=4096, rq_groups=4, use_lookup_free_quantizer=True, codebook_size=2, **base)
    SoundStream(codebook_dim=3, use_finite_scalar_quantizer=True, finite_scalar_quantizer_levels=[3, 7, 2],
                rq_num_quantizers=1, **base)
    SoundStream(codebook_dim=32, use_lookup_free_quantizer=True, codebook_size=1024,
                rq_kwargs=dict(entropy_loss_weight=0.1, quantize_dropout_multiple_of=2), **base)


def test_training_mode_raises():
    from audiolm_pytorch_b200 import SoundStream

    ss = SoundStream(channels=4, codebook_dim=32, use_local_attn=False, use_lookup_free_quantizer=True,
                     codebook_size=1024)
    with pytest.raises(NotImplementedError):
        ss.rq.train()(torch.zeros(1, 2, 32))


@pytest.mark.parametrize("levels, Q", [([8, 5, 5, 5], 4), ([2], 32), ([3, 7, 2, 16, 5], 6), ([5, 5, 4, 4], 1)])
def test_fsq_constants_are_the_quantizers(levels, Q):
    """the kernels' stage constants are bit-identical to the fp32 buffers of the restated quantizer"""
    from audiolm_pytorch_b200 import ops
    from oracle import scalar_quant as osq

    consts, ints = ops.fsq_constants(levels, Q)
    lv, basis, half_l, offset, shift, scales = osq.fsq_buffers(levels, Q)
    assert consts.dtype == torch.float32 and consts.shape == (4 + Q, len(levels))
    assert torch.equal(consts[0], half_l) and torch.equal(consts[1], offset) and torch.equal(consts[2], shift)
    assert torch.equal(consts[3], (lv // 2).float()) and torch.equal(consts[4:], scales)
    assert torch.equal(ints[0], lv) and torch.equal(ints[1], basis)
    # every code index is a distinct mixed-radix number below prod(L)
    digits = torch.stack(torch.meshgrid(*[torch.arange(l_) for l_ in levels], indexing="ij"), -1).reshape(-1, len(levels))
    idx = (digits * basis.long()).sum(-1)
    assert torch.equal(idx.sort().values, torch.arange(int(torch.tensor(levels).prod())))


def test_lfq_constants():
    from audiolm_pytorch_b200 import ops

    consts, ints = ops.lfq_constants(10, 5)
    assert torch.equal(consts[4:], torch.tensor([[2.0 ** -q] * 10 for q in range(5)]))
    assert ints[1].tolist() == [2 ** (9 - j) for j in range(10)]


@pytest.mark.parametrize("name", MODELS)
def test_oracle_matches_reference(g, name):
    from oracle import scalar_quant as osq

    case = g[name]
    kw, st = case["kwargs"], case["state"]
    enc, quant, idx = osq.soundstream_tokenize(kw, st, case["wave"])
    assert (enc - case["enc"]).abs().max() < 2e-5
    assert idx.dtype == case["idx"].dtype and str(idx.dtype) == case["idx_dtype"]
    assert torch.equal(idx, case["idx"])
    assert (quant - case["quant"]).abs().max() < 2e-5
    recon = osq.soundstream_decode_indices(kw, st, idx)
    assert (recon - case["recon_idx"]).abs().max() < 2e-5 * max(1.0, case["recon_idx"].abs().max().item())
    recon_c = osq.soundstream_decode_indices(kw, st, idx[..., :case["coarse_q"]])
    assert (recon_c - case["recon_coarse"]).abs().max() < 2e-5 * max(1.0, case["recon_coarse"].abs().max().item())


@pytest.mark.parametrize("mode", ["fsq", "lfq"])
def test_fp64_restatement_matches_oracle(mode):
    """the fp64 restatement the GPU tests use agrees with the fp32 quantizer on its margin-safe rows, and a corrupted
    index decodes to something else"""
    from oracle import scalar_quant as osq

    gen = torch.Generator().manual_seed(11)
    levels, cs, Q, D = [8, 5, 5, 5], 1024, 4, 32
    rq = (osq.GroupedResidualFSQ(dim=D, levels=levels, num_quantizers=Q) if mode == "fsq"
          else osq.GroupedResidualLFQ(dim=D, codebook_size=cs, num_quantizers=Q)).eval()
    x = torch.randn(2, 200, D, generator=gen)
    with torch.no_grad():
        out = rq(x)
    p = rq.rvqs[0]
    w = (p.project_in.weight[None], p.project_in.bias[None], p.project_out.weight[None], p.project_out.bias[None])
    kw = dict(mode=mode, levels=levels, codebook_dim=10, num_quantizers=Q)
    q64, i64, margin = osq.residual_sq_fp64(x.reshape(-1, D), groups=1, weights=w, fp32_projection_error=1e-5, **kw)
    safe = margin[0, :, -1] > 1
    assert safe.float().mean() > 0.5
    assert torch.equal(margin.cummin(-1).values, margin)   # a stage's margin covers the stages before it
    assert torch.equal(i64[0][safe], out[1][0].reshape(-1, Q).long()[safe])
    assert (q64[safe] - out[0].reshape(-1, D).double()[safe]).abs().max() < 1e-5
    dec = osq.decode_fp64(i64, weights=w, **kw)
    assert (dec - q64).abs().max() < 1e-9
    bad = i64.clone()
    bad[0, 0, 0] = (bad[0, 0, 0] + 1) % (1000 if mode == "fsq" else cs)
    assert (osq.decode_fp64(bad, weights=w, **kw)[0] - q64[0]).abs().max() > 1e-3
