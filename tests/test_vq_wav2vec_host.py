"""Host checks of FairseqVQWav2Vec: the oracle against the reference's ids (tests/golden/vq_wav2vec.pt), the checkpoint
loader with fairseq not importable (cfg and args forms, state-dict keys), the ValueError for missing config fields and
tensor / config disagreements, the reference's assertion for gumbel and quantizer-less models, the envelope errors at
construction, and the block-diagonal projection weight."""

import contextlib
import builtins
import sys

import pytest
import torch
import torch.nn.functional as F

from oracle import golden
from oracle import vq_wav2vec as ov

ARCH_KEYS = ("conv_feature_layers", "activation", "log_compression", "skip_connections_feat", "residual_scale",
             "vq_type")


@pytest.fixture(scope="module")
def g():
    return golden.load("vq_wav2vec.pt")


@contextlib.contextmanager
def without_fairseq():
    """`import fairseq` / `import omegaconf` fail inside the block"""
    real = builtins.__import__

    def guarded(name, *a, **k):
        if name.split(".")[0] in ("fairseq", "omegaconf"):
            raise ImportError(f"{name} is not importable here")
        return real(name, *a, **k)

    with pytest.MonkeyPatch.context() as mp:
        for n in [n for n in sys.modules if n.split(".")[0] in ("fairseq", "omegaconf")]:
            mp.delitem(sys.modules, n)
        mp.setattr(builtins, "__import__", guarded)
        yield


def _build(tmp_path, st, arch, form="args"):
    from audiolm_pytorch_b200.vq_wav2vec import FairseqVQWav2Vec

    ov.write_checkpoint(tmp_path / "vq.pt", st, arch, form)
    return FairseqVQWav2Vec(tmp_path / "vq.pt")


@pytest.mark.parametrize("name", ["A", "B"])
def test_oracle_matches_reference_ids(g, name):
    m = g[name]
    st = {k: v.double() for k, v in m["state"].items()}
    e = ov.codewords(st, 2)
    for wave, feats, ze_g, ids, flat in zip(m["waves"], m["features"], m["ze"], m["ids"], m["ids_flat"]):
        f = ov.features(st, m["arch"], wave.double())
        ze = ov.project(st, f)
        assert torch.allclose(f.float(), feats, rtol=1e-5, atol=1e-5)
        assert torch.allclose(ze.float(), ze_g, rtol=1e-5, atol=1e-5)
        assert ids.shape == (wave.shape[0], f.shape[1], 2) and ids.dtype == torch.int64
        assert torch.equal(ov.ids(ze, e), ids)
        assert torch.equal(flat, ids.reshape(ids.shape[0], -1))


@pytest.mark.parametrize("name", ["A", "B"])
@pytest.mark.parametrize("form", ["cfg", "args"])
def test_loader_without_fairseq(tmp_path, g, name, form):
    from audiolm_pytorch_b200.vq_wav2vec import FairseqVQWav2Vec

    m = g[name]
    ov.write_checkpoint(tmp_path / "vq.pt", m["state"], m["arch"], form)
    if form == "cfg":
        assert ov.FAKE_ENUM_MODULE.encode() in (tmp_path / "vq.pt").read_bytes()
    with without_fairseq():
        q = FairseqVQWav2Vec(tmp_path / "vq.pt")
    assert q.arch["activation"] == m["arch"]["activation"]
    assert (q.groups, q.codebook_size, q.downsample_factor, q.target_sample_hz) == (2, 320, 80, 24000)
    assert q.geo["combine_groups"] == m["arch"]["combine_groups"]
    assert q.geo["affine"] == [not m["arch"]["non_affine_group_norm"]] * 8
    sd = q.state_dict()
    assert sorted(sd) == sorted("model." + k for k in m["state"])
    assert all(torch.equal(sd["model." + k], v) for k, v in m["state"].items())
    assert "model.feature_aggregator.conv_layers.0.0.weight" in sd


@pytest.mark.parametrize("field", ARCH_KEYS)
def test_missing_field_names_it(tmp_path, g, field):
    m = g["A"]
    arch = {k: v for k, v in m["arch"].items() if k != field}
    with pytest.raises(ValueError, match=field):
        _build(tmp_path, m["state"], arch)


def test_no_config_raises(tmp_path, g):
    from audiolm_pytorch_b200.vq_wav2vec import FairseqVQWav2Vec

    torch.save({"model": g["A"]["state"]}, tmp_path / "vq.pt")
    with pytest.raises(ValueError, match="cannot read the vq-wav2vec architecture"):
        FairseqVQWav2Vec(tmp_path / "vq.pt")


@pytest.mark.parametrize("change, match", [
    (dict(vq_groups=4), "vq_groups"),
    (dict(vq_vars=100), "vq_vars"),
    (dict(combine_groups=False), "combine_groups"),
    (dict(non_affine_group_norm=True), "non_affine_group_norm"),
    (dict(conv_feature_layers="[(64, 10, 5), (64, 7, 4)] + [(64, 4, 2)] * 3 + [(64, 1, 1)] * 3"), "conv 1"),
    (dict(conv_feature_layers="[(64, 10, 5)] * 2"), "conv_feature_layers"),
])
def test_tensor_cfg_mismatch_raises(tmp_path, g, change, match):
    m = g["A"]
    with pytest.raises(ValueError, match=match):
        _build(tmp_path, m["state"], dict(m["arch"], **change))


def test_gumbel_and_quantizerless_models_fail_like_the_reference(tmp_path, g):
    from audiolm_pytorch_b200.vq_wav2vec import INVALID

    m = g["A"]
    gumbel = {k: v for k, v in m["state"].items() if k != ov.EMBEDDING}
    gumbel["vector_quantizer.vars"] = torch.randn(1, 640, 32)
    gumbel["vector_quantizer.weight_proj.weight"] = torch.randn(640, 64)
    with pytest.raises(AssertionError, match=INVALID):
        _build(tmp_path, gumbel, dict(m["arch"], vq_type="gumbel"))
    plain = {k: v for k, v in m["state"].items() if not k.startswith("vector_quantizer.")}
    with pytest.raises(AssertionError, match=INVALID):
        _build(tmp_path, plain, dict(m["arch"], vq_type="none"))
    with pytest.raises(AssertionError, match=INVALID):  # a k-means config without its codebook
        _build(tmp_path, plain, m["arch"])


@pytest.mark.parametrize("case, match", [("activation", "activation"), ("width", "multiples of 8"),
                                         ("var_dim", "var_dim"), ("vq_dim", "vq_dim")])
def test_envelope_errors_at_construction(tmp_path, g, case, match):
    arch = dict(g["A"]["arch"])
    kw = dict(groups=2, num_vars=320, combine_groups=True)
    if case == "activation":
        arch["activation"] = "tanh"
    elif case == "width":
        arch["conv_feature_layers"] = "[(60, 10, 5), (60, 8, 4)]"
    elif case == "var_dim":
        kw["groups"], arch["vq_groups"] = 16, 16
    else:
        arch["vq_dim"] = 32
    st = ov.random_state(arch, seed=1, **kw)
    with pytest.raises(NotImplementedError, match=match):
        _build(tmp_path, st, arch)


def test_published_shape_inside_envelope(tmp_path):
    from audiolm_pytorch_b200.hubert import receptive_field

    arch = ov.PUBLISHED
    st = ov.random_state(arch, seed=2, groups=2, num_vars=320, combine_groups=False)
    q = _build(tmp_path, st, arch, "cfg")
    assert (q.groups, q.codebook_size, q.geo["var_dim"]) == (2, 320, 256)
    assert receptive_field(q.geo["layers"]) == 465


@pytest.mark.parametrize("C, G", [(64, 2), (512, 2), (512, 4), (96, 3), (64, 1)])
def test_block_diagonal_projection_equals_grouped_conv(C, G):
    from audiolm_pytorch_b200.vq_wav2vec import block_diagonal_weight

    gen = torch.Generator().manual_seed(C + G)
    w = torch.randn(C, C // G, 1, generator=gen, dtype=torch.float64)
    x = torch.randn(3, C, 17, generator=gen, dtype=torch.float64)
    dense = block_diagonal_weight(w)
    assert dense.shape == (C, C)
    assert torch.equal(dense, ov.block_diagonal(w))
    assert torch.allclose(torch.einsum("oc,bct->bot", dense, x), F.conv1d(x, w, groups=G), rtol=1e-13, atol=1e-13)


def test_cpu_input_raises(tmp_path, g):
    from audiolm_pytorch_b200._lib import AlmError

    m = g["B"]
    q = _build(tmp_path, m["state"], m["arch"])
    with pytest.raises(AlmError):
        q(m["waves"][0])
