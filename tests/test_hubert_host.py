"""Host checks of HubertWithKmeans: the oracle against the reference's ids (tests/golden/hubert.pt), the checkpoint loader
with fairseq and omegaconf not importable (both cfg forms, both weight-norm key forms, state-dict keys, refusal of
unlisted globals), the envelope errors at construction and the positional conv weight-norm fold."""

import argparse
import builtins
import contextlib
import os
import pickle
import sys

import pytest
import torch

from oracle import golden
from oracle import hubert as oh


@pytest.fixture(scope="module")
def g():
    return golden.load("hubert.pt")


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


def _files(tmp_path, g, form="cfg", st=None, arch=None):
    ck, km = tmp_path / "hubert.pt", tmp_path / "km.bin"
    oh.write_checkpoint(ck, g["state"] if st is None else st, g["arch"] if arch is None else arch, form)
    oh.write_kmeans(km, g["centers"])
    return ck, km


def test_oracle_matches_reference_ids(g):
    st = {k: v.double() for k, v in g["state"].items()}
    for wave, feats, ids in zip(g["waves"], g["features"], g["ids"]):
        f = oh.extract_features(st, g["arch"], wave.double(), g["output_layer"])
        assert torch.allclose(f.float(), feats, rtol=1e-5, atol=1e-5)
        assert torch.equal(oh.assign(f, g["centers"]), ids)


@pytest.mark.parametrize("form", ["cfg", "args"])
@pytest.mark.parametrize("wn", ["weight_g", "parametrizations"])
def test_loader_without_fairseq(tmp_path, g, form, wn):
    from audiolm_pytorch_b200.hubert import HubertWithKmeans

    st = g["state"] if wn == "weight_g" else oh.parametrized_weight_norm(g["state"])
    ck, km = _files(tmp_path, g, form, st=st)
    if form == "cfg":
        assert b"fairseq.dataclass.constants" in ck.read_bytes()
    with without_fairseq():
        h = HubertWithKmeans(ck, km, output_layer=g["output_layer"])
    assert h.arch["extractor_mode"] == "default" and h.arch["encoder_embed_dim"] == g["arch"]["encoder_embed_dim"]
    assert (h.groups, h.codebook_size, h.downsample_factor) == (1, g["centers"].shape[0], 320)
    sd = h.state_dict()
    assert sorted(sd) == sorted(["cluster_centers"] + ["model." + k for k in st])
    assert all(torch.equal(sd["model." + k], v) for k, v in st.items())
    assert torch.equal(sd["cluster_centers"], g["centers"])
    assert {"model.final_proj.weight", "model.label_embs_concat", "model.mask_emb"} <= set(sd)


def test_loader_refuses_unlisted_global(tmp_path):
    from audiolm_pytorch_b200.hubert import load_checkpoint

    path = tmp_path / "evil.pt"
    torch.save({"model": {}, "cfg": {"model": {"x": os.getcwd}}}, path)
    with pytest.raises(pickle.UnpicklingError, match="posix.getcwd|os.getcwd"):
        load_checkpoint(path)


def test_unreadable_cfg_raises(tmp_path, g):
    from audiolm_pytorch_b200.hubert import HubertWithKmeans

    ck, km = _files(tmp_path, g)
    torch.save({"model": g["state"]}, ck)
    with pytest.raises(ValueError, match="cannot read the HuBERT architecture"):
        HubertWithKmeans(ck, km, output_layer=1)
    torch.save({"model": g["state"], "args": argparse.Namespace(encoder_layers=4)}, ck)
    with pytest.raises(ValueError, match="lacks"):
        HubertWithKmeans(ck, km, output_layer=1)


@pytest.mark.parametrize("change, match", [
    (dict(extractor_mode="other"), "extractor_mode"),
    (dict(encoder_embed_dim=1280, encoder_attention_heads=16, conv_pos_groups=16), "head width"),
    (dict(encoder_attention_heads=8), "head width"),
    (dict(encoder_ffn_embed_dim=250), "multiples of 8"),
    (dict(conv_pos_groups=32), "group width"),
])
def test_envelope_errors_at_construction(tmp_path, g, change, match):
    from audiolm_pytorch_b200.hubert import HubertWithKmeans

    ck, km = _files(tmp_path, g, "args", arch=dict(g["arch"], **change))
    with pytest.raises(NotImplementedError, match=match):
        HubertWithKmeans(ck, km, output_layer=1)


def test_published_families_inside_envelope():
    from audiolm_pytorch_b200.hubert import check_envelope, receptive_field, parse_conv_layers

    for arch in (oh.BASE, oh.LARGE):
        check_envelope(dict(arch, activation_fn="gelu"))
    assert receptive_field(parse_conv_layers(oh.BASE["conv_feature_layers"])) == 400


def test_output_layer_out_of_range(tmp_path, g):
    from audiolm_pytorch_b200.hubert import HubertWithKmeans

    ck, km = _files(tmp_path, g)
    with pytest.raises(ValueError, match="output_layer"):
        HubertWithKmeans(ck, km, output_layer=g["arch"]["encoder_layers"] + 1)


def test_cpu_input_raises(tmp_path, g):
    from audiolm_pytorch_b200._lib import AlmError
    from audiolm_pytorch_b200.hubert import HubertWithKmeans

    ck, km = _files(tmp_path, g)
    with pytest.raises(AlmError):
        HubertWithKmeans(ck, km, output_layer=1)(g["waves"][0])


@pytest.mark.parametrize("form", ["weight_g", "parametrizations"])
def test_pos_conv_fold_matches_oracle(g, form):
    from audiolm_pytorch_b200.hubert import fold_pos_conv_weight

    st = g["state"] if form == "weight_g" else oh.parametrized_weight_norm(g["state"])
    ref = oh.pos_conv_weight({k: v.double() for k, v in st.items()})
    assert torch.allclose(fold_pos_conv_weight(st).double(), ref, rtol=1e-6, atol=0)
