"""Host checks of the residual VQ's `rq_kwargs` (cosine-similarity and low-dimensional codebooks).

* SoundStream's residual VQ accepts `use_cosine_sim`, `codebook_dim` and the kwargs that only shape training, and
  refuses every other one by name; projections outside the envelope are refused at construction.
* State-dict keys follow the restated upstream module (oracle/rvq_options.py), and save / load /
  init_and_load_from round-trip the configuration and the projection weights.
* The oracle (oracle/rvq_options.py) reproduces tests/golden/rvq_options.pt, which the
  reference's soundstream.py wrote.
* With the C entry points replaced by a recorder, the default quantizer launches exactly what it launched before
  these options existed, and the new configurations reach only the new entry points and the GEMM.
"""

import pickle

import pytest
import torch

from oracle import golden
from oracle import rvq_options as ro

TRAINING_KWARGS = dict(decay=0.9, eps=1e-5, commitment_weight=0.5, kmeans_init=False, kmeans_iters=5, sync_kmeans=False,
                       threshold_ema_dead_code=1, stochastic_sample_codes=True, sample_codebook_temp=0.5,
                       straight_through=True, rotation_trick=False, reinmax=True, orthogonal_reg_weight=0.1,
                       orthogonal_reg_active_codes_only=True, orthogonal_reg_max_codes=64,
                       codebook_diversity_loss_weight=0.1, codebook_diversity_temperature=10.0, sync_codebook=False,
                       ema_update=False, learnable_codebook=True, commitment_use_cross_entropy_loss=True,
                       quantize_dropout_multiple_of=2, quantize_dropout_cutoff_index=0)
# SoundStream passes these itself (from its rq_* arguments), as the reference does
PASSED_BY_SOUNDSTREAM = {"decay", "commitment_weight", "quantize_dropout_multiple_of", "kmeans_init",
                         "threshold_ema_dead_code", "quantize_dropout", "quantize_dropout_cutoff_index",
                         "stochastic_sample_codes", "rotation_trick"}
REFUSED_KWARGS = dict(heads=2, shared_codebook=True, affine_param=True, implicit_neural_codebook=True, beam_size=4,
                      eval_beam_size=4, separate_codebook_per_head=True, use_cosine_similarity=True, channel_last=False)


def _ss(**kw):
    from audiolm_pytorch_b200.soundstream import SoundStream

    return SoundStream(**{**dict(channels=4, codebook_dim=32, codebook_size=64, rq_num_quantizers=3,
                                 use_local_attn=False), **kw})


# ---- kwarg validation ------------------------------------------------------------------------------------------------
def test_training_kwargs_accepted_together():
    kw = {k: v for k, v in TRAINING_KWARGS.items() if k not in PASSED_BY_SOUNDSTREAM}
    ss = _ss(rq_kwargs=dict(kw, use_cosine_sim=True, codebook_dim=16))
    rvq = ss.rq.rvqs[0]
    assert rvq.use_cosine_sim and rvq.codebook_dim == 16 and rvq.layers[0]._codebook.embed.shape == (1, 64, 16)


@pytest.mark.parametrize("name", sorted(TRAINING_KWARGS))
def test_training_kwarg_accepted(name):
    from audiolm_pytorch_b200.soundstream import GroupedResidualVQ

    rq = GroupedResidualVQ(dim=32, num_quantizers=3, codebook_size=64, groups=2, **{name: TRAINING_KWARGS[name]})
    assert not rq.rvqs[0].use_cosine_sim and not rq.rvqs[0].projected
    if name not in PASSED_BY_SOUNDSTREAM:
        assert not _ss(rq_kwargs={name: TRAINING_KWARGS[name]}).rq.rvqs[0].projected


@pytest.mark.parametrize("name", sorted(REFUSED_KWARGS))
def test_other_kwargs_refused_by_residual_vq(name):
    from audiolm_pytorch_b200.soundstream import ResidualVQ

    with pytest.raises(NotImplementedError, match=name):
        ResidualVQ(dim=32, num_quantizers=3, codebook_size=64, **{name: REFUSED_KWARGS[name]})


@pytest.mark.parametrize("name", sorted(REFUSED_KWARGS))
def test_other_kwargs_refused_by_name(name):
    with pytest.raises(NotImplementedError, match=name):
        _ss(rq_kwargs={name: REFUSED_KWARGS[name]})


def test_tuple_codebook_size_refused():
    with pytest.raises(NotImplementedError, match="codebook_size"):
        _ss(codebook_size=(64, 64))


def test_kwargs_the_reference_passes_stay_theirs():
    """rq_kwargs may not repeat a kwarg SoundStream already passes (the reference raises TypeError too)"""
    with pytest.raises(TypeError):
        _ss(rq_kwargs=dict(decay=0.9, kmeans_init=False))   # kmeans_init is always passed


@pytest.mark.parametrize("dim, groups, dc", [(32, 1, 12), (36, 1, 8), (40, 2, 8), (32, 1, 4), (20, 1, 16)])
def test_projection_envelope_refused(dim, groups, dc):
    """widths of the projection not multiples of 8 are refused at construction, naming them"""
    with pytest.raises(NotImplementedError, match=f"{dim // groups} -> {dc}"):
        _ss(codebook_dim=dim, rq_groups=groups, rq_kwargs=dict(codebook_dim=dc))


@pytest.mark.parametrize("dim, dc", [(32, 8), (32, 16), (32, 32), (50, 50), (64, 128)])
def test_projection_envelope_accepted(dim, dc):
    rvq = _ss(codebook_dim=dim, rq_kwargs=dict(codebook_dim=dc)).rq.rvqs[0]
    assert rvq.projected == (dim != dc)


def test_default_builds_as_before():
    ss = _ss()
    rvq = ss.rq.rvqs[0]
    assert not rvq.use_cosine_sim and not rvq.projected
    assert isinstance(rvq.project_in, torch.nn.Identity) and isinstance(rvq.project_out, torch.nn.Identity)
    assert not any("project" in k for k in ss.state_dict())


def test_fp32_search_refuses_the_new_options(monkeypatch):
    from audiolm_pytorch_b200 import soundstream

    monkeypatch.setattr(soundstream, "RVQ_ON_TENSOR_CORES", False)
    for kw in (dict(use_cosine_sim=True), dict(codebook_dim=8)):
        ss = _ss(rq_kwargs=kw).eval()
        for rvq in ss.rq.rvqs:
            for layer in rvq.layers:
                layer._codebook.initted.fill_(1)
        with pytest.raises(NotImplementedError, match="tensor-core"):
            ss.rq(torch.randn(1, 4, 32))


# ---- state dict and checkpoints --------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw", [dict(use_cosine_sim=True), dict(codebook_dim=8), dict(codebook_dim=8, use_cosine_sim=True),
                                dict(codebook_dim=64)])
@pytest.mark.parametrize("groups", [1, 2])
def test_state_dict_keys_match_the_oracle(kw, groups):
    ss = _ss(rq_groups=groups, rq_kwargs=kw)
    mine = {k[3:]: tuple(v.shape) for k, v in ss.state_dict().items() if k.startswith("rq.")}
    ref = ro.GroupedResidualVQ(dim=32, groups=groups, num_quantizers=3, codebook_size=64, **kw)
    assert mine == {k: tuple(v.shape) for k, v in ref.state_dict().items()}
    if kw.get("codebook_dim", 32 // groups) != 32 // groups:
        assert "rvqs.1.project_out.bias" in mine if groups == 2 else "rvqs.0.project_in.weight" in mine


def test_init_and_load_from_round_trip(tmp_path):
    from audiolm_pytorch_b200.soundstream import SoundStream

    torch.manual_seed(0)
    kw = dict(use_cosine_sim=True, codebook_dim=8, kmeans_iters=3)
    ss = _ss(rq_groups=2, rq_kwargs=kw)
    with torch.no_grad():
        for p_ in ss.rq.parameters():
            p_.normal_()
    path = tmp_path / "ss.pt"
    ss.save(path)
    back = SoundStream.init_and_load_from(path)
    assert back.configs["rq_kwargs"] == kw and pickle.loads(back._configs)["rq_groups"] == 2
    a, b = ss.state_dict(), back.state_dict()
    assert a.keys() == b.keys() and all(torch.equal(a[k], b[k]) for k in a)
    other = _ss(rq_groups=2, rq_kwargs=kw)
    other.load(path)
    assert torch.equal(other.rq.rvqs[1].project_out.weight, ss.rq.rvqs[1].project_out.weight)


# ---- the golden against the oracle -----------------------------------------------------------------------------------
G = golden.load("rvq_options.pt")


@pytest.mark.parametrize("name", sorted(G))
def test_oracle_reproduces_golden(name):
    g = G[name]
    st = {**ro.seeded_state(g["keys"], g["seed"]), **{f"rq.{k}": v for k, v in g["rq_state"].items()}}
    enc, quant, ids = ro.soundstream_tokenize(g["kwargs"], st, g["wave"])
    b, n = enc.shape[:2]
    assert torch.equal(ids.permute(1, 2, 0, 3).reshape(b, n, -1), g["ids"])
    assert (enc - g["enc"]).abs().max() <= 1e-5 * max(1.0, g["enc"].abs().max().item())
    assert (quant - g["quant"]).abs().max() <= 1e-5 * max(1.0, g["quant"].abs().max().item())
    recon = ro.soundstream_decode_indices(g["kwargs"], st, ids)
    assert (recon - g["recon_idx"]).abs().max() <= 1e-5 * max(1.0, g["recon_idx"].abs().max().item())
    # the product's module tree takes the same state strictly
    from audiolm_pytorch_b200.soundstream import SoundStream

    SoundStream(**g["kwargs"]).load_state_dict(
        {k: v for k, v in st.items() if k.split(".")[0] in ("encoder", "decoder", "rq")}, strict=True)


def test_golden_covers_the_configurations():
    assert sorted(G) == sorted(f"{c}/{q}" for c in ("tiny", "tc") for q in ("cosine", "proj8", "cosine_proj8_g2"))
    for name, g in G.items():
        kw = g["kwargs"]["rq_kwargs"]
        assert kw.get("use_cosine_sim", False) == ("cosine" in name)
        if name == "tc/cosine_proj8_g2":
            assert kw["codebook_dim"] == 16 and g["kwargs"]["rq_groups"] == 2
        emb = g["rq_state"]["rvqs.0.layers.0._codebook.embed"][0]
        assert not torch.allclose(emb.norm(dim=1), torch.ones(emb.shape[0]), atol=1e-2), "codebooks are not unit norm"


def test_cosine_oracle_rule():
    """argmax of F.normalize(r) . e on the stored rows, lowest index on ties, code 0 for a zero row"""
    e = torch.tensor([[1.0, 0.0], [2.0, 0.0], [0.0, 3.0], [2.0, 0.0]])
    x = torch.tensor([[0.0, 0.0], [5.0, 0.1], [0.1, 1.0]])
    assert ro.cosine_nearest(x, e).tolist() == [0, 1, 2]
    _, ids = ro.cosine_search_fp64(x, e[None])
    assert ids[:, 0].tolist() == [0, 1, 2]


# ---- launches --------------------------------------------------------------------------------------------------------
@pytest.fixture
def launches(monkeypatch):
    """the C entry points replaced by a recorder of (name, scalar arguments); ops run on CPU tensors"""
    from audiolm_pytorch_b200 import _lib, ops

    seen = []

    def record(name, *a):
        seen.append((name, tuple(v if isinstance(v, (int, float)) else tuple(v.shape) if torch.is_tensor(v) else None
                                  for v in a)))

    monkeypatch.setattr(_lib, "call", record)
    monkeypatch.setattr(ops, "_check_cuda", lambda *ts: None)
    return seen


def _run(ss):
    ss = ss.eval()
    for rvq in ss.rq.rvqs:
        for layer in rvq.layers:
            layer._codebook.initted.fill_(1)
            layer._codebook.embed.normal_()
    with torch.no_grad():
        ss.rq(torch.randn(2, 5, ss.codebook_dim))
        ss.rq.get_output_from_indices(torch.zeros(ss.rq_groups, 2, 5, 3, dtype=torch.long))


def _expected_default(N, D, C, Q, groups):
    """what the default quantizer launched before rq_kwargs reached it: per group pack, prepare, Q x (GEMM, select),
    then decode"""
    Dg = D // groups
    Dp = -(-Dg // 8) * 8
    out = []
    for _ in range(groups):
        out += [("alm_rvq_pack_codebooks", (Q * C, Dp)), ("alm_rvq_prepare", (N, Dg, Dp))]
        for q in range(Q):
            out += [("alm_gemm_bf16", (N, C, 3 * Dp)), ("alm_rvq_select", (N, Dp, C, int(q + 1 < Q)))]
    return out + [("alm_rvq_decode", (N, Dg, C, Q))] * groups


def _summary(seen):
    keep = {"alm_rvq_pack_codebooks": (3, 4), "alm_rvq_prepare": (6, 7, 8), "alm_gemm_bf16": (12, 13, 14),
            "alm_rvq_select": (10, 11, 12, 13), "alm_rvq_decode": (5, 6, 7, 8)}
    return [(n, tuple(a[i] for i in keep[n])) if n in keep else (n, None) for n, a in seen]


@pytest.mark.parametrize("D, groups", [(32, 1), (50, 1), (64, 2), (512, 1)])
def test_default_launches_unchanged(launches, D, groups):
    _run(_ss(codebook_dim=D, rq_groups=groups))
    assert _summary(launches) == _expected_default(10, D, 64, 3, groups)


@pytest.mark.parametrize("kw, groups", [(dict(use_cosine_sim=True), 1), (dict(codebook_dim=8), 1),
                                        (dict(use_cosine_sim=True, codebook_dim=8), 2)])
def test_option_launches(launches, kw, groups):
    _run(_ss(rq_groups=groups, rq_kwargs=kw))
    names = [n for n, _ in launches]
    cos, proj = kw.get("use_cosine_sim", False), "codebook_dim" in kw
    assert ("alm_rvq_select_cos" in names) == cos and ("alm_rvq_select" in names) == (not cos)
    assert ("alm_rvq_prepare_cos" in names) == cos and ("alm_rvq_prepare" in names) == (not cos)
    # per group: split rows + GEMM for project_in and project_out in the encode, project_out in the decode
    assert names.count("alm_split_rows") == (3 * groups if proj else 0)
    assert names.count("alm_gemm_bf16") == groups * (3 + (3 if proj else 0))
    assert "alm_rvq_encode" not in names
