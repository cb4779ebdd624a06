"""CPU: hyper-connections with 2 to 8 residual streams — the per-token aux row, the supported range, the state-dict
surface against the reference and the oracle against the goldens of tests/golden/streams.pt."""
import pytest
import torch

from oracle import golden
from oracle import transformer as ot

KEYS = ["semantic_s2", "semantic_s3", "semantic_s8", "coarse_s2"]


def close(a, b, tol=2e-4):
    return (a.float() - b.float()).abs().max().item() <= tol * max(1.0, b.float().abs().max().item())


def test_aux_row_floats():
    from audiolm_pytorch_b200 import ops

    assert ops.hc_aux_floats(4) == ops.HC_AUX == 56
    for S in range(ops.HC_MIN_STREAMS, ops.HC_MAX_STREAMS + 1):
        n = ops.hc_aux_floats(S)
        # ta[S(S+1)] tb[S] inv[S] z[S(S+1)+S], then at least mean and rstd, in whole 16-B bulk-copy units
        assert n % 4 == 0 and 2 * S * (S + 1) + 3 * S + 2 <= n < 2 * S * (S + 1) + 3 * S + 2 + 4 + 2


@pytest.mark.parametrize("S", [0, 9, 16])
def test_unsupported_stream_counts_raise(S):
    from audiolm_pytorch_b200.transformer import Transformer

    with pytest.raises(NotImplementedError, match="2..8"):
        Transformer(dim=64, depth=1, heads=2, num_residual_streams=S)


@pytest.mark.parametrize("S", [2, 3, 5, 8])
def test_supported_stream_counts_construct(S):
    from audiolm_pytorch_b200.transformer import Transformer

    tr = Transformer(dim=64, depth=1, heads=2, num_residual_streams=S)
    assert tr.layers[0][0].static_alpha.shape == (S, S + 1)
    assert tr.layers[0][2].dynamic_alpha_fn.shape == (64, S + 1)


@pytest.mark.parametrize("key", KEYS)
def test_state_dict_keys_match_reference_streams(key):
    from audiolm_pytorch_b200 import audiolm

    g = golden.load("streams.pt")[key]
    cls = audiolm.SemanticTransformer if g["kind"] == "semantic" else audiolm.CoarseTransformer
    m = cls(**g["kwargs"])
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == {k: tuple(v.shape) for k, v in g["state"].items()}
    m.load_state_dict(g["state"], strict=True)


@pytest.mark.parametrize("key", KEYS)
def test_oracle_reproduces_streams_golden(key):
    g = golden.load("streams.pt")[key]
    kw = g["kwargs"]
    S = kw["num_residual_streams"]
    if g["kind"] == "semantic":
        hk = dict(heads=kw["heads"], depth=kw["depth"], num_streams=S)
        assert close(ot.semantic_forward(g["state"], g["ids"], **hk)[0], g["logits"])
        assert close(ot.semantic_forward(g["state"], g["ids"], self_attn_mask=g["mask"], **hk)[0], g["logits_masked"])
    else:
        hk = dict(heads=kw["heads"], depth=kw["depth"], codebook_size=kw["codebook_size"],
                  num_coarse_quantizers=kw["num_coarse_quantizers"], num_streams=S)
        (sl, cl), _ = ot.coarse_forward(g["state"], g["sem"], g["coarse"], **hk)
        assert close(sl, g["sem_logits"]) and close(cl, g["coarse_logits"])
        (_, clm), _ = ot.coarse_forward(g["state"], g["sem"], g["coarse"], self_attn_mask=g["mask"], **hk)
        assert close(clm, g["coarse_logits_masked"])
