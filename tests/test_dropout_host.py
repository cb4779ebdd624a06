"""Dropout configuration of the transformers (no GPU): construction, state-dict keys, argument checks, and the
counter-based mask generator's reference restatement."""
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
import dropout_ref  # noqa: E402


def _models(p):
    from audiolm_pytorch_b200.audiolm import CoarseTransformer, FineTransformer, SemanticTransformer

    kw = dict(dim=64, depth=2, heads=2, attn_dropout=p, ff_dropout=p)
    torch.manual_seed(0)
    return [
        SemanticTransformer(num_semantic_tokens=50, **kw),
        CoarseTransformer(num_semantic_tokens=50, codebook_size=64, num_coarse_quantizers=2, **kw),
        FineTransformer(num_coarse_quantizers=2, num_fine_quantizers=2, codebook_size=64, **kw),
    ]


def test_transformers_construct_with_dropout_and_keep_state_dict_keys():
    for m0, m1 in zip(_models(0.0), _models(0.1)):
        assert list(m1.state_dict().keys()) == list(m0.state_dict().keys())
        tr = m1.transformer
        for attn, _, ff in tr.layers:
            assert attn.branch.attend.dropout == 0.1 and attn.branch.to_out[1].p == 0.1
            assert getattr(ff.branch, "4").p == 0.1
        m1.load_state_dict(m0.state_dict(), strict=True)


@pytest.mark.parametrize("p", [1.0, -0.1, 1.5])
@pytest.mark.parametrize("which", ["attn_dropout", "ff_dropout"])
def test_dropout_out_of_range_raises(p, which):
    from audiolm_pytorch_b200.audiolm import SemanticTransformer

    with pytest.raises(ValueError):
        SemanticTransformer(num_semantic_tokens=50, dim=64, depth=1, heads=2, **{which: p})


def test_dropout_plan_draws_nothing_when_off():
    """eval() or p == 0: no seed is drawn (the CPU generator does not move) and no layer gets a dropout site."""
    from audiolm_pytorch_b200.transformer import Transformer

    torch.manual_seed(1)
    tr0 = Transformer(dim=64, depth=2, heads=2).train()
    tr1 = Transformer(dim=64, depth=2, heads=2, attn_dropout=0.1, ff_dropout=0.2).eval()
    state = torch.get_rng_state()
    assert tr0._dropout_plan() is None and tr1._dropout_plan() is None
    assert torch.equal(torch.get_rng_state(), state)
    tr1.train()
    torch.manual_seed(5)
    plan = tr1._dropout_plan()
    torch.manual_seed(5)
    assert tr1._dropout_plan() == plan
    seeds = {s for layer in plan for (_, s, _) in layer}
    sites = [site for layer in plan for (_, _, site) in layer]
    assert len(seeds) == 1 and sorted(sites) == list(range(6))
    assert [p for (p, _, _) in plan[0]] == [0.1, 0.1, 0.2]


def test_philox_known_answers():
    """Philox4x32-10 known-answer vectors (Salmon et al., Random123)."""
    cases = [
        ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
        ((0xFFFFFFFF,) * 4, (0xFFFFFFFF, 0xFFFFFFFF), (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
        ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
         (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
    ]
    for ctr, key, want in cases:
        got = dropout_ref.philox4x32_10(*ctr, *key)
        assert tuple(int(w) for w in got) == want


def test_reference_mask_statistics():
    """the restated mask keeps 1 - p of a block, exactly (to 2^-16) in expectation"""
    rows, cols = np.arange(512), np.arange(512)
    for p in (0.1, 0.5):
        k = dropout_ref.keep(1234, 7, rows, cols, p)
        n = k.size
        assert abs(k.mean() - (1 - p)) < 5 * np.sqrt(p * (1 - p) / n)
        assert abs(dropout_ref.keep_threshold(p) / 65536 - (1 - p)) <= 2 ** -17
    a = dropout_ref.keep(1, 0, rows, cols, 0.5)
    b = dropout_ref.keep(1, 1, rows, cols, 0.5)
    c = dropout_ref.keep(2, 0, rows, cols, 0.5)
    n = a.size
    for x, y in ((a, b), (a, c)):
        assert abs(np.corrcoef(x.ravel(), y.ravel())[0, 1]) < 5 / np.sqrt(n)


@pytest.mark.parametrize("num_streams", [1, 4])
@pytest.mark.parametrize("flash", [True, False])
def test_stack_restatement_matches_oracle_without_dropout(num_streams, flash):
    """the masked restatement used by the GPU tests, given masks of ones, is the oracle's transformer"""
    from audiolm_pytorch_b200.transformer import Transformer
    from oracle import transformer as ot

    torch.manual_seed(3)
    tr = Transformer(dim=64, depth=2, heads=2, flash_attn=flash, num_residual_streams=num_streams)
    st = {k: v.detach().float() for k, v in tr.state_dict().items()}
    b, n = 2, 20
    x = torch.randn(b, n, 64)
    inner = tr.layers[0][2].branch.inner
    ones = [(torch.ones(b, 2, n, n), torch.ones(b, n, 64), torch.ones(b, n, inner))] * 2
    got = dropout_ref.transformer_with_dropout(st, x, heads=2, depth=2, num_streams=num_streams, dropout_masks=ones)
    want, _ = ot.transformer(st, x, heads=2, depth=2, num_streams=num_streams)
    torch.testing.assert_close(got, want, rtol=1e-5, atol=1e-5)
    none = [(None, None, None)] * 2
    assert torch.equal(dropout_ref.transformer_with_dropout(st, x, heads=2, depth=2, num_streams=num_streams,
                                                            dropout_masks=none), want)
