"""The decode engine's bias rule (alm_decode_bias_row) against the dense bias path's table indices, on the CPU.

For every query position L the slow KV-cache path would decode, and every key j <= L, the per-position coordinates
(u, cls, c) of the models' `decode_bias_coords` must select the same table entry (or the same per-head override) as
the dense index of the full sequence the slow path builds at that length: `RelativePositionBias.index`,
`CoarseTransformer._cross_index` and `FineTransformer._pos_bias_index`."""

import pytest
import torch


def rule_index(u, cls, c, L):
    """table row per key j <= L, -1 where the rule takes the override (what alm_decode_bias_row computes)"""
    u, cls = u.long(), cls.long()
    idx = u[L] - u[:L + 1] + c
    over = (cls[:L + 1] != cls[L]) | (cls[L] < 0)
    return torch.where(over, torch.full_like(idx, -1), idx)


def small(cls_name, **kw):
    from audiolm_pytorch_b200 import audiolm

    return getattr(audiolm, cls_name)(dim=32, depth=1, heads=2, **kw)


@pytest.mark.parametrize("prompt,max_len", [(0, 256), (9, 256), (200, 512)])
def test_semantic_rule_matches_relative_position_index(prompt, max_len):
    m = small("SemanticTransformer", num_semantic_tokens=20)
    u, cls, c = m.decode_bias_coords(max_len)
    assert u.dtype == cls.dtype == torch.int32 and u.shape == cls.shape == (max_len,)
    rp = m.transformer.rel_pos_bias
    # the engine reads rp.table(max_len) (centre max_len - 1), the dense path rp.table(n) (centre n - 1): the same
    # MLP input (relative offset) means the same value
    for L in range(prompt + 1, min(prompt + 60, max_len)):
        n = L + 1
        dense = rp.index(n, n)[-1].long() - (n - 1)
        got = rule_index(u, cls, c, L)
        assert (got >= 0).all()
        assert torch.equal(got - (max_len - 1), dense), L
        assert int(got.max()) < 2 * max_len - 1


@pytest.mark.parametrize("n_sem,n_coarse,max_len", [(5, 0, 256), (12, 7, 256), (40, 3 * 30 + 2, 512)])
def test_coarse_rule_matches_cross_index(n_sem, n_coarse, max_len):
    """n_coarse % 3 != 0: a primed coarse sequence ending in a remainder frame"""
    m = small("CoarseTransformer", num_semantic_tokens=50, codebook_size=16, num_coarse_quantizers=3)
    u, cls, c = m.decode_bias_coords(n_sem, max_len)
    start = n_sem + 1 + n_coarse            # [sem start | n_sem | coarse start | n_coarse]: first query decoded here
    for L in range(start, min(start + 40, max_len)):
        n = L + 1
        idx = m._cross_index(n, n_sem + 1, "cpu")[-1].long()
        dense = torch.where(idx < 0, idx, idx - (n - 1))
        got = rule_index(u, cls, c, L)
        got = torch.where(got < 0, got, got - (max_len - 1))
        assert torch.equal(got, dense), L
    assert (rule_index(u, cls, c, start) < 0).sum() == n_sem + 1   # the whole semantic segment takes cross_attn_bias


@pytest.mark.parametrize("qc,qf,n_coarse,n_fine0", [(3, 5, 12, 0), (3, 5, 14, 0), (2, 3, 10, 6), (3, 5, 13, 10)])
def test_fine_rule_matches_pos_bias_index(qc, qf, n_coarse, n_fine0):
    """n_coarse % qc != 0: a padded last coarse frame; n_fine0 > 0: primed fine frames"""
    m = small("FineTransformer", num_coarse_quantizers=qc, num_fine_quantizers=qf, codebook_size=16)
    steps = n_coarse // qc
    n_fine = steps * qf                  # the fine length the generation reaches
    max_len = 256
    u, cls, c = m.decode_bias_coords(n_coarse, n_fine, max_len)
    _, mlp_in = m._pos_bias_index(n_coarse, n_fine, "cpu")
    rows = mlp_in.shape[0]
    for nf in range(n_fine0, n_fine):    # the sequence holds nf fine tokens; the query is its last position
        L = 1 + n_coarse + nf            # (nf == 0: the fine start token)
        idx, mlp_nf = m._pos_bias_index(n_coarse, nf, "cpu")
        assert torch.equal(mlp_nf, mlp_in), nf               # the dense table does not change during generation
        got = rule_index(u, cls, c, L)
        assert torch.equal(got, idx[-1].long()), nf
        assert int(got.max()) < rows
    # the rule also reproduces the full matrix of the longest sequence (every query row)
    idx, _ = m._pos_bias_index(n_coarse, n_fine, "cpu")
    for L in range(idx.shape[0]):
        assert torch.equal(rule_index(u, cls, c, L), idx[L, :L + 1].long()), L


def test_fine_coords_refuse_a_table_that_would_change():
    m = small("FineTransformer", num_coarse_quantizers=3, num_fine_quantizers=5, codebook_size=16)
    with pytest.raises(AssertionError):
        m.decode_bias_coords(6, 3 * 5, 256)     # 3 fine frames against 2 coarse frames
