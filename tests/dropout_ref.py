"""Test references for dropout: a numpy restatement of the library's dropout mask keep(seed, site, row, col)
(csrc/alm_common.cuh), and an fp32 restatement of the transformer stack that applies given masks.

Philox4x32-10 keyed by the 64-bit seed; one draw decides the 8 elements rows {i0, i0+1, i0+8, i0+9} x cols {j0, j0+8}
(i0 % 16 in {0, 2, 4, 6}, j0 % 16 < 8) through the counter (row / 16, col / 16, site, 8 ((row % 8) / 2) + col % 8);
row i0 + r1 + 8 r8 reads word r1 + 2 r8, col j0 + 8 c8 its low (c8 = 0) or high 16 bits; keep iff that 16-bit
uniform < round(65536 (1 - p)).
"""
import numpy as np

_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)
_LO = np.uint64(0xFFFFFFFF)
_S32 = np.uint64(32)


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Philox4x32 with 10 rounds on uint64 arrays holding 32-bit values -> the four output words."""
    c0, c1, c2, c3 = (np.asarray(c, dtype=np.uint64) for c in (c0, c1, c2, c3))
    k0, k1 = np.uint64(k0), np.uint64(k1)
    for _ in range(10):
        p0, p1 = _M0 * c0, _M1 * c2
        c0, c1, c2, c3 = (p1 >> _S32) ^ c1 ^ k0, p1 & _LO, (p0 >> _S32) ^ c3 ^ k1, p0 & _LO
        k0, k1 = (k0 + _W0) & _LO, (k1 + _W1) & _LO
    return c0, c1, c2, c3


def keep_threshold(p):
    """the kernels' 16-bit threshold: p is a C float, 1 - p is taken in double"""
    return int((1.0 - float(np.float32(p))) * 65536.0 + 0.5)


def keep(seed, site, rows, cols, p):
    """bool array: keep(seed, site, rows[:, None], cols[None, :]) for 1-D index arrays rows, cols"""
    r = np.asarray(rows, dtype=np.uint64)[:, None]
    c = np.asarray(cols, dtype=np.uint64)[None, :]
    r, c = np.broadcast_arrays(r, c)
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    w = philox4x32_10(r >> np.uint64(4), c >> np.uint64(4), np.full(r.shape, site, dtype=np.uint64),
                      ((r & np.uint64(7)) >> np.uint64(1)) * np.uint64(8) + (c & np.uint64(7)),
                      seed & 0xFFFFFFFF, seed >> 32)
    idx = (r & np.uint64(1)) + np.uint64(2) * ((r >> np.uint64(3)) & np.uint64(1))
    word = np.choose(idx.astype(np.int64), w)
    u = np.where((c >> np.uint64(3)) & np.uint64(1), word >> np.uint64(16), word & np.uint64(0xFFFF))
    return u < np.uint64(keep_threshold(p))


# ---- fp32 restatement of the transformer stack with given dropout masks (training-mode forward) -----------------
# Built from the oracle's blocks (oracle/transformer.py); the masks are multiplicative factors (0 or 1/(1-p)) at the
# reference's three dropout sites: attention probabilities (attend.py:139-140), Attention.to_out[1]
# (audiolm_pytorch.py:302-305) and the FeedForward Dropout after the inner LayerNorm (audiolm_pytorch.py:256).
def _attend(q, k, v, mask, attn_bias, p_mask):
    import torch
    from oracle.transformer import NEG

    sim = torch.einsum("bhid,bjd->bhij", q, k) * q.shape[-1] ** -0.5
    if attn_bias is not None:
        sim = sim + attn_bias
    if mask is not None:
        sim = sim.masked_fill(~mask[:, None, None, :], NEG(sim.dtype))
    i, j = sim.shape[-2:]
    sim = sim.masked_fill(torch.ones(i, j, dtype=torch.bool, device=q.device).triu(j - i + 1), NEG(sim.dtype))
    attn = sim.softmax(-1)
    if p_mask is not None:
        attn = attn * p_mask
    return torch.einsum("bhij,bjd->bhid", attn, v)


def _attention(st, x, heads, mask, attn_bias, value_residual, p_mask, out_mask):
    from oracle.transformer import layer_norm

    xn = layer_norm(x, st["norm.gamma"])
    q = xn @ st["to_q.weight"].t()
    k, v = (x @ st["to_kv.weight"].t()).chunk(2, dim=-1)   # keys / values from the un-normalised input
    orig_v = v
    if value_residual is not None:
        v = 0.5 * (v + value_residual)
    b, n, _ = q.shape
    o = _attend(q.reshape(b, n, heads, -1).permute(0, 2, 1, 3), k, v, mask, attn_bias, p_mask)
    out = o.permute(0, 2, 1, 3).reshape(b, n, -1) @ st["to_out.0.weight"].t()
    if out_mask is not None:
        out = out * out_mask
    return out, orig_v


def _feed_forward(st, x, ff_mask):
    import torch.nn.functional as F
    from oracle.transformer import layer_norm

    a, gate = (layer_norm(x, st["0.gamma"]) @ st["1.weight"].t()).chunk(2, dim=-1)
    g = layer_norm(F.gelu(gate) * a, st["3.gamma"])
    if ff_mask is not None:
        g = g * ff_mask
    return g @ st["5.weight"].t()


def transformer_with_dropout(st, x, *, heads, depth, num_streams, dropout_masks, self_attn_mask=None,
                             add_value_residual=True):
    """oracle.transformer.transformer (no KV cache) with per-layer masks (probabilities [b h n n], attention output
    [b n d], feed-forward [b n inner]); returns the normed output [b n d]."""
    from oracle.transformer import hyper_depth, hyper_width, layer_norm, rel_pos_bias, sub

    n = x.shape[1]
    attn_bias = rel_pos_bias(sub(st, "rel_pos_bias"), n, n) if "rel_pos_bias.net.0.0.weight" in st else None
    if num_streams > 1:
        x = x.repeat_interleave(num_streams, dim=0)
    value_res = None
    for i in range(depth):
        a_st, f_st = sub(st, f"layers.{i}.0"), sub(st, f"layers.{i}.2")
        p_mask, out_mask, ff_mask = dropout_masks[i]
        xin, mixed, beta = hyper_width(a_st, x, num_streams) if num_streams > 1 else (x, None, None)
        out, values = _attention(sub(a_st, "branch"), xin, heads, self_attn_mask, attn_bias, value_res, p_mask,
                                 out_mask)
        x = hyper_depth(out, mixed, beta) if num_streams > 1 else x + out
        if add_value_residual and value_res is None:
            value_res = values
        xin, mixed, beta = hyper_width(f_st, x, num_streams) if num_streams > 1 else (x, None, None)
        out = _feed_forward(sub(f_st, "branch"), xin, ff_mask)
        x = hyper_depth(out, mixed, beta) if num_streams > 1 else x + out
    if num_streams > 1:
        x = x.reshape(x.shape[0] // num_streams, num_streams, *x.shape[1:]).sum(dim=1)
    return layer_norm(x, st["norm.gamma"])
