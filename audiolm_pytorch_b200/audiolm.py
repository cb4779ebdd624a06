"""The three AudioLM transformers, their training / sampling wrappers and the AudioLM orchestrator.

Drop-in surface of /root/reference/audiolm_pytorch/audiolm_pytorch.py:564-2254 (same class names, keyword
arguments, return conventions and state_dict keys) for the configuration the hot path covers: both the
`flash_attn=True` path and the `flash_attn=False` path with its relative-position attention bias
(rel_pos.py), no text / audio conditioning.  Token bookkeeping (ids, masks, sampling loops) is host-side
torch; the transformer stack, heads, loss and sampler run in libalm_b200.
"""
from __future__ import annotations

from pathlib import Path

import torch
import torch.nn.functional as F
from torch import nn

from . import heads as _heads_mod
from .heads import (HeadCache, LazyLogits, cross_entropy, generate_mask_with_prob, gumbel_sample, mask_out_after_eos_id, top_k)
from . import ops
from .decode import StackDecoder, TokenDecoder
from .rel_pos import gather_bias, mlp_table
from .transformer import Transformer, default, exists

USE_DECODE_GRAPHS = True  # False: the decode engine runs its steps eagerly (debugging / A-B timing)

__version__ = "2.4.0"  # checkpoint 'version' field of the reference this surface mirrors

# encoder widths of the T5 checkpoints the reference can be pointed at (t5.py:49-63 reads them from HF)
T5_DIMS = {"google/t5-v1_1-small": 512, "google/t5-v1_1-base": 768, "google/t5-v1_1-large": 1024,
           "google/t5-v1_1-xl": 2048, "google/t5-v1_1-xxl": 4096}
DEFAULT_T5_NAME = "google/t5-v1_1-base"


def ceil_div(a, b):
    return -(-a // b)


def append_eos_id(ids, eos_id):
    return F.pad(ids, (0, 1), value=eos_id)


def batch_unique_consecutive(t, pad_value=0.0):
    """per-row torch.unique_consecutive + pad_sequence (audiolm_pytorch.py:162-164) without the per-row host loop:
    keep[i] = t[i] != t[i-1], destination column = running count of kept elements, one scatter.  The only host
    round-trip left is the padded width (the output shape depends on the data)."""
    b, n = t.shape
    if n == 0:
        return t
    keep = torch.ones_like(t, dtype=torch.bool)
    keep[:, 1:] = t[:, 1:] != t[:, :-1]
    dest = keep.cumsum(dim=-1) - 1                       # column of each kept element
    width = int(keep.sum(dim=-1).max())
    out = torch.full((b, width + 1), pad_value, dtype=t.dtype, device=t.device)
    out.scatter_(1, torch.where(keep, dest, torch.full_like(dest, width)), t)  # dropped elements land in a spare column
    return out[:, :width]


def get_embeds(embeddings: nn.Embedding, codes, pad_id=-1, return_mask=False, mask_pad_pos_to=0):
    pad = codes == pad_id
    out = embeddings(codes.masked_fill(pad, 0))
    if exists(mask_pad_pos_to):
        out = out.masked_fill(pad[..., None], mask_pad_pos_to)
    return (out, ~pad) if return_mask else out


def _tile_rows(weight, n):
    """weight[(arange(n) % q)] as repeat + slice (audiolm_pytorch.py:903-905 does the same with einops.repeat): the
    backward is a strided sum instead of an index_put scatter over batch x positions."""
    q = weight.shape[0]
    return weight.repeat(ceil_div(n, q), 1)[:n]


def _rel_coords(cls):
    """(u, cls, c) of a relative-position bias over cache positions 0..max_len-1 (max_len = cls.shape[0]): u = t and
    c = max_len - 1, i.e. table row (L - j) + max_len - 1 of `RelativePositionBias.table(max_len)`."""
    max_len = cls.shape[0]
    return torch.arange(max_len, dtype=torch.int32, device=cls.device), cls, max_len - 1


def _pos_mlp_in(max_seq, rel_off, dev):
    """fp32 [(2 max_seq - 1) rel_off, 2] inputs of the fine transformer's pos_bias_mlp: (row // rel_off, row % rel_off)
    of every table row (the reference feeds the shifted, non-negative coordinates, :1278-1290)."""
    rows = torch.arange((2 * max_seq - 1) * rel_off, device=dev)
    return torch.stack((rows // rel_off, rows % rel_off), dim=-1).float()


def _quantizer_ids(n, q, device):
    return torch.arange(n, device=device) % q


class _EmbedGatherFn(torch.autograd.Function):
    """tokens [M, d] = sum of up to two rows of the parameter tables per position (alm_embed_gather); the backward is one
    vector-reduction scatter into fresh gradient tables (alm_embed_scatter) instead of a sort-based
    embedding_dense_backward per table."""

    @staticmethod
    def forward(ctx, src, d, *tables):
        flat = [t.detach().reshape(-1, d).float().contiguous() for t in tables]
        ctx.src, ctx.d, ctx.shapes = src, d, [t.shape for t in tables]
        return ops.embed_gather(src, flat, d)

    @staticmethod
    def backward(ctx, dout):
        d = ctx.d
        grads = [torch.zeros(shape, device=dout.device, dtype=torch.float32) for shape in ctx.shapes]
        ops.embed_scatter(ctx.src, [g.view(-1, d) for g in grads], dout.contiguous().float())
        return (None, None, *grads)


def _src(table_id, rows):
    """source-list entry (table_id << 24) | row for int64 row indices (rows < 0 stay -1 = no contribution)"""
    return torch.where(rows >= 0, rows + (table_id << 24), torch.full_like(rows, -1))


def _gather_tokens(src0, src1, tables, d):
    """src0 / src1 int64 [b, n] source lists -> tokens fp32 [b, n, d]"""
    b, n = src0.shape
    src = torch.stack((src0, src1), dim=-1).to(torch.int32).reshape(b * n, 2).contiguous()
    return _EmbedGatherFn.apply(src, d, *tables).view(b, n, d)


class _deferred_heads:
    """while active (a wrapper computing its loss), the transformer returns heads.LazyLogits instead of logits tensors,
    so that cross_entropy() can run the fused head + CE kernels; the public forward signatures stay the reference's."""

    def __init__(self, transformer, on):
        self.tr, self.on = transformer, bool(on) and _heads_mod.FUSED_HEAD_CE

    def __enter__(self):
        self.tr._defer_heads = self.on

    def __exit__(self, *exc):
        self.tr._defer_heads = False
        return False


class _TokenTransformer(nn.Module):
    """Shared scaffolding: conditioning guard, text projection parameter (kept for checkpoint
    compatibility), checkpoint loading, classifier-free-guidance wrapper."""

    _defer_heads = False   # set by _deferred_heads around a wrapper's loss forward

    def _init_common(self, dim, t5_name, cond_dim, has_condition, audio_text_condition, cond_drop_prob):
        if has_condition or audio_text_condition:
            raise NotImplementedError("text / audio conditioning is outside the accelerated hot path")
        self.has_condition = False
        self.cond_drop_prob = cond_drop_prob
        text_dim = default(cond_dim, T5_DIMS.get(t5_name, 768))
        self.proj_text_embed = nn.Linear(text_dim, dim, bias=False) if text_dim != dim else nn.Identity()
        self._heads = HeadCache()

    def embed_text(self, *a, **k):
        raise NotImplementedError("T5 text conditioning is outside the accelerated hot path")

    @property
    def device(self):
        return next(self.parameters()).device

    def load(self, path):
        path = Path(path)
        assert path.exists()
        pkg = torch.load(str(path), map_location=self.device)
        self.load_state_dict(pkg["model"])
        return pkg

    def _no_text(self, text, text_embeds):
        assert not (exists(text) or exists(text_embeds)), "this build has has_condition=False"


class SemanticTransformer(_TokenTransformer):
    """audiolm_pytorch.py:564-724."""

    def __init__(self, *, dim, depth, num_semantic_tokens, heads=8, attn_dropout=0.0, ff_dropout=0.0,
                 t5_name=DEFAULT_T5_NAME, cond_dim=None, has_condition=False, audio_text_condition=False,
                 cond_as_self_attn_prefix=False, cond_drop_prob=0.5, grad_shrink_alpha=0.1, rel_pos_bias=True,
                 flash_attn=False, **kwargs):
        super().__init__()
        self._init_common(dim, t5_name, cond_dim, has_condition, audio_text_condition, cond_drop_prob)
        self.num_semantic_tokens = num_semantic_tokens
        self.start_token = nn.Parameter(torch.randn(dim))
        self.semantic_embedding = nn.Embedding(num_semantic_tokens + 1, dim)
        self.eos_id = num_semantic_tokens
        self.transformer = Transformer(dim=dim, depth=depth, heads=heads, attn_dropout=attn_dropout,
                                       ff_dropout=ff_dropout, grad_shrink_alpha=grad_shrink_alpha,
                                       rel_pos_bias=rel_pos_bias and not flash_attn, flash_attn=flash_attn, **kwargs)
        self.to_logits = nn.Linear(dim, num_semantic_tokens + 1)

    def forward_with_cond_scale(self, *args, cond_scale=3, kv_cache=None, return_kv_cache=False, **kwargs):
        cache = None if kv_cache is None else kv_cache[0]
        logits, new_cache = self.forward(*args, cond_drop_prob=0.0, kv_cache=cache, return_kv_cache=True, **kwargs)
        return (logits, new_cache[None]) if return_kv_cache else logits

    def decode_bias_coords(self, max_len, dev=None):
        """(u, cls, c) of the decode engine's bias rule (decode.StackDecoder.set_bias) for cache positions
        0..max_len-1: the relative-position bias of keys j <= L for the query at position L is table row
        u[L] - u[j] + c of `rel_pos_bias.table(max_len)`, the row RelativePositionBias.index picks in the dense path."""
        return _rel_coords(torch.zeros(max_len, dtype=torch.int32, device=dev))

    def decode_bias(self, max_len):
        """(table, override, u, cls, c) of the decode engine's bias for a cache of max_len positions, None without a
        relative-position bias (flash_attn=True)."""
        rp = self.transformer.rel_pos_bias
        if not exists(rp):
            return None
        u, cls, c = self.decode_bias_coords(max_len, self.device)
        return rp.table(max_len), None, u, cls, c

    def forward(self, *, ids=None, return_loss=False, text=None, text_embeds=None, self_attn_mask=None,
                cond_drop_prob=None, unique_consecutive=None, kv_cache=None, return_kv_cache=False):
        self._no_text(text, text_embeds)
        if return_loss:
            ids = ids[:, :-1]
        # [start token | embedding rows] in one gather launch (padding ids contribute nothing, audiolm_pytorch.py:166-187)
        zero = torch.zeros((ids.shape[0], 1), dtype=torch.long, device=ids.device)  # (ids may have 0 columns)
        src0 = torch.cat((_src(0, zero), _src(1, ids.long())), dim=1)
        tokens = _gather_tokens(src0, src0.new_full(src0.shape, -1), [self.start_token, self.semantic_embedding.weight],
                                self.start_token.shape[-1])
        if exists(self_attn_mask):
            self_attn_mask = F.pad(self_attn_mask, (1, 0), value=True)
        tokens, kv = self.transformer(tokens, self_attn_mask=self_attn_mask, kv_cache=kv_cache, return_kv_cache=True) \
            if (return_kv_cache or exists(kv_cache)) else (self.transformer(tokens, self_attn_mask=self_attn_mask), None)
        b, n, d = tokens.shape
        if self._defer_heads:   # the wrapper's loss path: head + cross entropy run fused, no logits tensor
            logits = LazyLogits(self._heads, tokens, self.to_logits.weight, self.to_logits.bias, "sem", False)
        else:
            logits = self._heads.linear(tokens.reshape(-1, d), self.to_logits.weight, self.to_logits.bias, "sem")
            logits = logits.view(b, n, -1)
        return (logits, kv) if return_kv_cache else logits


class CoarseTransformer(_TokenTransformer):
    """audiolm_pytorch.py:726-990."""

    def __init__(self, *, codebook_size, num_coarse_quantizers, dim, depth, num_semantic_tokens, heads=8,
                 attn_dropout=0.0, ff_dropout=0.0, t5_name=DEFAULT_T5_NAME, has_condition=False, cond_dim=None,
                 audio_text_condition=False, cond_as_self_attn_prefix=False, cond_drop_prob=0.5,
                 grad_shrink_alpha=0.1, project_semantic_logits=True, rel_pos_bias=True, flash_attn=False, **kwargs):
        super().__init__()
        self._init_common(dim, t5_name, cond_dim, has_condition, audio_text_condition, cond_drop_prob)
        self.num_semantic_tokens = num_semantic_tokens
        self.semantic_start_token = nn.Parameter(torch.randn(dim))
        self.coarse_start_token = nn.Parameter(torch.randn(dim))
        self.semantic_eos_id = num_semantic_tokens
        self.semantic_embedding = nn.Embedding(num_semantic_tokens + 1, dim)
        self.coarse_eos_id = codebook_size
        self.coarse_embedding = nn.Embedding(num_coarse_quantizers * (codebook_size + 1), dim)
        self.coarse_quantize_embedding = nn.Embedding(num_coarse_quantizers, dim)
        rel = rel_pos_bias and not flash_attn
        self.cross_attn_bias = nn.Parameter(torch.zeros(heads, 1, 1)) if rel else None
        self.transformer = Transformer(dim=dim, depth=depth, heads=heads, attn_dropout=attn_dropout,
                                       ff_dropout=ff_dropout, grad_shrink_alpha=grad_shrink_alpha,
                                       rel_pos_bias=rel, flash_attn=flash_attn, **kwargs)
        self._bias_idx = {}
        self.codebook_size = codebook_size
        self.num_coarse_quantizers = num_coarse_quantizers
        self.to_semantic_logits = nn.Linear(dim, num_semantic_tokens + 1) if project_semantic_logits else None
        self.coarse_logit_weights = nn.Parameter(torch.randn(num_coarse_quantizers, codebook_size + 1, dim))

    def forward_with_cond_scale(self, *args, cond_scale=3, return_kv_cache=False, kv_cache=None, embed_cache=None,
                                **kwargs):
        kv = None if kv_cache is None else kv_cache[0]
        emb = None if embed_cache is None else embed_cache[0]
        logits, (new_kv, new_emb) = self.forward(*args, cond_drop_prob=0.0, return_cache=True, kv_cache=kv,
                                                 embed_cache=emb, **kwargs)
        return (logits, (new_kv[None], new_emb[None])) if return_kv_cache else logits

    def decode_bias_coords(self, num_semantic, max_len, dev=None):
        """(u, cls, c) of the decode engine's bias rule for the sequence [semantic start | num_semantic semantic
        tokens | coarse start | coarse tokens ...] over cache positions 0..max_len-1: the relative-position row as
        `_cross_index`, and `cross_attn_bias` between the semantic segment (class 1) and the coarse one (class 2)."""
        t = torch.arange(max_len, device=dev)
        return _rel_coords(torch.where(t <= num_semantic, 1, 2).to(torch.int32))

    def decode_bias(self, num_semantic, max_len):
        """(table, override, u, cls, c) of the decode engine's bias (see decode_bias_coords), None on the flash path."""
        rp = self.transformer.rel_pos_bias
        if not exists(rp):
            return None
        u, cls, c = self.decode_bias_coords(num_semantic, max_len, self.device)
        return rp.table(max_len), self.cross_attn_bias.reshape(-1), u, cls, c

    def _cross_index(self, n, n_sem, dev):
        """table row per (i, j) as RelativePositionBias.index, -1 where exactly one of i, j is semantic."""
        key = (n, n_sem, str(dev))
        if self._bias_idx.get("key") != key:
            idx = self.transformer.rel_pos_bias.index(n, n).clone()
            is_sem = torch.arange(n, device=dev) < n_sem
            idx[is_sem[:, None] ^ is_sem[None, :]] = -1
            self._bias_idx = dict(key=key, idx=idx)
        return self._bias_idx["idx"]

    def forward(self, *, semantic_token_ids, coarse_token_ids, self_attn_mask=None, text=None, text_embeds=None,
                cond_drop_prob=None, return_only_coarse_logits=False, return_cache=False, kv_cache=None,
                embed_cache=None):
        self._no_text(text, text_embeds)
        dev = semantic_token_ids.device
        b = semantic_token_ids.shape[0]
        q = self.num_coarse_quantizers
        coarse_token_ids = coarse_token_ids.reshape(b, -1)
        semantic_token_ids = semantic_token_ids.reshape(b, -1)
        nc = coarse_token_ids.shape[-1]
        qid = _quantizer_ids(nc, q, dev)
        S = semantic_token_ids.shape[1]
        # the reference offsets ids by codebook_size (not codebook_size+1) per quantizer (:896-899)
        # [semantic start | semantic rows | coarse start | coarse rows + quantizer rows] in one gather launch
        zero = torch.zeros((b, 1), dtype=torch.long, device=dev)
        none = torch.full((b, 1), -1, dtype=torch.long, device=dev)
        src0 = torch.cat((_src(0, zero), _src(1, semantic_token_ids), _src(2, zero),
                          _src(3, coarse_token_ids + qid * self.codebook_size)), dim=1)
        src1 = torch.cat((none.expand(b, S + 2), _src(4, qid.expand(b, nc))), dim=1)
        tokens = _gather_tokens(src0, src1, [self.semantic_start_token, self.semantic_embedding.weight,
                                             self.coarse_start_token, self.coarse_embedding.weight,
                                             self.coarse_quantize_embedding.weight],
                                self.semantic_start_token.shape[-1])
        # relative position bias, except between the semantic and the coarse segment where one learned scalar
        # per head is used so cross attention is not dominated by relative positions (:920-936)
        attn_bias = None
        rp = self.transformer.rel_pos_bias
        if exists(rp):
            seq_len = tokens.shape[-2]
            attn_bias = gather_bias(rp.table(seq_len), self.cross_attn_bias, self._cross_index(seq_len, S + 1, dev))
        want_cache = return_cache or exists(kv_cache)
        tokens = self.transformer(tokens, self_attn_mask=self_attn_mask, attn_bias=attn_bias, kv_cache=kv_cache,
                                  return_kv_cache=want_cache)
        tokens, new_kv = tokens if want_cache else (tokens, None)
        if exists(embed_cache):
            tokens = torch.cat((embed_cache.to(tokens.dtype), tokens), dim=-2)
        new_embed_cache = tokens
        pred_sem, pred_coarse = tokens[:, :S], tokens[:, S + 1:]
        sem_logits = None
        if self._defer_heads:   # the wrapper's loss path: heads + cross entropy run fused, no logits tensors
            if not return_only_coarse_logits and exists(self.to_semantic_logits):
                sem_logits = LazyLogits(self._heads, pred_sem, self.to_semantic_logits.weight,
                                        self.to_semantic_logits.bias, "sem", False)
            logits = (sem_logits, LazyLogits(self._heads, pred_coarse, self.coarse_logit_weights, None, "coarse", True))
            return (logits, (new_kv, new_embed_cache)) if return_cache else logits
        if not return_only_coarse_logits and exists(self.to_semantic_logits):
            d = pred_sem.shape[-1]
            sem_logits = self._heads.linear(pred_sem.reshape(-1, d), self.to_semantic_logits.weight,
                                            self.to_semantic_logits.bias, "sem").view(b, S, -1)
        coarse_logits = self._heads.grouped(pred_coarse, self.coarse_logit_weights, "coarse")
        logits = (sem_logits, coarse_logits)
        return (logits, (new_kv, new_embed_cache)) if return_cache else logits


class FineTransformer(_TokenTransformer):
    """audiolm_pytorch.py:992-1368."""

    def __init__(self, *, num_coarse_quantizers, num_fine_quantizers, codebook_size, dim, depth, heads=8,
                 attn_dropout=0.0, ff_dropout=0.0, t5_name=DEFAULT_T5_NAME, has_condition=False, cond_dim=None,
                 audio_text_condition=False, cond_as_self_attn_prefix=False, cond_drop_prob=0.5,
                 grad_shrink_alpha=0.1, project_coarse_logits=True, pad_id=-1, rel_pos_bias=True, flash_attn=False,
                 **kwargs):
        super().__init__()
        self._init_common(dim, t5_name, cond_dim, has_condition, audio_text_condition, cond_drop_prob)
        rel = rel_pos_bias and not flash_attn
        self.num_coarse_quantizers = num_coarse_quantizers
        self.num_fine_quantizers = num_fine_quantizers
        self.codebook_size = codebook_size
        self.coarse_start_token = nn.Parameter(torch.randn(dim))
        self.fine_start_token = nn.Parameter(torch.randn(dim))
        self.coarse_embedding = nn.Embedding(num_coarse_quantizers * codebook_size, dim)
        self.fine_embedding = nn.Embedding(num_fine_quantizers * codebook_size, dim)
        self.coarse_quantize_embedding = nn.Embedding(num_coarse_quantizers, dim)
        self.fine_quantize_embedding = nn.Embedding(num_fine_quantizers, dim)
        self.pad_id = pad_id
        self.eos_id = codebook_size
        self.transformer = Transformer(dim=dim, depth=depth, heads=heads, attn_dropout=attn_dropout,
                                       ff_dropout=ff_dropout, rel_pos_bias=False,
                                       grad_shrink_alpha=grad_shrink_alpha, flash_attn=flash_attn, **kwargs)
        # 2-D (frame distance, quantizer distance) bias MLP + the start tokens' own bias (:1059-1071)
        self.null_pos_bias = nn.Parameter(torch.randn(heads, 1, 1)) if rel else None
        mlp_dim = dim // 2
        self.pos_bias_mlp = nn.Sequential(
            nn.Linear(2, mlp_dim), nn.SiLU(), nn.Linear(mlp_dim, mlp_dim), nn.SiLU(), nn.Linear(mlp_dim, heads)
        ) if rel else None
        self._bias_cache = HeadCache()
        self._bias_idx = {}
        self.coarse_logit_weights = (nn.Parameter(torch.randn(num_coarse_quantizers, codebook_size, dim))
                                     if project_coarse_logits else None)
        self.fine_logit_weights = nn.Parameter(torch.randn(num_fine_quantizers, codebook_size, dim))

    def forward_with_cond_scale(self, *args, cond_scale=3, return_kv_cache=False, kv_cache=None, embed_cache=None,
                                **kwargs):
        kv = None if kv_cache is None else kv_cache[0]
        emb = None if embed_cache is None else embed_cache[0]
        logits, (new_kv, new_emb) = self.forward(*args, cond_drop_prob=0.0, return_cache=True, kv_cache=kv,
                                                 embed_cache=emb, **kwargs)
        return (logits, (new_kv[None], new_emb[None])) if return_kv_cache else logits

    def _pos_coords(self, n, nf, dev):
        """per token of [coarse start | n coarse | fine start | nf fine]: frame position (-1 for the two start tokens)
        and quantizer offset (fine offsets follow the coarse ones); plus the frame count N = max_seq, the number of
        offsets and the table row stride rel_off = 2 * num_off - 1."""
        qc, qf = self.num_coarse_quantizers, self.num_fine_quantizers
        max_seq = max(ceil_div(n, qc), ceil_div(nf, qf))
        num_off = qc + qf
        rel_off = 2 * num_off - 1
        ar = lambda m: torch.arange(m, device=dev)  # noqa: E731
        minus1 = torch.full((1,), -1, device=dev)
        zero = torch.zeros(1, dtype=torch.long, device=dev)
        pos = torch.cat((minus1, ar(n) // qc, minus1, ar(nf) // qf))
        off = torch.cat((zero, ar(n) % qc, zero, ar(nf) % qf + qc))
        return pos, off, max_seq, num_off, rel_off

    def _pos_bias_index(self, n, nf, dev):
        """(idx int32 [L, L], mlp inputs fp32 [P, 2]) of the engineered coarse/fine bias (:1229-1298).

        Token t has a frame position and a quantizer offset (`_pos_coords`); the bias of (i, j) is the MLP at
        (frame_i - frame_j, offset_i - offset_j), shifted to non-negative table coordinates; rows / columns of the
        two start tokens use `null_pos_bias` (idx -1)."""
        key = (n, nf, str(dev))
        if self._bias_idx.get("key") != key:
            pos, off, max_seq, num_off, rel_off = self._pos_coords(n, nf, dev)
            pc = pos.clamp(min=0)
            idx = (pc[:, None] - pc[None, :] + max_seq - 1) * rel_off + (off[:, None] - off[None, :] + num_off - 1)
            start = pos == -1
            idx[start[:, None] | start[None, :]] = -1
            self._bias_idx = dict(key=key, val=(idx.to(torch.int32).contiguous(), _pos_mlp_in(max_seq, rel_off, dev)))
        return self._bias_idx["val"]

    def decode_bias_coords(self, num_coarse, num_fine, max_len, dev=None):
        """(u, cls, c) of the decode engine's bias rule for [coarse start | num_coarse coarse | fine start | fine
        tokens] over cache positions 0..max_len-1, while the sequence holds at most num_fine fine tokens:
        u = frame * rel_off + offset and c = (N - 1) * rel_off + num_off - 1, so u[L] - u[j] + c is the row
        `_pos_bias_index` picks; the start tokens are class -1 (null_pos_bias).  The table (and N) of the dense path
        depends on the fine length; it is the same at every length the sequence passes through only while the fine
        frames do not outnumber the coarse ones, which is asserted."""
        qc, qf = self.num_coarse_quantizers, self.num_fine_quantizers
        assert ceil_div(num_fine, qf) <= ceil_div(num_coarse, qc), \
            "the fine frames outnumber the coarse frames: the bias table would change during decoding"
        pos, off, max_seq, num_off, rel_off = self._pos_coords(num_coarse, num_fine, dev)
        n_all = pos.shape[0]
        assert n_all <= max_len
        u = torch.zeros(max_len, dtype=torch.int32, device=dev)
        cls = torch.full((max_len,), -1, dtype=torch.int32, device=dev)
        u[:n_all] = (pos.clamp(min=0) * rel_off + off).to(torch.int32)
        cls[:n_all] = torch.where(pos < 0, -1, 0).to(torch.int32)
        return u, cls, (max_seq - 1) * rel_off + num_off - 1

    def decode_bias(self, num_coarse, num_fine, max_len):
        """(table, override, u, cls, c) of the decode engine's bias (see decode_bias_coords), None on the flash path.
        The table is the pos_bias_mlp over the dense path's table rows, so both paths read the same values."""
        if not exists(self.pos_bias_mlp):
            return None
        u, cls, c = self.decode_bias_coords(num_coarse, num_fine, max_len, self.device)
        _, _, max_seq, _, rel_off = self._pos_coords(num_coarse, num_fine, "cpu")
        m = self.pos_bias_mlp
        table = mlp_table(_pos_mlp_in(max_seq, rel_off, self.device), m[0], [m[2]], m[4], self._bias_cache, "pos")
        return table, self.null_pos_bias.reshape(-1), u, cls, c

    def forward(self, coarse_token_ids, fine_token_ids, text=None, text_embeds=None, cond_drop_prob=None,
                self_attn_mask=None, kv_cache=None, embed_cache=None, return_cache=False,
                return_only_fine_logits=False):
        self._no_text(text, text_embeds)
        dev = coarse_token_ids.device
        b = coarse_token_ids.shape[0]
        coarse_token_ids = coarse_token_ids.reshape(b, -1)
        fine_token_ids = fine_token_ids.reshape(b, -1)
        n, nf = coarse_token_ids.shape[-1], fine_token_ids.shape[-1]
        # padded / eos coarse positions are never attended to (:1175-1184)
        keep = (coarse_token_ids != self.pad_id) & (coarse_token_ids != self.eos_id)
        coarse_token_ids = coarse_token_ids.masked_fill(~keep, 0)
        keep = F.pad(keep, (1, nf + 1), value=True)
        self_attn_mask = keep if self_attn_mask is None else (self_attn_mask & keep)
        qc, qf = self.num_coarse_quantizers, self.num_fine_quantizers
        cq, fq = _quantizer_ids(n, qc, dev), _quantizer_ids(nf, qf, dev)
        zero = torch.zeros((b, 1), dtype=torch.long, device=dev)
        none = torch.full((b, 1), -1, dtype=torch.long, device=dev)
        src0 = torch.cat((_src(0, zero), _src(1, coarse_token_ids + cq * self.codebook_size), _src(2, zero),
                          _src(3, fine_token_ids + fq * self.codebook_size)), dim=1)
        src1 = torch.cat((none, _src(4, cq.expand(b, n)), none, _src(5, fq.expand(b, nf))), dim=1)
        tokens = _gather_tokens(src0, src1, [self.coarse_start_token, self.coarse_embedding.weight,
                                             self.fine_start_token, self.fine_embedding.weight,
                                             self.coarse_quantize_embedding.weight,
                                             self.fine_quantize_embedding.weight], self.coarse_start_token.shape[-1])
        attn_bias = None
        if exists(self.pos_bias_mlp):
            idx, mlp_in = self._pos_bias_index(n, nf, dev)
            m = self.pos_bias_mlp
            table = mlp_table(mlp_in, m[0], [m[2]], m[4], self._bias_cache, "pos")
            attn_bias = gather_bias(table, self.null_pos_bias, idx)
        want_cache = return_cache or exists(kv_cache)
        tokens = self.transformer(tokens, self_attn_mask=self_attn_mask, attn_bias=attn_bias, kv_cache=kv_cache,
                                  return_kv_cache=want_cache)
        tokens, new_kv = tokens if want_cache else (tokens, None)
        if exists(embed_cache):
            tokens = torch.cat((embed_cache.to(tokens.dtype), tokens), dim=-2)
        new_embed_cache = tokens
        pred_coarse, pred_fine = tokens[:, :n], tokens[:, n + 1:]
        coarse_logits = None
        if self._defer_heads:   # the wrapper's loss path: heads + cross entropy run fused, no logits tensors
            if not return_only_fine_logits and exists(self.coarse_logit_weights):
                coarse_logits = LazyLogits(self._heads, pred_coarse, self.coarse_logit_weights, None, "coarse", True)
            logits = (coarse_logits, LazyLogits(self._heads, pred_fine, self.fine_logit_weights, None, "fine", True))
            return (logits, (new_kv, new_embed_cache)) if return_cache else logits
        if not return_only_fine_logits and exists(self.coarse_logit_weights):
            coarse_logits = self._heads.grouped(pred_coarse, self.coarse_logit_weights, "coarse")
        fine_logits = self._heads.grouped(pred_fine, self.fine_logit_weights, "fine")
        logits = (coarse_logits, fine_logits)
        return (logits, (new_kv, new_embed_cache)) if return_cache else logits


# ----------------------------------------------------------------------------------------------
# training / sampling wrappers
# ----------------------------------------------------------------------------------------------
def _eval_no_grad(fn):
    def inner(self, *a, **k):
        was = self.training
        self.eval()
        with torch.inference_mode():
            out = fn(self, *a, **k)
        self.train(was)
        return out
    return inner


def _cached_engine(owner, stack, batch, max_len, filter_thres, temperature, *, embed_fn, logits_fn, bias_fn=None):
    """one TokenDecoder (static KV cache + captured graphs) per wrapper, rebuilt when shapes or weights change (the
    graphs hold pointers to the packed bf16 weight copies of the current parameter versions).

    bias_fn(max_len) -> (table, override, u, cls, c) or None: the additive attention bias of the model
    (decode.StackDecoder.set_bias), recomputed for every call and written into the engine's static buffers."""
    # the captured graphs hold raw pointers to the fp32 parameters and to their packed bf16 copies: key on storage
    # address AND version of every parameter (`p.data = ...`, load_state_dict(assign=True), .to(...) change the
    # address without bumping the version)
    ver = hash(tuple((p.data_ptr(), p._version) for p in owner.parameters()))
    max_len = -(-max_len // 256) * 256  # fewer distinct cache sizes -> fewer graph captures
    gens = (stack._packed.generation, owner.transformer._heads._pk.generation)
    bias = None if bias_fn is None else bias_fn(max_len)
    # the captured bias-row launch holds the table's size and the constant c (the fine table's size depends on the
    # number of frames)
    bias_key = None if bias is None else (tuple(bias[0].shape), bias[1] is None, int(bias[4]))
    key = (batch, max_len, float(filter_thres), float(temperature), ver, gens, str(stack.norm.gamma.device), bias_key)
    eng = getattr(owner, "_engine", None)
    if eng is None or eng[0] != key:
        dec = TokenDecoder(StackDecoder(stack, batch, max_len), embed_fn, logits_fn, filter_thres=filter_thres,
                           temperature=temperature, use_graph=USE_DECODE_GRAPHS)
        owner._engine = eng = (key, dec)
    eng[1].stack.set_key_mask(None)
    if bias is not None:
        eng[1].stack.set_bias(*bias)
    return eng[1]


def _sample_next(last_logits, filter_thres, temperature):
    """top_k(thres) + gumbel_sample (audiolm_pytorch.py:1498-1499): the uniform noise comes from torch (same
    draw as `zeros_like(t).uniform_(0, 1)`), the filter + Gumbel-max runs in one alm_topk_gumbel_sample launch."""
    last_logits = last_logits.float().contiguous()
    k = max(int((1 - filter_thres) * last_logits.shape[-1]), 1)
    noise = torch.zeros_like(last_logits).uniform_(0, 1)
    return ops.topk_gumbel_sample(last_logits, noise, k=k, temperature=temperature)[:, None]


class SemanticTransformerWrapper(nn.Module):
    """audiolm_pytorch.py:1372-1567."""

    def __init__(self, *, transformer: SemanticTransformer, wav2vec=None, audio_conditioner=None, pad_id=-1,
                 unique_consecutive=True, mask_prob=0.15):
        super().__init__()
        assert audio_conditioner is None, "audio conditioning is outside the accelerated hot path"
        self.wav2vec = wav2vec
        self.transformer = transformer
        self.to(transformer.device)
        self.audio_conditioner = None
        assert not exists(wav2vec) or wav2vec.codebook_size == transformer.num_semantic_tokens
        self.unique_consecutive = unique_consecutive
        self.pad_id = pad_id
        self.eos_id = transformer.eos_id
        self.mask_prob = mask_prob

    @property
    def device(self):
        return next(self.parameters()).device

    @_eval_no_grad
    def generate(self, *, max_length, text=None, text_embeds=None, prime_wave=None, prime_wave_input_sample_hz=None,
                 prime_ids=None, batch_size=1, cond_scale=3, filter_thres=0.9, temperature=1.0, use_kv_cache=True,
                 include_eos_in_output=True, **kwargs):
        dev = self.device
        if exists(prime_wave):
            assert not exists(prime_ids) and exists(self.wav2vec)
            ids = self.wav2vec(prime_wave.to(dev), flatten=False, input_sample_hz=prime_wave_input_sample_hz)
        elif exists(prime_ids):
            ids = prime_ids
        else:
            ids = torch.empty((batch_size, 0), dtype=torch.long, device=dev)
        if self.unique_consecutive:
            ids = batch_unique_consecutive(ids, pad_value=self.pad_id)
        batch, start = ids.shape
        out = ids.clone()
        if use_kv_cache and start < max_length and bool((ids != self.pad_id).all()):
            return self._generate_graphed(out, max_length, filter_thres, temperature)
        last = (ids != self.pad_id).sum(dim=-1).long()
        kv_cache, logits = None, None
        for _ in range(start, max_length):
            new_logits, new_kv = self.transformer.forward_with_cond_scale(ids=out, cond_scale=cond_scale,
                                                                          kv_cache=kv_cache, return_kv_cache=True,
                                                                          **kwargs)
            if use_kv_cache:
                kv_cache = new_kv
                logits = new_logits if logits is None else torch.cat((logits, new_logits), dim=-2)
            else:
                logits = new_logits
            last_logits = logits.gather(1, last[:, None, None].expand(batch, 1, logits.shape[-1]))[:, 0]
            out = torch.cat((out, _sample_next(last_logits, filter_thres, temperature)), dim=-1)
            if (out == self.eos_id).any(dim=-1).all():
                break
            last = last + 1
        return mask_out_after_eos_id(out, self.eos_id, keep_eos=False)

    def _generate_graphed(self, out, max_length, filter_thres, temperature):
        """KV-cache sampling loop on the CUDA-graph decode engine (decode.py): the prompt goes through the normal
        forward once, every further token is one graph replay + an EOS poll."""
        tr = self.transformer
        batch = out.shape[0]
        logits, kv = tr.forward_with_cond_scale(ids=out, return_kv_cache=True)
        out = torch.cat((out, _sample_next(logits[:, -1], filter_thres, temperature)), dim=-1)
        dec = _cached_engine(self, tr.transformer, batch, max_length + 2, filter_thres, temperature,
                             embed_fn=lambda tok, _key: tr.semantic_embedding(tok),
                             logits_fn=lambda o, _key: tr._heads.linear_decode(o, tr.to_logits.weight, tr.to_logits.bias, "sem"),
                             bias_fn=tr.decode_bias)
        dec.stack.load_cache(kv[0])
        dec.tok.copy_(out[:, -1])
        for _ in range(out.shape[1], max_length):
            if (out == self.eos_id).any(dim=-1).all():
                break
            dec.advance()
            out = torch.cat((out, dec.tok[:, None]), dim=-1)
        return mask_out_after_eos_id(out, self.eos_id, keep_eos=False)

    def forward(self, *, semantic_token_ids=None, raw_wave=None, text=None, text_embeds=None, return_loss=False,
                **kwargs):
        assert exists(raw_wave) or exists(semantic_token_ids)
        if not exists(semantic_token_ids):
            assert exists(self.wav2vec), "VQWav2Vec must be be provided if given raw wave for training"
            semantic_token_ids = self.wav2vec(raw_wave, flatten=False)
        ids = semantic_token_ids.reshape(semantic_token_ids.shape[0], -1)
        if self.training:
            ids = append_eos_id(ids, self.transformer.eos_id)
        if self.unique_consecutive:
            ids = batch_unique_consecutive(ids, pad_value=self.pad_id)
        input_ids = ids[:, :-1] if return_loss else ids
        mask = None
        if self.mask_prob > 0.0 and self.training:
            mask = generate_mask_with_prob(input_ids.shape, self.mask_prob, input_ids.device)
        with _deferred_heads(self.transformer, return_loss):
            logits = self.transformer(ids=input_ids, self_attn_mask=mask, **kwargs)
        if not return_loss:
            return logits
        return cross_entropy(logits, ids, ignore_index=self.pad_id)


def _frame_sampler(step_fn, n_quantizers, time_steps, seq, filter_thres, temperature, use_kv_cache):
    """shared double loop of Coarse/Fine generate (:1677-1706, :1965-1994): one token per (frame, quantizer),
    EOS only allowed at a frame boundary."""
    kv_cache = embed_cache = None
    for t in time_steps:
        for qi in range(n_quantizers):
            at_boundary = qi == 0 and t > 0
            logits, (nkv, nemb) = step_fn(seq, kv_cache, embed_cache)
            if use_kv_cache:
                kv_cache, embed_cache = nkv, nemb
            last = logits[:, -1].clone()
            if not at_boundary:
                last[:, -1] = float("-inf")
            seq = torch.cat((seq, _sample_next(last, filter_thres, temperature)), dim=-1)
    return seq


def _frame_sampler_graphed(owner, stack, step_fn, n_quantizers, time_steps, seq, filter_thres, temperature, *,
                           embed_fn, head_fn, prefix_len, key_mask=None, bias_fn=None):
    """`_frame_sampler` with the KV cache on the CUDA-graph decode engine (decode.py): the first token goes through
    the normal forward (which also fills the cache), every further token is one graph replay.  One graph per
    quantizer index of the token being fed back (embedding offset, next head, EOS rule all depend on it only).

    embed_fn(tok, q) -> [b, d];  head_fn(out, q_next) -> fp32 logits of the token with quantizer index q_next."""
    time_steps = list(time_steps)
    total = len(time_steps) * n_quantizers
    if total == 0:
        return seq
    batch = seq.shape[0]
    logits, (kv, _) = step_fn(seq, None, None)
    last = logits[:, -1].clone()
    if not time_steps[0] > 0:
        last[:, -1] = float("-inf")
    buf = torch.empty(batch, total, device=seq.device, dtype=torch.long)
    buf[:, 0] = _sample_next(last, filter_thres, temperature)[:, 0]

    def logits_fn(out, q_in):  # EOS (the last class) only at a frame boundary (:1699-1700, 1987-1988)
        q_next = (q_in + 1) % n_quantizers
        lg = head_fn(out, q_next)
        if q_next != 0:
            lg[:, -1] = float("-inf")
        return lg

    dec = _cached_engine(owner, stack, batch, prefix_len + total + 1, filter_thres, temperature, embed_fn=embed_fn,
                         logits_fn=logits_fn, bias_fn=bias_fn)
    dec.stack.load_cache(kv[0])
    if exists(key_mask):
        dec.stack.set_key_mask(key_mask)
    dec.tok.copy_(buf[:, 0])
    for i in range(1, total):
        dec.advance(key=(i - 1) % n_quantizers)
        buf[:, i] = dec.tok
    return torch.cat((seq, buf), dim=-1)


class CoarseTransformerWrapper(nn.Module):
    """audiolm_pytorch.py:1569-1854."""

    def __init__(self, *, transformer: CoarseTransformer, codec=None, wav2vec=None, audio_conditioner=None,
                 pad_id=-1, unique_consecutive=True, semantic_cross_entropy_loss_weight=1.0, mask_prob=0.15):
        super().__init__()
        assert audio_conditioner is None, "audio conditioning is outside the accelerated hot path"
        self.codec = codec
        self.wav2vec = wav2vec
        self.transformer = transformer
        self.to(transformer.device)
        self.audio_conditioner = None
        self.unique_consecutive = unique_consecutive
        self.pad_id = pad_id
        self.semantic_cross_entropy_loss_weight = semantic_cross_entropy_loss_weight
        self.num_coarse_quantizers = transformer.num_coarse_quantizers * codec.rq_groups
        self.semantic_eos_id = transformer.semantic_eos_id
        self.coarse_eos_id = transformer.coarse_eos_id
        self.mask_prob = mask_prob

    @property
    def device(self):
        return next(self.parameters()).device

    def _codec_ids(self, wave, input_sample_hz=None):
        with torch.inference_mode():
            self.codec.eval()
            _, indices, _ = self.codec(wave, return_encoded=True, input_sample_hz=input_sample_hz)
        return indices.long()   # FSQ codecs emit int32 ids; labels and sampled sequences are int64

    @_eval_no_grad
    def generate(self, *, semantic_token_ids, prime_wave=None, prime_wave_input_sample_hz=None,
                 prime_coarse_token_ids=None, text=None, text_embeds=None, max_time_steps=512, cond_scale=3.0,
                 filter_thres=0.9, temperature=1.0, reconstruct_wave=False, use_kv_cache=True, **kwargs):
        dev = self.device
        batch = semantic_token_ids.shape[0]
        semantic_token_ids = semantic_token_ids.to(dev)
        assert not (exists(prime_wave) and exists(prime_coarse_token_ids))
        if exists(prime_coarse_token_ids):
            coarse = prime_coarse_token_ids.long()
        elif exists(prime_wave):
            assert exists(self.codec)
            coarse = self._codec_ids(prime_wave.to(dev), prime_wave_input_sample_hz)[..., :self.num_coarse_quantizers]
            coarse = coarse.reshape(batch, -1)
        else:
            coarse = torch.empty((batch, 0), device=dev, dtype=torch.long)
        if self.unique_consecutive:
            semantic_token_ids = batch_unique_consecutive(semantic_token_ids, pad_value=self.pad_id)

        def step(seq, kv, emb):
            (_, cl), caches = self.transformer.forward_with_cond_scale(
                coarse_token_ids=seq, semantic_token_ids=semantic_token_ids, cond_scale=cond_scale,
                return_kv_cache=True, kv_cache=kv, embed_cache=emb, return_only_coarse_logits=True, **kwargs)
            return cl, caches

        tr = self.transformer
        q_n = self.num_coarse_quantizers
        if use_kv_cache and not kwargs and coarse.shape[-1] % q_n == 0 and max_time_steps > 0:
            cb = tr.codebook_size
            n_sem = semantic_token_ids.reshape(batch, -1).shape[-1]
            seq = _frame_sampler_graphed(
                self, tr.transformer, step, q_n, range(0, max_time_steps), coarse.clone(), filter_thres, temperature,
                embed_fn=lambda tok, q: tr.coarse_embedding(tok + q * cb) + tr.coarse_quantize_embedding.weight[q],
                head_fn=lambda o, q: tr._heads.linear_decode(o, tr.coarse_logit_weights[q], None, ("coarse", q)),
                prefix_len=n_sem + 2 + coarse.shape[-1], bias_fn=lambda ml: tr.decode_bias(n_sem, ml))
        else:
            seq = _frame_sampler(step, q_n, range(0, max_time_steps), coarse.clone(), filter_thres, temperature,
                                 use_kv_cache)
        seq = mask_out_after_eos_id(seq, self.coarse_eos_id, keep_eos=False)
        seq = seq.reshape(batch, -1, self.num_coarse_quantizers)
        if not reconstruct_wave:
            return seq
        assert exists(self.codec)
        if not (seq == -1).any():
            return self.codec.decode_from_codebook_indices(seq)[:, 0]
        wavs = []
        for sample in seq:
            pad = (sample == -1).any(dim=-1)
            wavs.append(None if pad.all() else self.codec.decode_from_codebook_indices(sample[~pad][None])[0, 0])
        return wavs

    def forward(self, *, semantic_token_ids=None, raw_wave=None, raw_wave_for_codec=None, text=None,
                text_embeds=None, coarse_token_ids=None, return_loss=False, **kwargs):
        assert exists(raw_wave) or exists(semantic_token_ids)
        raw_wave_for_codec = default(raw_wave_for_codec, raw_wave)
        assert exists(raw_wave_for_codec) or exists(coarse_token_ids)
        assert not all(map(exists, (raw_wave, raw_wave_for_codec, semantic_token_ids, coarse_token_ids)))
        if not exists(semantic_token_ids):
            assert exists(self.wav2vec), "VQWav2Vec must be be provided if given raw wave for training"
            semantic_token_ids = self.wav2vec(raw_wave, flatten=False)
        if not exists(coarse_token_ids):
            assert exists(self.codec), "Codec must be provided if given raw wave for training"
            indices = self._codec_ids(raw_wave_for_codec)
            batch, T = raw_wave_for_codec.shape
            assert indices.shape[0] == batch and indices.shape[1] == int(T / self.codec.seq_len_multiple_of)
            coarse_token_ids = indices[..., :self.num_coarse_quantizers]
        b = semantic_token_ids.shape[0]
        sem = semantic_token_ids.reshape(b, -1)
        coarse = coarse_token_ids.reshape(b, -1).long()
        if self.training:
            sem = append_eos_id(sem, self.transformer.semantic_eos_id)
            coarse = append_eos_id(coarse, self.transformer.coarse_eos_id)
        if self.unique_consecutive:
            sem = batch_unique_consecutive(sem, pad_value=self.pad_id)
        if return_loss:
            sem_labels, coarse_labels = sem, coarse.clone()
            coarse = coarse[:, :-1]
        # padding and the semantic EOS are never attended to (:1801-1805)
        mask = (sem != self.pad_id) & (sem != self.semantic_eos_id)
        sem = sem.masked_fill(~mask, 0)
        mask = F.pad(mask, (1, coarse.shape[-1] + 1), value=True)
        if self.mask_prob > 0 and self.training:
            mask = mask & generate_mask_with_prob(mask.shape, self.mask_prob, device=mask.device)
        with _deferred_heads(self.transformer, return_loss):
            sem_logits, coarse_logits = self.transformer(semantic_token_ids=sem, coarse_token_ids=coarse,
                                                         self_attn_mask=mask, **kwargs)
        if not return_loss:
            return sem_logits, coarse_logits
        if self.unique_consecutive:
            n_coarse, n_sem_all = coarse_labels.numel(), (sem_labels != self.pad_id).sum()
        else:
            n_coarse, n_sem_all = coarse_logits.shape[1], sem_logits.shape[1]
        sem_loss, n_sem = 0.0, 0
        if self.semantic_cross_entropy_loss_weight > 0 and exists(sem_logits):
            n_sem = n_sem_all
            sem_loss = cross_entropy(sem_logits, sem_labels, ignore_index=self.pad_id)
        coarse_loss = cross_entropy(coarse_logits, coarse_labels, ignore_index=self.pad_id)
        return (sem_loss * n_sem * self.semantic_cross_entropy_loss_weight + coarse_loss * n_coarse) / \
            (n_sem + n_coarse)


class FineTransformerWrapper(nn.Module):
    """audiolm_pytorch.py:1856-2137."""

    def __init__(self, *, transformer: FineTransformer, codec=None, audio_conditioner=None,
                 coarse_cross_entropy_loss_weight=1.0, pad_id=-1, mask_prob=0.15):
        super().__init__()
        assert audio_conditioner is None, "audio conditioning is outside the accelerated hot path"
        self.codec = codec
        self.transformer = transformer
        self.to(transformer.device)
        self.audio_conditioner = None
        self.num_fine_quantizers = transformer.num_fine_quantizers * codec.rq_groups
        self.num_coarse_quantizers = transformer.num_coarse_quantizers * codec.rq_groups
        assert (self.num_fine_quantizers + self.num_coarse_quantizers) == codec.num_quantizers * codec.rq_groups
        self.eos_id = transformer.eos_id
        assert self.num_coarse_quantizers > 0
        self.pad_id = pad_id
        self.coarse_cross_entropy_loss_weight = coarse_cross_entropy_loss_weight
        self.mask_prob = mask_prob

    @property
    def device(self):
        return next(self.parameters()).device

    @_eval_no_grad
    def generate(self, *, coarse_token_ids, prime_wave=None, prime_wave_input_sample_hz=None,
                 prime_fine_token_ids=None, text=None, text_embeds=None, cond_scale=3.0, filter_thres=0.9,
                 temperature=1.0, reconstruct_wave=False, use_kv_cache=True, mask_out_generated_fine_tokens=False,
                 **kwargs):
        dev = self.device
        batch = coarse_token_ids.shape[0]
        coarse = coarse_token_ids.reshape(batch, -1).to(dev).long()
        assert not (exists(prime_wave) and exists(prime_fine_token_ids))
        if exists(prime_fine_token_ids):
            fine = prime_fine_token_ids.long()
        elif exists(prime_wave):
            assert exists(self.codec)
            with torch.inference_mode():
                self.codec.eval()
                _, ids, _ = self.codec(prime_wave.to(dev), return_encoded=True,
                                       input_sample_hz=prime_wave_input_sample_hz)
            fine = ids[..., self.num_coarse_quantizers:].reshape(batch, -1).long()
        else:
            fine = torch.empty((batch, 0), device=dev, dtype=torch.long)
        first = fine.shape[-1] // self.num_fine_quantizers
        steps = coarse.shape[1] // self.num_coarse_quantizers

        def step(seq, kv, emb):
            (_, fl), caches = self.transformer.forward_with_cond_scale(
                coarse_token_ids=coarse, fine_token_ids=seq, cond_scale=cond_scale, return_only_fine_logits=True,
                kv_cache=kv, embed_cache=emb, return_kv_cache=True, **kwargs)
            return fl, caches

        tr = self.transformer
        q_n = self.num_fine_quantizers
        if use_kv_cache and not kwargs and fine.shape[-1] % q_n == 0 and steps > first:
            cb = tr.codebook_size
            # padded / eos coarse positions are never attended to (FineTransformer.forward, :1175-1184)
            keep = F.pad((coarse != tr.pad_id) & (coarse != tr.eos_id), (1, 0), value=True)
            seq = _frame_sampler_graphed(
                self, tr.transformer, step, q_n, range(first, steps), fine.clone(), filter_thres, temperature,
                embed_fn=lambda tok, q: tr.fine_embedding(tok + q * cb) + tr.fine_quantize_embedding.weight[q],
                head_fn=lambda o, q: tr._heads.linear_decode(o, tr.fine_logit_weights[q], None, ("fine", q)),
                prefix_len=coarse.shape[-1] + 2 + fine.shape[-1], key_mask=None if bool(keep.all()) else keep,
                bias_fn=lambda ml: tr.decode_bias(coarse.shape[-1], steps * q_n, ml))
        else:
            seq = _frame_sampler(step, q_n, range(first, steps), fine.clone(), filter_thres, temperature,
                                 use_kv_cache)
        seq = mask_out_after_eos_id(seq, self.eos_id, keep_eos=False)
        seq = seq.reshape(batch, -1, self.num_fine_quantizers)
        coarse3 = coarse.reshape(batch, -1, self.num_coarse_quantizers)
        if mask_out_generated_fine_tokens:
            seq = seq.masked_fill((coarse3 == self.pad_id).all(dim=-1, keepdim=True), self.pad_id)
        if not reconstruct_wave:
            return seq
        assert exists(self.codec)
        both = torch.cat((coarse3, seq), dim=-1)
        pad = (both == self.pad_id).any(dim=-1)
        if not pad.any():
            return self.codec.decode_from_codebook_indices(both)[:, 0]
        return [self.codec.decode_from_codebook_indices(ids[~m][None])[0, 0] for ids, m in zip(both, pad)]

    def forward(self, *, raw_wave=None, text=None, text_embeds=None, token_ids=None, coarse_token_ids=None,
                fine_token_ids=None, return_loss=False, **kwargs):
        assert exists(raw_wave) ^ (exists(token_ids) ^ (exists(coarse_token_ids) and exists(fine_token_ids)))
        if exists(raw_wave):
            assert exists(self.codec), "Codec must be provided if given raw wave for training"
            with torch.inference_mode():
                self.codec.eval()
                _, token_ids, _ = self.codec(raw_wave, return_encoded=True)
            batch, T = raw_wave.shape
            frames = int(T / self.codec.seq_len_multiple_of)
            assert token_ids.shape == (batch, frames, self.num_coarse_quantizers + self.num_fine_quantizers)
        if exists(token_ids):
            coarse_token_ids = token_ids[..., :self.num_coarse_quantizers]
            fine_token_ids = token_ids[..., self.num_coarse_quantizers:]
        b = coarse_token_ids.shape[0]
        coarse = coarse_token_ids.reshape(b, -1).long()
        fine = fine_token_ids.reshape(b, -1).long()
        if return_loss:
            coarse_labels, fine_labels = coarse, fine
            fine = fine[:, :-1]
        mask = None
        if self.mask_prob > 0 and self.training:
            mask = generate_mask_with_prob((b, coarse.shape[-1] + fine.shape[-1] + 2), self.mask_prob, self.device)
        with _deferred_heads(self.transformer, return_loss):
            coarse_logits, fine_logits = self.transformer(coarse_token_ids=coarse, fine_token_ids=fine,
                                                          self_attn_mask=mask, **kwargs)
        if not return_loss:
            return coarse_logits, fine_logits
        n_fine = fine_logits.shape[1]
        n_coarse, coarse_loss = 0, 0.0
        if self.coarse_cross_entropy_loss_weight > 0 and exists(coarse_logits):
            n_coarse = coarse_logits.shape[1]
            coarse_loss = cross_entropy(coarse_logits, coarse_labels, ignore_index=self.pad_id)
        fine_loss = cross_entropy(fine_logits, fine_labels, ignore_index=self.pad_id)
        return (coarse_loss * n_coarse * self.coarse_cross_entropy_loss_weight + fine_loss * n_fine) / \
            (n_coarse + n_fine)


class AudioLM(nn.Module):
    """audiolm_pytorch.py:2141-2254: semantic -> coarse -> fine -> codec decode."""

    def __init__(self, *, wav2vec, codec, semantic_transformer: SemanticTransformer,
                 coarse_transformer: CoarseTransformer, fine_transformer: FineTransformer, audio_conditioner=None,
                 unique_consecutive=True):
        super().__init__()
        assert audio_conditioner is None, "audio conditioning is outside the accelerated hot path"
        self.audio_conditioner = None
        assert semantic_transformer.num_semantic_tokens == coarse_transformer.num_semantic_tokens
        assert coarse_transformer.codebook_size == fine_transformer.codebook_size
        assert coarse_transformer.num_coarse_quantizers == fine_transformer.num_coarse_quantizers
        assert fine_transformer.num_coarse_quantizers + fine_transformer.num_fine_quantizers == codec.num_quantizers
        self.needs_text = False
        self.semantic = SemanticTransformerWrapper(wav2vec=wav2vec, transformer=semantic_transformer,
                                                   unique_consecutive=unique_consecutive)
        self.coarse = CoarseTransformerWrapper(wav2vec=wav2vec, codec=codec, transformer=coarse_transformer,
                                               unique_consecutive=unique_consecutive)
        self.fine = FineTransformerWrapper(codec=codec, transformer=fine_transformer)

    @property
    def device(self):
        return next(self.parameters()).device

    @_eval_no_grad
    def forward(self, *, batch_size=1, text=None, text_embeds=None, prime_wave=None, prime_wave_input_sample_hz=None,
                prime_wave_path=None, max_length=2048, return_coarse_generated_wave=False,
                mask_out_generated_fine_tokens=False):
        assert not (exists(text) or exists(text_embeds)), "text conditioning is outside the accelerated hot path"
        assert not (exists(prime_wave) and exists(prime_wave_path))
        if exists(prime_wave):
            assert exists(prime_wave_input_sample_hz)
            prime_wave = prime_wave.to(self.device)
        elif exists(prime_wave_path):
            import torchaudio
            prime_wave, prime_wave_input_sample_hz = torchaudio.load(str(prime_wave_path))
            prime_wave = prime_wave.to(self.device)
        sem = self.semantic.generate(batch_size=batch_size, prime_wave=prime_wave,
                                     prime_wave_input_sample_hz=prime_wave_input_sample_hz, max_length=max_length)
        coarse = self.coarse.generate(semantic_token_ids=sem, prime_wave=prime_wave,
                                      prime_wave_input_sample_hz=prime_wave_input_sample_hz,
                                      reconstruct_wave=return_coarse_generated_wave)
        if return_coarse_generated_wave:
            return coarse
        return self.fine.generate(coarse_token_ids=coarse, prime_wave=prime_wave,
                                  prime_wave_input_sample_hz=prime_wave_input_sample_hz, reconstruct_wave=True,
                                  mask_out_generated_fine_tokens=mask_out_generated_fine_tokens)
