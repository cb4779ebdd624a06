"""Additive attention bias of the flash_attn=False path (SURVEY §8 row a7).

Reference: RelativePositionBias (audiolm_pytorch.py:202-242), the coarse transformer's cross-attention
override (:926-936) and the fine transformer's 2-D (position, quantizer) bias MLP (:1229-1298).

All three are "a small MLP evaluated on a few thousand relative offsets -> table [P, heads] -> gathered
into a dense [heads, i, j] bias, with some positions replaced by a learned per-head scalar".  Here the
D x D layers of the MLP run on the wgmma GEMM (through heads._LinearPacked: forward, dgrad, wgrad),
the gather / scatter-add over the 134 MB dense bias is `alm_bias_gather_fwd/bwd`, and the attention
kernels add the bias to the scores and accumulate d(bias) (`alm_mqa_attn_fwd/bwd`).  Only the first
layer (fan-in 1 or 2: an outer product, not a GEMM) and the SiLUs on the [P, D] table are torch
elementwise ops.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F
from torch import nn

from . import ops
from .heads import HeadCache

f32 = torch.float32


class _BiasGatherFn(torch.autograd.Function):
    """bias[h, i, j] = idx[i, j] >= 0 ? table[idx[i, j], h] : override[h]  (fp32 [H, n_q, pad4(n_k)])."""

    @staticmethod
    def forward(ctx, table, override, idx):
        ctx.idx = idx
        ctx.rows = table.shape[0]
        ctx.over_shape = None if override is None else override.shape
        flat = None if override is None else override.detach().reshape(-1).to(f32)
        return ops.bias_gather_fwd(table.detach().to(f32).contiguous(), idx, flat)

    @staticmethod
    def backward(ctx, dbias):
        dtable, dover = ops.bias_gather_bwd(dbias.contiguous(), ctx.idx, ctx.rows,
                                            want_override=ctx.over_shape is not None)
        return dtable, (None if dover is None else dover.view(ctx.over_shape)), None


def gather_bias(table, override, idx):
    """dense bias [H, n_q, n_k] (a view of the padded [H, n_q, pad4(n_k)] buffer the kernels read)."""
    n_k = idx.shape[1]
    return _BiasGatherFn.apply(table, override, idx)[..., :n_k]


def mlp_table(x, first, hidden, last, cache: HeadCache, key):
    """x [P, k_in] fp32 -> [P, heads] fp32 through Linear(k_in, D)+SiLU, (Linear(D, D)+SiLU)*, Linear(D, heads)."""
    w0 = first.weight                                  # [D, k_in], k_in in (1, 2): an outer product, not a GEMM
    h = first.bias + x[:, 0:1] * w0[:, 0]
    for k in range(1, x.shape[1]):
        h = h + x[:, k:k + 1] * w0[:, k]
    h = F.silu(h)
    for li, lin in enumerate(hidden):
        h = F.silu(cache.linear(h, lin.weight, lin.bias, (key, li)))
    return cache.linear(h, last.weight, last.bias, (key, "out"))


def as_kernel_bias(bias):
    """[H, i, j] fp32 tensor whose row stride is a multiple of 4 elements (what alm_mqa_attn_* reads)."""
    assert bias.dim() == 3, "attention bias must be [heads, i, j]"
    bias = bias.to(f32)
    if bias.stride(2) == 1 and bias.stride(1) % 4 == 0 and bias.stride(0) == bias.shape[1] * bias.stride(1):
        base = getattr(bias, "_base", None)
        if bias.is_contiguous():
            return bias
        if base is not None and base.dim() == 3 and base.is_contiguous() and base.shape[:2] == bias.shape[:2] \
                and base.data_ptr() == bias.data_ptr() and base.dtype == f32:
            return base                                 # the padded buffer `gather_bias` sliced
    pad = (-bias.shape[2]) % 4
    return F.pad(bias, (0, pad)).contiguous()


class RelativePositionBias(nn.Module):
    """audiolm_pytorch.py:202-242 (state-dict keys net.{k}.0.{weight,bias}, net.{layers}.{weight,bias})."""

    def __init__(self, *, dim, heads, layers=3):
        super().__init__()
        self.net = nn.ModuleList([])
        self.net.append(nn.Sequential(nn.Linear(1, dim), nn.SiLU()))
        for _ in range(layers - 1):
            self.net.append(nn.Sequential(nn.Linear(dim, dim), nn.SiLU()))
        self.net.append(nn.Linear(dim, heads))
        self._cache = HeadCache()
        self._idx = {}

    @property
    def device(self):
        return next(self.parameters()).device

    def table(self, j):
        """MLP over the 2j-1 relative offsets -(j-1) .. (j-1)  ->  [2j-1, heads]."""
        x = torch.arange(-j + 1, j, device=self.device, dtype=f32)[:, None]
        return mlp_table(x, self.net[0][0], [blk[0] for blk in self.net[1:-1]], self.net[-1], self._cache, "rel")

    def index(self, i, j):
        """int32 [i, j] row of `table` used by (query i, key j); queries are right-aligned (:232-236)."""
        key = (i, j, str(self.device))
        if key not in self._idx:
            if len(self._idx) > 8:
                self._idx.clear()
            i_pos = torch.arange(i, device=self.device) + (j - i)
            j_pos = torch.arange(j, device=self.device)
            self._idx[key] = (i_pos[:, None] - j_pos[None, :] + (j - 1)).to(torch.int32).contiguous()
        return self._idx[key]

    def forward(self, i, j):
        assert j >= i
        return gather_bias(self.table(j), None, self.index(i, j))
