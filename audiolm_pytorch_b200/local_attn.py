"""SoundStream's bottleneck `LocalTransformer` (soundstream.py:397-440) on libalm_b200 — inference path.

The reference builds it from the un-vendored `local-attention` package (`LocalMHA` + `FeedForward`,
soundstream.py:414-428): windowed causal attention (window w, one window of look-back, exact window size: query i sees
keys i-w..i), l2-normalised q / k with learned per-channel scales and a fixed score scale 8, rotary + xpos position
embedding over the 2w-key bucket, a sigmoid value gate per head, pre-LayerNorm, then a GEGLU feed-forward.  PARITY
UNPINNED upstream (package absent offline); the arithmetic here follows oracle/third_party.py::LocalMHA, which restates
the published implementation and is what the reference's own soundstream.py runs on when the goldens are generated.

Mapping onto the kernels: the (b, head, window) triples become the batch of `alm_mqa_attn_fwd` with one head, 128...w
queries against the 2w keys of [previous window | own window]; the lower edge of the band and the missing previous
window of the first bucket are an additive score bias / key-mask bits; projections and the feed-forward are
`alm_gemm_bf16` GEMMs.  Parameter names follow upstream so reference checkpoints load unchanged.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F
from torch import nn

from . import ops
from .transformer import _PackedWeights, pack_plain

bf16 = torch.bfloat16
f32 = torch.float32


class _RelPos(nn.Module):
    """holds `inv_freq` under the upstream key attn_fn.rel_pos.inv_freq"""

    def __init__(self, dim, theta=10000):
        super().__init__()
        self.register_buffer("inv_freq", 1.0 / (theta ** (torch.arange(0, dim, 2).float() / dim)))


class _AttnFn(nn.Module):
    def __init__(self, dim_head):
        super().__init__()
        self.rel_pos = _RelPos(dim_head)


def _rotate_half(x):
    x1, x2 = x.reshape(*x.shape[:-1], 2, x.shape[-1] // 2).unbind(dim=-2)
    return torch.cat((-x2, x1), dim=-1)


class LocalMHA(nn.Module):
    """local_attention.LocalMHA as the reference configures it (causal, prenorm, qk_rmsnorm, xpos rotary, per-head value
    gates).  forward(x [b, n, dim] fp32) -> [b, n, dim] fp32 (without the residual)."""

    def __init__(self, *, dim, window_size, dim_head=64, heads=8, causal=True, prenorm=True, qk_rmsnorm=True, qk_scale=8,
                 use_xpos=True, xpos_scale_base=None, use_rotary_pos_emb=True, gate_values_per_head=True, dropout=0.0,
                 **_):
        super().__init__()
        if not (causal and prenorm and qk_rmsnorm and use_xpos and use_rotary_pos_emb and gate_values_per_head):
            raise NotImplementedError("LocalMHA is built for the configuration soundstream.py:418-427 uses")
        if dim_head not in ops.ATTN_HEAD_WIDTHS:
            raise NotImplementedError(f"the sm_90a attention kernels are built for dim_head in {ops.ATTN_HEAD_WIDTHS}")
        if dim % 8 != 0:
            raise ValueError("dim must be a multiple of 8")
        inner = dim_head * heads
        self.heads, self.dim_head, self.window_size, self.qk_scale = heads, dim_head, window_size, float(qk_scale)
        self.xpos_scale_base = window_size // 2 if xpos_scale_base is None else xpos_scale_base
        self.norm = nn.LayerNorm(dim)
        self.to_qkv = nn.Linear(dim, inner * 3, bias=False)
        self.q_scale = nn.Parameter(torch.ones(dim_head))
        self.k_scale = nn.Parameter(torch.ones(dim_head))
        self.attn_fn = _AttnFn(dim_head)
        self.to_v_gate = nn.Sequential(nn.Linear(dim, heads))
        self.to_out = nn.Linear(inner, dim, bias=False)
        self._packed = _PackedWeights()
        self._tables = {}

    def _pos_tables(self, dev):
        """cos / sin / xpos scale of the 2w bucket positions (SinusoidalEmbeddings.forward) and the band bias"""
        key = str(dev)
        if key not in self._tables:
            w, dh = self.window_size, self.dim_head
            inv_freq = self.attn_fn.rel_pos.inv_freq.to(dev, f32)
            t = torch.arange(2 * w, device=dev, dtype=f32)
            freqs = torch.einsum("i,j->ij", t, inv_freq)
            freqs = torch.cat((freqs, freqs), dim=-1)
            base = (torch.arange(0, dh, 2, device=dev, dtype=f32) + 0.4 * dh) / (1.4 * dh)
            power = (t - (2 * w) // 2) / self.xpos_scale_base
            scale = base[None, :] ** power[:, None]
            scale = torch.cat((scale, scale), dim=-1)
            # exact window: query r of the bucket (key position w + r) sees key positions r .. w + r; the upper edge is
            # the kernel's (right-aligned) causal rule, the lower edge is this additive bias
            r = torch.arange(w, device=dev)[:, None]
            j = torch.arange(2 * w, device=dev)[None, :]
            ld = (2 * w + 3) // 4 * 4
            bias = torch.zeros(1, w, ld, device=dev, dtype=f32)
            bias[0, :, :2 * w] = torch.where(j < r, -1e30, 0.0)
            self._tables[key] = (freqs.cos(), freqs.sin(), scale, bias)
        return self._tables[key]

    def forward(self, x):
        if not x.is_cuda:
            raise ops._lib.AlmError("LocalMHA needs CUDA tensors (no CPU fallback)")
        b, n, dim = x.shape
        h, dh, w = self.heads, self.dim_head, self.window_size
        pk = self._packed
        wqkv = pk.get("qkv", [self.to_qkv.weight], lambda: pack_plain(self.to_qkv.weight))
        wo = pk.get("o", [self.to_out.weight], lambda: pack_plain(self.to_out.weight))
        xn = F.layer_norm(x.to(f32), (dim,), self.norm.weight, self.norm.bias, self.norm.eps)
        xb = xn.reshape(b * n, dim).to(bf16)
        qkv = ops.gemm(xb, wqkv).view(b, n, 3, h, dh).float()                     # wgmma GEMM
        q, k, v = (qkv[:, :, i].transpose(1, 2) for i in range(3))               # [b, h, n, dh]
        q = F.normalize(q, dim=-1) * self.q_scale
        k = F.normalize(k, dim=-1) * self.k_scale
        pad = (-n) % w
        if pad:
            q, k, v = (F.pad(t, (0, 0, 0, pad)) for t in (q, k, v))
        W = (n + pad) // w
        cos, sin, xs, bias = self._pos_tables(x.device)
        bq, bk, bv = (t.reshape(b, h, W, w, dh) for t in (q, k, v))
        # rotary + xpos at bucket positions: queries and the "own window" keys sit at positions w..2w-1, the same keys
        # seen from the NEXT window sit at 0..w-1 (local_attention applies the embedding after bucketing)
        cq, sq, xq = cos[w:], sin[w:], xs[w:]
        cp, sp, xp = cos[:w], sin[:w], xs[:w]
        q_rot = bq * cq * xq + _rotate_half(bq) * sq * xq
        k_own = bk * cq / xq + _rotate_half(bk) * sq / xq
        k_prev = bk * cp / xp + _rotate_half(bk) * sp / xp
        zeros = torch.zeros_like(bk[:, :, :1])
        keys = torch.cat((torch.cat((zeros, k_prev[:, :, :-1]), dim=2), k_own), dim=3)    # [b, h, W, 2w, dh]
        vals = torch.cat((torch.cat((zeros, bv[:, :, :-1]), dim=2), bv), dim=3)
        Bp = b * h * W
        key_mask = torch.ones(b, h, W, 2 * w, dtype=torch.bool, device=x.device)
        key_mask[:, :, 0, :w] = False                                              # the first bucket has no look-back
        o, _ = ops.mqa_attn_fwd(q_rot.reshape(Bp, w, dh).to(bf16).contiguous(),
                                keys.reshape(Bp, 2 * w, dh).to(bf16).contiguous(),
                                vals.reshape(Bp, 2 * w, dh).to(bf16).contiguous(), heads=1,
                                key_mask=key_mask.reshape(Bp, 2 * w), causal=True, scale=self.qk_scale,
                                return_lse=False, bias=bias)
        out = o.view(b, h, W * w, dh)[:, :, :n].float()
        gates = F.linear(xn, self.to_v_gate[0].weight, self.to_v_gate[0].bias)      # [b, n, h]
        out = out * gates.transpose(1, 2)[..., None].sigmoid()
        out = out.transpose(1, 2).reshape(b * n, h * dh).to(bf16)
        return ops.gemm(out, wo, out_dtype=f32).view(b, n, dim)


class _FFLinear(nn.Linear):
    pass


class FeedForward(nn.Sequential):
    """local_attention.transformer.FeedForward: LayerNorm, Linear(dim, 2*inner), GEGLU, Dropout, Linear(inner, dim)
    under the upstream Sequential indices 0, 1, (2, 3), 4."""

    def __init__(self, dim, mult=4):
        inner = int(dim * mult * 2 / 3)
        super().__init__(nn.LayerNorm(dim), nn.Linear(dim, inner * 2, bias=False), nn.Identity(), nn.Identity(),
                         nn.Linear(inner, dim, bias=False))
        self.inner = inner
        self._packed = _PackedWeights()

    def forward(self, x):
        b, n, dim = x.shape
        ln, w1, w2 = self[0], self[1], self[4]
        inner, ip = self.inner, (self.inner + 7) // 8 * 8
        pk = self._packed
        w1p = pk.get("w1", [w1.weight], lambda: pack_plain(w1.weight))
        w2p = pk.get("w2", [w2.weight], lambda: pack_plain(w2.weight))               # K padded to a multiple of 8
        xn = F.layer_norm(x.to(f32), (dim,), ln.weight, ln.bias, ln.eps).reshape(b * n, dim).to(bf16)
        hcat = ops.gemm(xn, w1p).float()                                              # [M, 2*inner]
        a, gate = hcat[:, :inner], hcat[:, inner:]
        g = torch.zeros(b * n, ip, device=x.device, dtype=bf16)
        g[:, :inner] = (a * F.gelu(gate)).to(bf16)
        return ops.gemm(g, w2p, out_dtype=f32).view(b, n, dim)


class LocalTransformer(nn.Module):
    """soundstream.py:397-440"""

    def __init__(self, *, dim, depth, heads, window_size, dynamic_pos_bias=False, **kwargs):
        super().__init__()
        if dynamic_pos_bias:
            raise NotImplementedError("attn_dynamic_pos_bias=True (DynamicPositionBias) is not built")
        self.window_size = window_size
        self.pos_bias = None
        self.layers = nn.ModuleList([
            nn.ModuleList([LocalMHA(dim=dim, heads=heads, qk_rmsnorm=True, window_size=window_size,
                                    use_rotary_pos_emb=True, gate_values_per_head=True, use_xpos=True, **kwargs),
                           FeedForward(dim=dim)])
            for _ in range(depth)])

    def forward(self, x):
        x = x.to(f32)
        for attn, ff in self.layers:
            x = attn(x) + x
            x = ff(x) + x
        return x
