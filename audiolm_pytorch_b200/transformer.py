"""Transformer blocks of the AudioLM hot path, running on libalm_b200 (sm_90a).

Class names, constructor kwargs and state_dict keys follow the reference
(/root/reference/audiolm_pytorch/audiolm_pytorch.py:191-560, attend.py:35-146) so checkpoints load
unchanged; the arithmetic is one hand-orchestrated forward/backward over the C-ABI kernels:

    per branch:   [residual step + LayerNorm]  ->  wgmma GEMMs / attention / GEGLU+LN
    end of stack: [residual exit + final LayerNorm]

One forward walk (`Transformer._walk_forward`) serves training, the no-grad forward and KV-cache inference, and one
backward walk serves both residual modes.  Only the residual step differs between them: hyper-connections
(`_HyperStreams`: hc_pre = depth(prev) + width + LayerNorm over a bf16 [M, 4, d] stream, hc_post = depth +
reduce_streams + final LayerNorm) or the plain residual (`_PlainStream`: resid_ln over an fp32 [M, d] stream).

Activations are bf16 with fp32 accumulation (the reference's bf16-autocast numerics), parameters stay
fp32 `nn.Parameter`s; padded bf16 operand copies are rebuilt only when a parameter's version changes.
"""
from __future__ import annotations

import torch
from torch import nn

from . import ops

bf16 = torch.bfloat16
f32 = torch.float32


def exists(v):
    return v is not None


def default(v, d):
    return v if exists(v) else d


def _pad8(n: int) -> int:
    return (n + 7) // 8 * 8


def _check_dropout(p, name="dropout"):
    if not 0.0 <= float(p) < 1.0:
        raise ValueError(f"{name} must be in [0, 1), got {p}")


def _draw_dropout_seed() -> int:
    """one 63-bit seed from torch's default CPU generator: `torch.manual_seed` reproduces a step, and drawing it
    needs no device synchronisation."""
    return int(torch.randint(0, 2 ** 63 - 1, (), dtype=torch.int64))


# ----------------------------------------------------------------------------------------------
# parameter containers (same attribute names -> same state_dict keys as the reference)
# ----------------------------------------------------------------------------------------------
class LayerNorm(nn.Module):
    """gamma parameter + zero `beta` buffer (audiolm_pytorch.py:191-198)."""

    def __init__(self, dim):
        super().__init__()
        self.gamma = nn.Parameter(torch.ones(dim))
        self.register_buffer("beta", torch.zeros(dim))


class Attend(nn.Module):
    """attend.py:35-146.  Holds the configuration; the math runs in alm_mqa_attn_fwd/bwd."""

    def __init__(self, dropout=0.0, causal=False, flash=False):
        super().__init__()
        _check_dropout(dropout)
        self.dropout = dropout
        self.causal = causal
        self.flash = flash

    def forward(self, q, k, v, mask=None, attn_bias=None):
        """q [b h n d], k/v [b j d] -> [b h n d], d = dim_head in {32, 64, 128} (inference helper; training goes
        through Transformer)."""
        b, h, n, d = q.shape
        if exists(attn_bias):
            assert not self.flash, "attention bias not supported for flash attention"  # attend.py:112
            from .rel_pos import as_kernel_bias
            attn_bias = as_kernel_bias(attn_bias.detach())
        qf = q.permute(0, 2, 1, 3).reshape(b, n, h * d).to(bf16).contiguous()
        drop = (self.dropout, _draw_dropout_seed(), 0) if self.training and self.dropout > 0 else None
        o, _ = ops.mqa_attn_fwd(qf, k.to(bf16).contiguous(), v.to(bf16).contiguous(), heads=h, key_mask=mask,
                                causal=self.causal, return_lse=False, bias=attn_bias, dropout=drop)
        return o.reshape(b, n, h, d).permute(0, 2, 1, 3)


class Attention(nn.Module):
    """Parameter holder for audiolm_pytorch.py:264-406 (self-attention, multi-query, dim_head 32, 64 or 128)."""

    def __init__(self, dim, causal=False, dim_head=64, dim_context=None, heads=8, norm_context=False,
                 num_null_kv=0, dropout=0.1, scale=8, flash=False):
        super().__init__()
        if dim_head not in ops.ATTN_HEAD_WIDTHS:
            raise NotImplementedError(f"the sm_90a attention kernels are built for dim_head in {ops.ATTN_HEAD_WIDTHS}, "
                                      f"got {dim_head}")
        if num_null_kv > 0 or exists(dim_context) and dim_context != dim:
            raise NotImplementedError("cross attention / null kv (text conditioning) is out of scope")
        self.heads = heads
        self.dim_head = dim_head
        self.causal = causal
        inner = dim_head * heads
        self.norm = LayerNorm(dim)
        self.to_q = nn.Linear(dim, inner, bias=False)
        self.to_kv = nn.Linear(dim, dim_head * 2, bias=False)
        self.attend = Attend(flash=flash, dropout=dropout, causal=causal)
        self.to_out = nn.Sequential(nn.Linear(inner, dim, bias=False), nn.Dropout(dropout))


class FeedForward(nn.Module):
    """audiolm_pytorch.py:251-260 with the reference's Sequential indices as attribute names
    (0: LayerNorm, 1: Linear(d, 2*inner), 3: LayerNorm(inner), 4: Dropout, 5: Linear(inner, d))."""

    def __init__(self, dim, mult=4, dropout=0.1):
        super().__init__()
        _check_dropout(dropout)
        inner = int(dim * 2 * mult / 3)
        self.inner = inner
        self.add_module("0", LayerNorm(dim))
        self.add_module("1", nn.Linear(dim, inner * 2, bias=False))
        self.add_module("3", LayerNorm(inner))
        self.add_module("4", nn.Dropout(dropout))
        self.add_module("5", nn.Linear(inner, dim, bias=False))


class _StreamNorm(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.gamma = nn.Parameter(torch.zeros(dim))


class HyperConnections(nn.Module):
    """Parameters of hyper_connections.HyperConnections (third party; audiolm_pytorch.py:446-454)."""

    def __init__(self, num_residual_streams, *, dim, branch, layer_index=None):
        super().__init__()
        s = num_residual_streams
        self.num_residual_streams = s
        self.branch = branch
        self.norm = _StreamNorm(dim)
        init = (layer_index if exists(layer_index) else int(torch.randint(0, s, ()).item())) % s
        self.static_beta = nn.Parameter(torch.ones(s))
        a0 = torch.zeros(s, 1)
        a0[init, 0] = 1.0
        self.static_alpha = nn.Parameter(torch.cat((a0, torch.eye(s)), dim=1))
        self.dynamic_alpha_fn = nn.Parameter(torch.zeros(dim, s + 1))
        self.dynamic_alpha_scale = nn.Parameter(torch.ones(()) * 1e-2)
        self.dynamic_beta_fn = nn.Parameter(torch.zeros(dim))
        self.dynamic_beta_scale = nn.Parameter(torch.ones(()) * 1e-2)

    def kernel_params(self):
        return dict(gamma=self.norm.gamma, dyn_alpha=self.dynamic_alpha_fn, dyn_beta=self.dynamic_beta_fn,
                    static_alpha=self.static_alpha, static_beta=self.static_beta,
                    alpha_scale=self.dynamic_alpha_scale, beta_scale=self.dynamic_beta_scale)


class PlainResidual(nn.Module):
    """num_residual_streams == 1: the reference wraps the branch in Residual(branch) (audiolm_pytorch.py:446)."""

    def __init__(self, *, dim=None, branch):
        super().__init__()
        self.branch = branch

    def kernel_params(self):
        return {}


# ----------------------------------------------------------------------------------------------
# bf16 operand cache
# ----------------------------------------------------------------------------------------------
class _PackedWeights:
    """bf16 (zero-padded) GEMM operand copies of fp32 parameters, refreshed when `_version` moves."""

    def __init__(self):
        self._cache = {}
        self.generation = 0  # bumped by clear(): captured CUDA graphs hold raw pointers into these copies

    def clear(self):
        self._cache.clear()
        self.generation += 1

    def get(self, key, params, build):
        ver = tuple((p.data_ptr(), p._version) for p in params)
        hit = self._cache.get(key)
        if hit is not None and hit[0] == ver:
            return hit[1]
        # inference_mode(False): a copy first built inside generate() (torch.inference_mode) must stay usable by the
        # next training forward
        with torch.inference_mode(False), torch.no_grad():
            val = build()
        self._cache[key] = (ver, val)
        return val


def pack_plain(w):
    """[N, K] fp32 -> bf16 [N, pad8(K)]."""
    return ops.cast_pad(w.detach(), _pad8(w.shape[1]))


def pack_w1(w, inner):
    """FeedForward W1 [2*inner, d]: a-rows then gate-rows, each block padded to a multiple of 8 rows."""
    ip = _pad8(inner)
    out = torch.zeros(2 * ip, w.shape[1], device=w.device, dtype=bf16)
    ops.cast_pad(w.detach()[:inner], out=out[:inner])
    ops.cast_pad(w.detach()[inner:], out=out[ip:ip + inner])
    return out


def gemm_block_n(N):
    """BLOCK_N of alm_gemm_bf16 for N output columns: a copy of pick_block_n in csrc/gemm_wgmma.cu"""
    return 64 if N <= 64 else (128 if N <= 128 or (-(-N // 128) * 128) * 10 < (-(-N // 256) * 256) * 9 else 256)


def best_split_k(M, N, K, n_sm=None):
    """split-K factor for weight-gradient GEMMs (few output tiles, very long K); n_sm: SMs of the current device (132,
    the H100 SXM's count, when no device is present: the heuristic itself is host logic)."""
    if n_sm is None:
        n_sm = ops.num_sms() if torch.cuda.is_available() else 132
    tiles = -(-M // 128) * -(-N // gemm_block_n(N))
    kb = -(-K // 64)
    best, best_t = 1, None
    for s in range(1, min(64, kb) + 1):
        t = -(-tiles * s // n_sm) * (-(-kb // s) + 6)  # +6: pipeline fill / epilogue per tile
        if best_t is None or t < best_t:
            best, best_t = s, t
    return best


def wgrad(dy, x, out):
    """out[N, K] (fp32, zero-initialised or accumulating) += dy[M, N]^T x[M, K]."""
    Mtok = dy.shape[0]
    s = best_split_k(dy.shape[1], x.shape[1], Mtok)
    ops.gemm(dy, x, a_mn=True, b_mn=True, out=out, acc_mode=2 if s > 1 else 1, split_k=s)


# ----------------------------------------------------------------------------------------------
# the stack
# ----------------------------------------------------------------------------------------------
class _StackFn(torch.autograd.Function):
    """Whole Transformer stack as one autograd node: explicit forward + backward over C-ABI kernels."""

    @staticmethod
    def forward(ctx, tr, x, mask, bias, drop, want_kv, *params):
        out, kv, saved = tr._walk_forward(x, mask, bias, drop, save=any(ctx.needs_input_grad), want_kv=want_kv)
        ctx.tr = tr
        ctx.saved = saved
        ctx.bias_grad = bias is not None and ctx.needs_input_grad[3]
        ctx.mark_non_differentiable(kv)
        return out, kv

    @staticmethod
    def backward(ctx, dout, _dkv):
        tr = ctx.tr
        S = ctx.saved
        # d(bias) is accumulated by every layer's attention backward (atomic adds over batches and layers)
        S["dbias"] = torch.zeros_like(S["bias"]) if ctx.bias_grad else None
        dx, grads = tr._walk_backward(S, dout)
        dbias = S["dbias"]
        ctx.saved = None
        return (None, dx, None, dbias, None, None, *grads)


# ----------------------------------------------------------------------------------------------
# the residual stream: one step before every branch (`enter` before the first), `exit` after the last.  A step adds the
# previous branch's output Y to the stream and returns the branch input LayerNorm(stream) as `xn` plus the
# un-normalised input `bin`, which feeds to_kv.  The `*_bwd` methods run the steps backward in reverse order; each
# returns the gradient of the previous branch's output (`enter_bwd`: of x).  `hc` / `g_hc` are the hyper-connection
# parameters of the branch's wrapper and their gradient buffers (empty dicts for the plain residual).
# ----------------------------------------------------------------------------------------------
class _HyperStreams:
    """num_residual_streams = S in 2..8: a bf16 [M, S, d] stream; depth (of the previous branch), width and LayerNorm
    are one hc_pre kernel, which writes `bin` only when the branch asks for it.  Saves per step its inputs (R, Y, beta) and the kernel's aux state; the
    exit saves its LN stats."""

    def __init__(self, save, streams):
        self.saved = [] if save else None
        self.S = streams

    def _pre(self, inputs, hc, gamma, want_bin=True):
        self.R, bin_, xn, self.beta, aux = ops.hc_pre_fwd(hc, gamma, **inputs, M=self.M, d=self.d, streams=self.S,
                                                          want_bin=want_bin)
        if self.saved is not None:
            self.saved.append((inputs, aux))
        return xn, bin_

    def enter(self, x2, hc, gamma):
        self.M, self.d = x2.shape
        return self._pre(dict(x_expand=x2), hc, gamma)

    def step(self, Y, hc, gamma, want_bin):
        return self._pre(dict(R_in=self.R, Y=Y, beta_prev=self.beta), hc, gamma, want_bin)

    def exit(self, Y, gamma):
        out, stats = ops.hc_post_fwd(self.R, Y, self.beta, gamma, M=self.M, d=self.d, streams=self.S)
        if self.saved is not None:
            self.saved.append(((self.R, Y, self.beta), stats))
        return out

    def exit_bwd(self, gamma, dout, g_gamma):
        (R, Y, beta), stats = self.saved.pop()
        self.dR, dY, self.dbeta = ops.hc_post_bwd(R, Y, beta, gamma, stats, dout, g_gamma, M=self.M, d=self.d,
                                                  streams=self.S)
        return dY

    def _pre_bwd(self, hc, gamma, g_hc, g_gamma, dxn, dbin, **kw):
        inputs, aux = self.saved.pop()
        return ops.hc_pre_bwd(hc, gamma, g_hc, g_gamma, aux, self.dR, dxn, self.dbeta, dbin_extra=dbin, **inputs, **kw,
                              M=self.M, d=self.d, streams=self.S)

    def step_bwd(self, hc, gamma, g_hc, g_gamma, dxn, dbin=None):
        self.dR, dY, self.dbeta = self._pre_bwd(hc, gamma, g_hc, g_gamma, dxn, dbin)
        return dY

    def enter_bwd(self, hc, gamma, g_hc, g_gamma, dxn, dbin, scale):
        return self._pre_bwd(hc, gamma, g_hc, g_gamma, dxn, dbin, dx_scale=scale)


class _PlainStream:
    """num_residual_streams == 1: an fp32 [M, d] stream r += Y, then LayerNorm (resid_ln); `bin` is a bf16 copy of r,
    written only when the branch asks for it.  Saves per step the updated stream and its LN stats."""

    def __init__(self, save):
        self.saved = [] if save else None
        self.dr = None

    def _fwd(self, r, Y, gamma, **kw):
        self.r, xn, raw, st = ops.resid_ln_fwd(r, Y, gamma, **kw)
        if self.saved is not None:
            self.saved.append((self.r, st))
        return xn, raw

    def enter(self, x2, hc, gamma):
        return self._fwd(x2, None, gamma, want_raw=True)

    def step(self, Y, hc, gamma, want_bin):
        return self._fwd(self.r, Y, gamma, want_raw=want_bin)

    def exit(self, Y, gamma):
        return self._fwd(self.r, Y, gamma)[0]

    def _bwd(self, gamma, g_gamma, dxn, dbin, **kw):
        r, st = self.saved.pop()
        self.dr, dr_b = ops.resid_ln_bwd(r, gamma, st, self.dr, dxn, dbin, g_gamma, **kw)
        return dr_b

    def exit_bwd(self, gamma, dout, g_gamma):
        return self._bwd(gamma, g_gamma, dout, None)

    def step_bwd(self, hc, gamma, g_hc, g_gamma, dxn, dbin=None):
        return self._bwd(gamma, g_gamma, dxn, dbin)

    def enter_bwd(self, hc, gamma, g_hc, g_gamma, dxn, dbin, scale):
        self._bwd(gamma, g_gamma, dxn, dbin, out_scale=scale)
        return self.dr


def _grad_targets(params, direct_ok=False):
    """Where the backward accumulates parameter gradients.

    Default: fresh zero buffers (one flat allocation, one memset) are returned to autograd, so AccumulateGrad,
    parameter hooks (torch DDP / accelerate reducers), `torch.autograd.grad` and optimizer-in-backward all see
    ordinary gradients.

    Opt-in (`Transformer.accumulate_into_grad = True`, set by `parallel.FlatGradBucket.attach`): if every parameter
    owns a contiguous fp32 `.grad`, the kernels accumulate straight into it (wgrad GEMMs in accumulate mode, atomics
    for the small tensors) and autograd is handed `None` — no temporaries, no 130 `grad += tmp` launches.  In that
    mode parameter hooks do NOT fire for the stack's parameters; the bucket's own all-reduce replaces them."""
    direct = direct_ok and all(p.grad is not None and p.grad.dtype == f32 and p.grad.is_contiguous() for p in params)
    if direct:
        return [p.grad for p in params], [None] * len(params)
    total = sum(p.numel() for p in params)
    flat = torch.zeros(total, device=params[0].device, dtype=f32)
    out, off = [], 0
    for p in params:
        out.append(flat[off:off + p.numel()].view(p.shape))
        off += p.numel()
    return out, out


class Transformer(nn.Module):
    """audiolm_pytorch.py:410-560 (self-attention stack with hyper-connections and value residual)."""

    def __init__(self, *, dim, depth, heads, dim_context=None, cross_attend=False, attn_dropout=0.0,
                 ff_dropout=0.0, grad_shrink_alpha=0.1, cond_as_self_attn_prefix=False, rel_pos_bias=True,
                 flash_attn=False, add_value_residual=True, num_residual_streams=4, **kwargs):
        super().__init__()
        rel_pos_bias = rel_pos_bias and not flash_attn
        if cross_attend or cond_as_self_attn_prefix:
            raise NotImplementedError("text / audio conditioning is outside the accelerated hot path")
        if num_residual_streams != 1 and not ops.HC_MIN_STREAMS <= num_residual_streams <= ops.HC_MAX_STREAMS:
            raise NotImplementedError(f"residual-stream kernels are built for num_residual_streams = 1 or "
                                      f"{ops.HC_MIN_STREAMS}..{ops.HC_MAX_STREAMS}")
        _check_dropout(attn_dropout, "attn_dropout")
        _check_dropout(ff_dropout, "ff_dropout")
        if dim % 8 != 0:
            raise ValueError("dim must be a multiple of 8")
        self.dim = dim
        self.depth = depth
        self.heads = heads
        self.dim_context = default(dim_context, dim)
        self.cond_as_self_attn_prefix = False
        self.grad_shrink_alpha = grad_shrink_alpha
        self.num_residual_streams = num_residual_streams
        self.add_value_residual = add_value_residual
        if rel_pos_bias:
            from .rel_pos import RelativePositionBias  # (rel_pos imports heads, which imports this module)
            self.rel_pos_bias = RelativePositionBias(dim=dim // 2, heads=heads)
        else:
            self.rel_pos_bias = None

        self.layers = nn.ModuleList([])
        if num_residual_streams == 1:
            wrap = lambda branch: PlainResidual(dim=dim, branch=branch)  # noqa: E731
        else:
            wrap = lambda branch: HyperConnections(num_residual_streams, dim=dim, branch=branch)  # noqa: E731
        for _ in range(depth):
            self.layers.append(nn.ModuleList([
                wrap(Attention(dim=dim, heads=heads, dropout=attn_dropout, flash=flash_attn, causal=True, **kwargs)),
                None,
                wrap(FeedForward(dim=dim, dropout=ff_dropout)),
            ]))
        self.dim_head = kwargs.get("dim_head", 64)
        self.norm = LayerNorm(dim)
        self._packed = _PackedWeights()
        # called with the layer index once that layer's parameter gradients are complete in the backward
        # (parallel.FlatGradBucket.reduce_range_async overlaps the gradient all-reduce with the remaining layers)
        self.grad_ready_hook = None
        # opt-in direct accumulation into existing `.grad` buffers (see _grad_targets); off by default so that torch
        # DDP / accelerate hooks keep working
        self.accumulate_into_grad = False

    def invalidate_weight_cache(self):
        """drop the bf16 operand copies (they are rebuilt on the next forward, as autocast re-casts weights)."""
        self._packed.clear()

    # ---- parameter plumbing ------------------------------------------------------------------
    def _layer_params(self):
        """Per layer, the parameters the kernels read in four groups: (attention wrapper, attention, feed-forward
        wrapper, feed-forward).  A wrapper group is its hyper-connection parameters (empty for the plain residual).
        `_param_list` is these groups in order, then the final LayerNorm; the backward groups the gradients alike."""
        layout = []
        for attn_w, _, ff_w in self.layers:
            a, f = attn_w.branch, ff_w.branch
            layout.append((attn_w.kernel_params(),
                           dict(ln=a.norm.gamma, wq=a.to_q.weight, wkv=a.to_kv.weight, wo=a.to_out[0].weight),
                           ff_w.kernel_params(),
                           dict(ln=getattr(f, "0").gamma, w1=getattr(f, "1").weight, ln2=getattr(f, "3").gamma,
                                w2=getattr(f, "5").weight)))
        return layout

    def _param_list(self):
        return [p for layer in self._layer_params() for group in layer for p in group.values()] + [self.norm.gamma]

    def _pack_all(self):
        """re-pack the bf16 operand copies of EVERY Linear of the stack in one launch (alm_cast_pad_multi) whenever a
        weight changed (optimizer step) or the cache was invalidated; the destination buffers are persistent, so captured
        decode graphs keep pointing at live memory."""
        pk = self._packed
        items = []  # (cache key, param, source rows view, destination view)
        bufs = self.__dict__.setdefault("_pack_bufs", {})

        def buf(key, rows, cols, dev):
            b = bufs.get(key)
            if b is None or b.shape != (rows, cols) or b.device != dev:
                with torch.inference_mode(False), torch.no_grad():
                    b = bufs[key] = torch.zeros(rows, cols, device=dev, dtype=bf16)
            return b

        for i, (attn_w, _, ff_w) in enumerate(self.layers):
            a, f = attn_w.branch, ff_w.branch
            for name, w in (("q", a.to_q.weight), ("kv", a.to_kv.weight), ("o", a.to_out[0].weight),
                            ("w2", getattr(f, "5").weight)):
                dst = buf((i, name), w.shape[0], _pad8(w.shape[1]), w.device)
                items.append(((i, name), w, w.detach(), dst, dst))
            w1 = getattr(f, "1").weight
            ip = _pad8(f.inner)
            dst = buf((i, "w1"), 2 * ip, w1.shape[1], w1.device)   # a rows then gate rows, each block padded to ip rows
            items.append(((i, "w1"), w1, w1.detach()[:f.inner], dst[:f.inner], dst))
            items.append(((i, "w1"), w1, w1.detach()[f.inner:], dst[ip:ip + f.inner], dst))
        ver_all = tuple((w.data_ptr(), w._version) for _, w, _, _, _ in items)
        if self.__dict__.get("_pack_ver") == (ver_all, pk.generation):
            return
        sig = tuple((src.data_ptr(), d.data_ptr()) for _, _, src, d, _ in items)
        if self.__dict__.get("_pack_sig") != sig:
            rows = [[src.data_ptr(), d.data_ptr(), src.shape[0], src.shape[1], d.shape[1], src.stride(0), d.stride(0)]
                    for _, _, src, d, _ in items]
            with torch.inference_mode(False):
                self.__dict__["_pack_desc"] = torch.tensor(rows, dtype=torch.int64, device=items[0][1].device)
            self.__dict__["_pack_sig"] = sig
        ops.cast_pad_multi(self.__dict__["_pack_desc"])
        for key, w, _, _, full in items:
            pk._cache[key] = (((w.data_ptr(), w._version),), full)
        self.__dict__["_pack_ver"] = (ver_all, pk.generation)

    def _weights(self, i):
        wq_ = self.layers[i][0].branch.to_q.weight
        hit = self._packed._cache.get((i, "q"))
        if wq_.is_cuda and (hit is None or hit[0] != ((wq_.data_ptr(), wq_._version),)):
            self._pack_all()   # stale (optimizer step / invalidate): refresh every layer's copies in one launch
        attn_hc, _, ff_hc = self.layers[i]
        a, f = attn_hc.branch, ff_hc.branch
        pk = self._packed
        w1 = getattr(f, "1").weight
        w2 = getattr(f, "5").weight
        return dict(
            wq=pk.get((i, "q"), [a.to_q.weight], lambda: pack_plain(a.to_q.weight)),
            wkv=pk.get((i, "kv"), [a.to_kv.weight], lambda: pack_plain(a.to_kv.weight)),
            wo=pk.get((i, "o"), [a.to_out[0].weight], lambda: pack_plain(a.to_out[0].weight)),
            w1=pk.get((i, "w1"), [w1], lambda: pack_w1(w1, f.inner)),
            w2=pk.get((i, "w2"), [w2], lambda: pack_plain(w2)),
        )

    # ---- dropout ---------------------------------------------------------------------------------
    def _dropout_plan(self):
        """Per layer: (attention probabilities, attention output, feed-forward) dropout as (p, seed, site) or None.
        None overall in eval mode or when every p is 0: then no seed is drawn and the dropout-free kernels run.
        One seed per forward; site 3 i + k names layer i's k-th dropout, so every mask is independent."""
        if not self.training:
            return None
        ps = [(a.branch.attend.dropout, a.branch.to_out[1].p, getattr(f.branch, "4").p) for a, _, f in self.layers]
        if not any(p > 0 for layer in ps for p in layer):
            return None
        seed = _draw_dropout_seed()
        return [tuple((p, seed, 3 * i + k) if p > 0 else None for k, p in enumerate(layer))
                for i, layer in enumerate(ps)]

    # ---- forward -------------------------------------------------------------------------------
    def forward(self, x, self_attn_mask=None, context=None, context_mask=None, attn_bias=None,
                return_kv_cache=False, kv_cache=None):
        if exists(context):
            raise NotImplementedError("conditioning context is outside the accelerated hot path")
        if not x.is_cuda:
            raise ops._lib.AlmError("Transformer needs CUDA tensors (no CPU fallback)")
        # relative positional bias over the FULL sequence, then the rows of the new tokens (:497-506)
        n = x.shape[1]
        bias = attn_bias if exists(attn_bias) else (self.rel_pos_bias(n, n) if exists(self.rel_pos_bias) else None)
        if exists(bias):
            from .rel_pos import as_kernel_bias
            bias = as_kernel_bias(bias)
        drop = self._dropout_plan()
        if exists(kv_cache):
            # x is the FULL sequence; only the positions after the cache are processed (audiolm_pytorch.py:489-496)
            cache_len = kv_cache.shape[-2]
            if exists(bias):
                bias = bias[:, cache_len:, :]
            with torch.no_grad():
                out, kv, _ = self._walk_forward(x[:, cache_len:], self_attn_mask, bias, drop, save=False,
                                                want_kv=return_kv_cache, kv_cache=kv_cache)
        else:
            out, kv = _StackFn.apply(self, x, self_attn_mask, bias, drop, bool(return_kv_cache), *self._param_list())
        if not return_kv_cache:
            return out
        return out, kv

    def _walk_forward(self, x, mask, bias, drop, *, save, want_kv, kv_cache=None):
        """The stack's forward over the kernels, for both residual modes.  Returns (out, kv, saved):
        kv is the [depth, 2, b, cache_len + n, dim_head] cache tensor when `want_kv` (stacking it is a copy a training step
        does not need), else an empty tensor; `saved` is what `_walk_backward` reads when `save`, else None.
        `kv_cache`: keys / values of the positions before x."""
        b, n, d = x.shape
        M = b * n
        x2 = x.detach().reshape(M, d).to(f32).contiguous()
        S = dict(shape=(b, n, d), x_dtype=x.dtype, mask=ops.pack_key_mask(mask),  # bits, packed once for every layer
                 bias=bias, drop=drop)
        P = self._layer_params()
        res = _PlainStream(save) if self.num_residual_streams == 1 else _HyperStreams(save, self.num_residual_streams)
        xn, bin_ = res.enter(x2, P[0][0], P[0][1]["ln"])
        L, kvs, v_first = [], [], None
        for i, (_, _, hc_f, p_f) in enumerate(P):
            W = self._weights(i)
            d_attn, d_out, d_ff = drop[i] if drop else (None, None, None)
            rec = dict(xn_a=xn, bin_a=bin_)
            Y, k, v, v_first = self._attn_fwd(S, W, rec, v_first, None if kv_cache is None else kv_cache[i], save,
                                              d_attn, d_out)
            if want_kv:
                kvs += (k, v)
            rec["xn_f"], _ = res.step(Y, hc_f, p_f["ln"], want_bin=False)
            Y = self._ff_fwd(i, W, rec, d_ff)
            if save:
                L.append(rec)
            if i + 1 < self.depth:
                xn, bin_ = res.step(Y, P[i + 1][0], P[i + 1][1]["ln"], want_bin=True)
        out = res.exit(Y, self.norm.gamma)
        # kv cache tensor [depth, 2, b, n, dim_head] as the reference returns it (audiolm_pytorch.py:370, 560)
        kv = torch.stack(kvs).unflatten(0, (self.depth, 2)) if want_kv else torch.empty(0, device=x.device, dtype=bf16)
        if not save:
            return out.view(b, n, d), kv, None
        S.update(L=L, res=res)
        return out.view(b, n, d), kv, S

    def _attn_fwd(self, S, W, rec, v_first, cache, save, d_attn, d_out):
        """q / kv projections, value residual, KV cache, attention, output projection (+ their dropout) from
        rec["xn_a"] / rec["bin_a"]; records q, kv, o, lse in `rec`.  Returns (Y, k, v, v_first), k / v including
        the cached positions."""
        b, n, _ = S["shape"]
        H, D = self.heads, self.dim_head
        q = ops.gemm(rec["xn_a"], W["wq"])                 # [M, H*D]
        kv = ops.gemm(rec["bin_a"], W["wkv"])              # [M, 2*D]  (k | v) from the UN-normalised input
        if self.add_value_residual and v_first is not None:
            ops.axpby(kv[:, D:], 0.5, v_first, 0.5, out=kv[:, D:])
        elif self.add_value_residual:
            v_first = kv[:, D:].clone()                    # layer-0 values before any mixing (:355-358)
        k = kv[:, :D].unflatten(0, (b, n))
        v = kv[:, D:].unflatten(0, (b, n))
        if cache is not None:
            k = torch.cat((cache[0].to(bf16), k), dim=1).contiguous()
            v = torch.cat((cache[1].to(bf16), v), dim=1).contiguous()
        # without a backward to feed, the kernel skips writing the row LSE
        o, lse = ops.mqa_attn_fwd(q.view(b, n, H * D), k, v, heads=H, key_mask=S["mask"], causal=True,
                                  return_lse=save, bias=S["bias"], dropout=d_attn)
        o = o.view(b * n, H * D)
        Y = ops.gemm(o, W["wo"])
        if d_out:
            ops.dropout_(Y, *d_out)
        rec.update(q=q, kv=kv, o=o, lse=lse)
        return Y, k, v, v_first

    def _ff_fwd(self, i, W, rec, d_ff):
        """W1 -> GEGLU + LayerNorm (+ dropout) -> W2 from rec["xn_f"]; records h, gn, st in `rec`.  Returns Y."""
        f = self.layers[i][2].branch
        h = ops.gemm(rec["xn_f"], W["w1"])                 # [M, 2*ip]
        gn, st = ops.geglu_ln_fwd(h, getattr(f, "3").gamma, inner=f.inner, inner_pad=_pad8(f.inner), dropout=d_ff)
        rec.update(h=h, gn=gn, st=st)
        return ops.gemm(gn, W["w2"])

    # ---- backward ------------------------------------------------------------------------------
    def _walk_backward(self, S, dout):
        b, n, d = S["shape"]
        M = b * n
        dout = dout.reshape(M, d).to(bf16).contiguous()
        P = self._layer_params()
        grads, returned = _grad_targets(self._param_list(), self.accumulate_into_grad)
        it = iter(grads)
        G = [tuple({k: next(it) for k in group} for group in layer) for layer in P]  # grouped like P
        res = S["res"]
        dY = res.exit_bwd(self.norm.gamma, dout, grads[-1])
        dv_first = None
        for i in reversed(range(self.depth)):
            hc_a, p_a, hc_f, p_f = P[i]
            g_hc_a, g_a, g_hc_f, g_f = G[i]
            W = self._weights(i)
            rec = S["L"][i]
            d_attn, d_out, d_ff = S["drop"][i] if S["drop"] else (None, None, None)
            dxn = self._ff_bwd(i, W, rec, dY, g_f, d_ff)
            dY = res.step_bwd(hc_f, p_f["ln"], g_hc_f, g_f["ln"], dxn)
            dxn, dbin, dv_first = self._attn_bwd(S, i, W, rec, dY, g_a, dv_first, d_attn, d_out)
            if i > 0:
                dY = res.step_bwd(hc_a, p_a["ln"], g_hc_a, g_a["ln"], dxn, dbin)
            else:
                dx = res.enter_bwd(hc_a, p_a["ln"], g_hc_a, g_a["ln"], dxn, dbin, self.grad_shrink_alpha)
            if self.grad_ready_hook is not None and returned[0] is None:
                self.grad_ready_hook(i)  # layer i's gradients are final in their `.grad` buffers (direct accumulation)
        return dx.view(b, n, d).to(S["x_dtype"]), returned

    def _ff_bwd(self, i, W, rec, dY, g, d_ff):
        """backward of _ff_fwd: accumulates the W1 / LN / W2 gradients into `g`, returns d(xn_f)."""
        f = self.layers[i][2].branch
        inner, ip = f.inner, _pad8(f.inner)
        dgn = ops.gemm(dY, W["w2"], b_mn=True)             # [M, ip]
        _wgrad_cols(dY, rec["gn"], g["w2"], inner)
        dh = ops.geglu_ln_bwd(rec["h"], getattr(f, "3").gamma, rec["st"], dgn, g["ln2"], inner=inner, inner_pad=ip,
                              dropout=d_ff)
        dxn = ops.gemm(dh, W["w1"], b_mn=True)             # [M, d]
        wgrad(dh[:, :inner], rec["xn_f"], g["w1"][:inner])
        wgrad(dh[:, ip:ip + inner], rec["xn_f"], g["w1"][inner:])
        return dxn

    def _attn_bwd(self, S, i, W, rec, dY, g, dv_first, d_attn, d_out):
        """backward of _attn_fwd for layer i: accumulates the q / kv / out projection gradients into `g`.
        dv_first: gradient of layer 0's values from the layers above (value residual).  Returns (dxn, dbin, dv_first)."""
        b, n, _ = S["shape"]
        M = b * n
        H, D = self.heads, self.dim_head
        if d_out:
            ops.dropout_(dY, *d_out)  # dY is read by nothing else
        dO = ops.gemm(dY, W["wo"], b_mn=True)              # [M, H*D]
        wgrad(dY, rec["o"], g["wo"])
        kv = rec["kv"]
        k3 = kv[:, :D].unflatten(0, (b, n))
        v3 = kv[:, D:].unflatten(0, (b, n))
        dq, dk, dv = ops.mqa_attn_bwd(rec["q"].view(b, n, H * D), k3, v3, rec["o"].view(b, n, H * D),
                                      dO.view(b, n, H * D), rec["lse"], heads=H, key_mask=S["mask"], causal=True,
                                      bias=S["bias"], dbias=S["dbias"], dropout=d_attn)
        dkv = torch.empty(M, 2 * D, device=dY.device, dtype=bf16)
        ops.axpby(dk.view(M, D), 1.0, None, 0.0, out=dkv[:, :D])
        dv2 = dv.view(M, D)
        if self.add_value_residual and i > 0:
            ops.axpby(dv2, 0.5, None, 0.0, out=dkv[:, D:])
            dv_first = ops.axpby(dv2, 0.5, dv_first, 1.0) if dv_first is not None else ops.axpby(dv2, 0.5, None, 0.0)
        elif self.add_value_residual and dv_first is not None:
            ops.axpby(dv2, 1.0, dv_first, 1.0, out=dkv[:, D:])
        else:
            ops.axpby(dv2, 1.0, None, 0.0, out=dkv[:, D:])
        dq2 = dq.view(M, H * D)
        dxn = ops.gemm(dq2, W["wq"], b_mn=True)
        dbin = ops.gemm(dkv, W["wkv"], b_mn=True)
        wgrad(dq2, rec["xn_a"], g["wq"])
        wgrad(dkv, rec["bin_a"], g["wkv"])
        return dxn, dbin, dv_first


def _wgrad_cols(dy, x_padded, out, cols):
    """weight gradient when the activation operand carries zero padding columns: out [N, cols]."""
    Mtok = dy.shape[0]
    s = best_split_k(dy.shape[1], cols, Mtok)
    ops.gemm(dy, x_padded[:, :cols], a_mn=True, b_mn=True, out=out, acc_mode=2 if s > 1 else 1, split_k=s)
