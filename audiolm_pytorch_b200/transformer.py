"""Transformer blocks of the AudioLM hot path, running on libalm_b200 (sm_90a).

Class names, constructor kwargs and state_dict keys follow the reference
(/root/reference/audiolm_pytorch/audiolm_pytorch.py:191-560, attend.py:35-146) so checkpoints load
unchanged; the arithmetic is one hand-orchestrated forward/backward over the C-ABI kernels:

    per branch:   [hc_pre: depth(prev) + width + LayerNorm]  ->  wgmma GEMMs / attention / GEGLU+LN
    end of stack: [hc_post: depth + reduce_streams + final LayerNorm]

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
        """q [b h n 64], k/v [b j 64] -> [b h n 64] (inference helper; training goes through Transformer)."""
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
    """Parameter holder for audiolm_pytorch.py:264-406 (self-attention, multi-query, dim_head 64)."""

    def __init__(self, dim, causal=False, dim_head=64, dim_context=None, heads=8, norm_context=False,
                 num_null_kv=0, dropout=0.1, scale=8, flash=False):
        super().__init__()
        if dim_head != 64:
            raise NotImplementedError("the sm_90a attention kernels are built for dim_head=64")
        if num_null_kv > 0 or exists(dim_context) and dim_context != dim:
            raise NotImplementedError("cross attention / null kv (text conditioning) is out of scope")
        self.heads = heads
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


HC_KEYS = ("gamma", "dyn_alpha", "dyn_beta", "static_alpha", "static_beta", "alpha_scale", "beta_scale")


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


def best_split_k(M, N, K, n_sm=None):
    """split-K factor for weight-gradient GEMMs (few output tiles, very long K); n_sm: SMs of the current device (132,
    the H100 SXM's count, when no device is present: the heuristic itself is host logic)."""
    if n_sm is None:
        n_sm = ops.num_sms() if torch.cuda.is_available() else 132
    bn = 64 if N <= 64 else (128 if N <= 128 or (-(-N // 128) * 128) * 10 < (-(-N // 256) * 256) * 9 else 256)
    tiles = -(-M // 128) * -(-N // bn)
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
    def forward(ctx, tr, x, mask, bias, drop, *params):
        out, saved = tr._run_forward(x, mask, bias, save=any(ctx.needs_input_grad), drop=drop)
        ctx.tr = tr
        ctx.saved = saved
        ctx.bias_grad = bias is not None and ctx.needs_input_grad[3]
        kv = saved["kv"]
        ctx.mark_non_differentiable(kv)
        return out, kv

    @staticmethod
    def backward(ctx, dout, _dkv):
        tr = ctx.tr
        S = ctx.saved
        # d(bias) is accumulated by every layer's attention backward (atomic adds over batches and layers)
        S["dbias"] = torch.zeros_like(S["bias"]) if ctx.bias_grad else None
        dx, grads = tr._run_backward(S, dout)
        dbias = S["dbias"]
        ctx.saved = None
        return (None, dx, None, dbias, None, *grads)


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
        if num_residual_streams not in (1, 4):
            raise NotImplementedError("residual-stream kernels are built for num_residual_streams in (1, 4)")
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
    def _param_list(self):
        if self.num_residual_streams == 1:
            ps = []
            for attn_w, _, ff_w in self.layers:
                a, f = attn_w.branch, ff_w.branch
                ps += [a.norm.gamma, a.to_q.weight, a.to_kv.weight, a.to_out[0].weight, getattr(f, "0").gamma,
                       getattr(f, "1").weight, getattr(f, "3").gamma, getattr(f, "5").weight]
            ps.append(self.norm.gamma)
            return ps
        ps = []
        for attn_hc, _, ff_hc in self.layers:
            a, f = attn_hc.branch, ff_hc.branch
            ps += [*attn_hc.kernel_params().values(), a.norm.gamma, a.to_q.weight, a.to_kv.weight,
                   a.to_out[0].weight]
            ps += [*ff_hc.kernel_params().values(), getattr(f, "0").gamma, getattr(f, "1").weight,
                   getattr(f, "3").gamma, getattr(f, "5").weight]
        ps.append(self.norm.gamma)
        return ps

    PER_LAYER = 2 * len(HC_KEYS) + 4 + 4

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
            if exists(bias):
                bias = bias[:, kv_cache.shape[-2]:, :]
            out, kv = self._forward_cached(x, self_attn_mask, kv_cache, bias, drop)
        else:
            # the [depth, 2, b, n, 64] cache tensor is only materialised when the caller asks for it (a training
            # step does not: stacking it costs six strided copies per forward)
            self._want_kv = bool(return_kv_cache)
            out, kv = _StackFn.apply(self, x, self_attn_mask, bias, drop, *self._param_list())
        if not return_kv_cache:
            return out
        return out, kv

    def _run_forward(self, x, mask, bias, save, drop=None):
        if self.num_residual_streams == 1:
            return self._run_forward_plain(x, mask, bias, save, drop=drop)
        b, n, d = x.shape
        M = b * n
        H = self.heads
        x2 = x.detach().reshape(M, d).to(f32).contiguous()
        mask_u8 = ops.pack_key_mask(mask)  # bits, packed once for every layer and the backward
        L = []
        hc0 = self.layers[0][0]
        R, bin_, xn, beta, aux = ops.hc_pre_fwd(hc0.kernel_params(), hc0.branch.norm.gamma, x_expand=x2, M=M, d=d)
        v_first = None
        kvs = []
        for i, (attn_hc, _, ff_hc) in enumerate(self.layers):
            W = self._weights(i)
            f = ff_hc.branch
            inner, ip = f.inner, _pad8(f.inner)
            d_attn, d_out, d_ff = drop[i] if drop else (None, None, None)
            rec = dict(R_a=R, bin_a=bin_, xn_a=xn, beta_a=beta, aux_a=aux)
            q = ops.gemm(xn, W["wq"])                      # [M, H*64]
            kv = ops.gemm(bin_, W["wkv"])                  # [M, 128]  (k | v) from the UN-normalised input
            if self.add_value_residual and v_first is not None:
                ops.axpby(kv[:, 64:], 0.5, v_first, 0.5, out=kv[:, 64:])
            elif self.add_value_residual:
                v_first = kv[:, 64:].clone()               # layer-0 values before any mixing (:355-358)
            k3 = kv[:, :64].unflatten(0, (b, n))
            v3 = kv[:, 64:].unflatten(0, (b, n))
            o, lse = ops.mqa_attn_fwd(q.view(b, n, H * 64), k3, v3, heads=H, key_mask=mask_u8, causal=True, bias=bias,
                                      dropout=d_attn)
            o2 = o.view(M, H * 64)
            Y = ops.gemm(o2, W["wo"])
            if d_out:
                ops.dropout_(Y, *d_out)
            rec.update(q=q, kv=kv, o=o2, lse=lse, Y_a=Y)
            kvs.append(kv)
            R2, bin2, xn2, beta2, aux2 = ops.hc_pre_fwd(ff_hc.kernel_params(), getattr(f, "0").gamma, R_in=R, Y=Y,
                                                        beta_prev=beta, M=M, d=d)
            h = ops.gemm(xn2, W["w1"])                     # [M, 2*ip]
            gn, st = ops.geglu_ln_fwd(h, getattr(f, "3").gamma, inner=inner, inner_pad=ip, dropout=d_ff)
            Y2 = ops.gemm(gn, W["w2"])
            rec.update(R_f=R2, xn_f=xn2, beta_f=beta2, aux_f=aux2, h=h, gn=gn, st=st, Y_f=Y2)
            L.append(rec)
            if i + 1 < self.depth:
                nxt = self.layers[i + 1][0]
                R, bin_, xn, beta, aux = ops.hc_pre_fwd(nxt.kernel_params(), nxt.branch.norm.gamma, R_in=R2, Y=Y2,
                                                        beta_prev=beta2, M=M, d=d)
        last = L[-1]
        out, stats = ops.hc_post_fwd(last["R_f"], last["Y_f"], last["beta_f"], self.norm.gamma, M=M, d=d)
        # kv cache tensor [depth, 2, b, n, 64] as the reference returns it (audiolm_pytorch.py:370, 560)
        if getattr(self, "_want_kv", True):
            kv_t = torch.stack([kv.view(b, n, 2, 64).permute(2, 0, 1, 3) for kv in kvs])
        else:
            kv_t = torch.empty(0, device=x.device, dtype=bf16)
        saved = dict(kv=kv_t)
        if save:
            saved.update(L=L, x2=x2, mask=mask_u8, bias=bias, stats=stats, shape=(b, n, d), x_dtype=x.dtype, drop=drop)
        return out.view(b, n, d), saved

    # ---- backward ------------------------------------------------------------------------------
    def _run_backward(self, S, dout):
        if self.num_residual_streams == 1:
            return self._run_backward_plain(S, dout)
        b, n, d = S["shape"]
        M = b * n
        H = self.heads
        dev = dout.device
        L = S["L"]
        dout = dout.reshape(M, d).to(bf16).contiguous()
        params = self._param_list()
        grads, returned = _grad_targets(params, self.accumulate_into_grad)
        PL = self.PER_LAYER
        nk = len(HC_KEYS)

        def slot(i):
            g = grads[i * PL:(i + 1) * PL]
            a_hc = dict(zip(HC_KEYS, g[:nk]))
            g_ln_a, g_wq, g_wkv, g_wo = g[nk:nk + 4]
            f_hc = dict(zip(HC_KEYS, g[nk + 4:2 * nk + 4]))
            g_ln_f, g_w1, g_ln2, g_w2 = g[2 * nk + 4:]
            return a_hc, g_ln_a, g_wq, g_wkv, g_wo, f_hc, g_ln_f, g_w1, g_ln2, g_w2

        last = L[-1]
        dR, dY, dbeta = ops.hc_post_bwd(last["R_f"], last["Y_f"], last["beta_f"], self.norm.gamma, S["stats"], dout,
                                        grads[-1], M=M, d=d)
        dv_first = None
        dx = None
        for i in reversed(range(self.depth)):
            attn_hc, _, ff_hc = self.layers[i]
            a, f = attn_hc.branch, ff_hc.branch
            inner, ip = f.inner, _pad8(f.inner)
            W = self._weights(i)
            rec = L[i]
            a_hc, g_ln_a, g_wq, g_wkv, g_wo, f_hc, g_ln_f, g_w1, g_ln2, g_w2 = slot(i)
            d_attn, d_out, d_ff = S["drop"][i] if S["drop"] else (None, None, None)
            # ---- feed-forward branch ----
            dgn = ops.gemm(dY, W["w2"], b_mn=True)                       # [M, ip]
            _wgrad_cols(dY, rec["gn"], g_w2, inner)
            dh = ops.geglu_ln_bwd(rec["h"], getattr(f, "3").gamma, rec["st"], dgn, g_ln2, inner=inner, inner_pad=ip,
                                  dropout=d_ff)
            dxn_f = ops.gemm(dh, W["w1"], b_mn=True)                     # [M, d]
            wgrad(dh[:, :inner], rec["xn_f"], g_w1[:inner])
            wgrad(dh[:, ip:ip + inner], rec["xn_f"], g_w1[inner:])
            dR_a, dY_a, dbeta_a = ops.hc_pre_bwd(ff_hc.kernel_params(), getattr(f, "0").gamma, f_hc, g_ln_f,
                                                 rec["aux_f"], dR, dxn_f, dbeta, R_in=rec["R_a"], Y=rec["Y_a"],
                                                 beta_prev=rec["beta_a"], M=M, d=d)
            # ---- attention branch ----
            if d_out:
                ops.dropout_(dY_a, *d_out)
            dO = ops.gemm(dY_a, W["wo"], b_mn=True)                      # [M, H*64]
            wgrad(dY_a, rec["o"], g_wo)
            kv = rec["kv"]
            k3 = kv[:, :64].unflatten(0, (b, n))
            v3 = kv[:, 64:].unflatten(0, (b, n))
            dq, dk, dv = ops.mqa_attn_bwd(rec["q"].view(b, n, H * 64), k3, v3, rec["o"].view(b, n, H * 64),
                                          dO.view(b, n, H * 64), rec["lse"], heads=H, key_mask=S["mask"], causal=True,
                                          bias=S["bias"], dbias=S["dbias"], dropout=d_attn)
            dkv = torch.empty(M, 128, device=dev, dtype=bf16)
            ops.axpby(dk.view(M, 64), 1.0, None, 0.0, out=dkv[:, :64])
            dv2 = dv.view(M, 64)
            if self.add_value_residual and i > 0:
                ops.axpby(dv2, 0.5, None, 0.0, out=dkv[:, 64:])
                dv_first = ops.axpby(dv2, 0.5, dv_first, 1.0) if dv_first is not None else ops.axpby(dv2, 0.5, None, 0.0)
            elif self.add_value_residual and dv_first is not None:
                ops.axpby(dv2, 1.0, dv_first, 1.0, out=dkv[:, 64:])
            else:
                ops.axpby(dv2, 1.0, None, 0.0, out=dkv[:, 64:])
            dq2 = dq.view(M, H * 64)
            dxn_a = ops.gemm(dq2, W["wq"], b_mn=True)
            dbin_a = ops.gemm(dkv, W["wkv"], b_mn=True)
            wgrad(dq2, rec["xn_a"], g_wq)
            wgrad(dkv, rec["bin_a"], g_wkv)
            if i > 0:
                prev = L[i - 1]
                dR, dY, dbeta = ops.hc_pre_bwd(attn_hc.kernel_params(), a.norm.gamma, a_hc, g_ln_a, rec["aux_a"], dR_a,
                                               dxn_a, dbeta_a, dbin_extra=dbin_a, R_in=prev["R_f"], Y=prev["Y_f"],
                                               beta_prev=prev["beta_f"], M=M, d=d)
            else:
                dx = ops.hc_pre_bwd(attn_hc.kernel_params(), a.norm.gamma, a_hc, g_ln_a, rec["aux_a"], dR_a, dxn_a,
                                    dbeta_a, dbin_extra=dbin_a, x_expand=S["x2"], dx_scale=self.grad_shrink_alpha,
                                    M=M, d=d)
            if self.grad_ready_hook is not None and returned[0] is None:
                self.grad_ready_hook(i)  # layer i's gradients are final in their `.grad` buffers (direct accumulation)
        return dx.view(b, n, d).to(S["x_dtype"]), returned


    # ---- num_residual_streams == 1: plain residual stream (fp32) ---------------------------------
    def _attn_branch_fwd(self, i, xn, raw, b, n, mask_u8, v_first, cache=None, bias=None, d_attn=None, d_out=None):
        """q/kv projections, value residual, (optional KV cache), attention, output projection (+ their dropout)."""
        H = self.heads
        W = self._weights(i)
        M = b * n
        q = ops.gemm(xn, W["wq"])
        kv = ops.gemm(raw, W["wkv"])
        if self.add_value_residual and v_first is not None:
            ops.axpby(kv[:, 64:], 0.5, v_first, 0.5, out=kv[:, 64:])
        elif self.add_value_residual:
            v_first = kv[:, 64:].clone()
        k3 = kv[:, :64].unflatten(0, (b, n))
        v3 = kv[:, 64:].unflatten(0, (b, n))
        if cache is not None:
            k3 = torch.cat((cache[0].to(bf16), k3), dim=1).contiguous()
            v3 = torch.cat((cache[1].to(bf16), v3), dim=1).contiguous()
        o, lse = ops.mqa_attn_fwd(q.view(b, n, H * 64), k3, v3, heads=H, key_mask=mask_u8, causal=True, bias=bias,
                                  dropout=d_attn)
        o2 = o.view(M, H * 64)
        Y = ops.gemm(o2, W["wo"])
        if d_out:
            ops.dropout_(Y, *d_out)
        return q, kv, o2, lse, Y, v_first, torch.stack((k3, v3))

    def _run_forward_plain(self, x, mask, bias, save, kv_cache=None, drop=None):
        b, n, d = x.shape
        M = b * n
        r = x.detach().reshape(M, d).to(f32).contiguous()
        x2 = r
        mask_u8 = ops.pack_key_mask(mask)  # bits, packed once for every layer and the backward
        L, kvs = [], []
        a0 = self.layers[0][0].branch
        r, xn, raw, st = ops.resid_ln_fwd(r, None, a0.norm.gamma, want_raw=True)
        v_first = None
        for i, (attn_w, _, ff_w) in enumerate(self.layers):
            a, f = attn_w.branch, ff_w.branch
            W = self._weights(i)
            inner, ip = f.inner, _pad8(f.inner)
            d_attn, d_out, d_ff = drop[i] if drop else (None, None, None)
            q, kv, o2, lse, Y, v_first, kv_t = self._attn_branch_fwd(
                i, xn, raw, b, n, mask_u8, v_first, None if kv_cache is None else kv_cache[i], bias, d_attn, d_out)
            kvs.append(kv_t)
            r_f, xn_f, _, st_f = ops.resid_ln_fwd(r, Y, getattr(f, "0").gamma)
            h = ops.gemm(xn_f, W["w1"])
            gn, stg = ops.geglu_ln_fwd(h, getattr(f, "3").gamma, inner=inner, inner_pad=ip, dropout=d_ff)
            Y2 = ops.gemm(gn, W["w2"])
            L.append(dict(r_a=r, st_a=st, xn_a=xn, raw_a=raw, q=q, kv=kv, o=o2, lse=lse, r_f=r_f, st_f=st_f, xn_f=xn_f,
                          h=h, gn=gn, stg=stg))
            if i + 1 < self.depth:
                nxt = self.layers[i + 1][0].branch
                r, xn, raw, st = ops.resid_ln_fwd(r_f, Y2, nxt.norm.gamma, want_raw=True)
        r_last, out, _, st_last = ops.resid_ln_fwd(r_f, Y2, self.norm.gamma)
        saved = dict(kv=torch.stack(kvs))
        if save:
            saved.update(L=L, mask=mask_u8, bias=bias, r_last=r_last, st_last=st_last, shape=(b, n, d),
                         x_dtype=x.dtype, drop=drop)
        return out.view(b, n, d), saved

    def _run_backward_plain(self, S, dout):
        b, n, d = S["shape"]
        M = b * n
        H = self.heads
        dev = dout.device
        L = S["L"]
        dout = dout.reshape(M, d).to(bf16).contiguous()
        params = self._param_list()
        grads, returned = _grad_targets(params, self.accumulate_into_grad)
        dr, dr_b = ops.resid_ln_bwd(S["r_last"], self.norm.gamma, S["st_last"], None, dout, None, grads[-1])
        dv_first = None
        for i in reversed(range(self.depth)):
            attn_w, _, ff_w = self.layers[i]
            a, f = attn_w.branch, ff_w.branch
            inner, ip = f.inner, _pad8(f.inner)
            W = self._weights(i)
            rec = L[i]
            g_ln_a, g_wq, g_wkv, g_wo, g_ln_f, g_w1, g_ln2, g_w2 = grads[i * 8:(i + 1) * 8]
            d_attn, d_out, d_ff = S["drop"][i] if S["drop"] else (None, None, None)
            # feed-forward branch (its output gradient is the residual-stream gradient)
            dgn = ops.gemm(dr_b, W["w2"], b_mn=True)
            _wgrad_cols(dr_b, rec["gn"], g_w2, inner)
            dh = ops.geglu_ln_bwd(rec["h"], getattr(f, "3").gamma, rec["stg"], dgn, g_ln2, inner=inner, inner_pad=ip,
                                  dropout=d_ff)
            dxn_f = ops.gemm(dh, W["w1"], b_mn=True)
            wgrad(dh[:, :inner], rec["xn_f"], g_w1[:inner])
            wgrad(dh[:, ip:ip + inner], rec["xn_f"], g_w1[inner:])
            dr, dr_b = ops.resid_ln_bwd(rec["r_f"], getattr(f, "0").gamma, rec["st_f"], dr, dxn_f, None, g_ln_f)
            # attention branch
            if d_out:
                ops.dropout_(dr_b, *d_out)  # dr_b is read by nothing else
            dO = ops.gemm(dr_b, W["wo"], b_mn=True)
            wgrad(dr_b, rec["o"], g_wo)
            kv = rec["kv"]
            k3 = kv[:, :64].unflatten(0, (b, n))
            v3 = kv[:, 64:].unflatten(0, (b, n))
            dq, dk, dv = ops.mqa_attn_bwd(rec["q"].view(b, n, H * 64), k3, v3, rec["o"].view(b, n, H * 64),
                                          dO.view(b, n, H * 64), rec["lse"], heads=H, key_mask=S["mask"], causal=True,
                                          bias=S["bias"], dbias=S["dbias"], dropout=d_attn)
            dkv = torch.empty(M, 128, device=dev, dtype=bf16)
            ops.axpby(dk.view(M, 64), 1.0, None, 0.0, out=dkv[:, :64])
            dv2 = dv.view(M, 64)
            if self.add_value_residual and i > 0:
                ops.axpby(dv2, 0.5, None, 0.0, out=dkv[:, 64:])
                dv_first = ops.axpby(dv2, 0.5, dv_first, 1.0) if dv_first is not None else ops.axpby(dv2, 0.5, None, 0.0)
            elif self.add_value_residual and dv_first is not None:
                ops.axpby(dv2, 1.0, dv_first, 1.0, out=dkv[:, 64:])
            else:
                ops.axpby(dv2, 1.0, None, 0.0, out=dkv[:, 64:])
            dq2 = dq.view(M, H * 64)
            dxn_a = ops.gemm(dq2, W["wq"], b_mn=True)
            dbin_a = ops.gemm(dkv, W["wkv"], b_mn=True)
            wgrad(dq2, rec["xn_a"], g_wq)
            wgrad(dkv, rec["raw_a"], g_wkv)
            dr, dr_b = ops.resid_ln_bwd(rec["r_a"], a.norm.gamma, rec["st_a"], dr, dxn_a, dbin_a, g_ln_a,
                                        out_scale=self.grad_shrink_alpha if i == 0 else 1.0)
        return dr.view(b, n, d).to(S["x_dtype"]), returned

    # ---- incremental (KV-cache) inference ------------------------------------------------------
    @torch.no_grad()
    def _forward_cached(self, x, mask, kv_cache, bias=None, drop=None):
        """x is the FULL sequence; only x[:, cache_len:] is processed (audiolm_pytorch.py:489-496)."""
        cache_len = kv_cache.shape[-2]
        x = x[:, cache_len:]
        if self.num_residual_streams == 1:
            out, saved = self._run_forward_plain(x, mask, bias, save=False, kv_cache=kv_cache, drop=drop)
            return out, saved["kv"]
        b, n, d = x.shape
        M = b * n
        H = self.heads
        x2 = x.reshape(M, d).to(f32).contiguous()
        mask_u8 = ops.pack_key_mask(mask)  # bits, packed once for every layer and the backward
        hc0 = self.layers[0][0]
        R, bin_, xn, beta, _ = ops.hc_pre_fwd(hc0.kernel_params(), hc0.branch.norm.gamma, x_expand=x2, M=M, d=d)
        v_first = None
        new_cache = []
        for i, (attn_hc, _, ff_hc) in enumerate(self.layers):
            W = self._weights(i)
            f = ff_hc.branch
            inner, ip = f.inner, _pad8(f.inner)
            d_attn, d_out, d_ff = drop[i] if drop else (None, None, None)
            q = ops.gemm(xn, W["wq"])
            kv = ops.gemm(bin_, W["wkv"])
            if self.add_value_residual and v_first is not None:
                ops.axpby(kv[:, 64:], 0.5, v_first, 0.5, out=kv[:, 64:])
            elif self.add_value_residual:
                v_first = kv[:, 64:].clone()
            ck, cv = kv_cache[i][0].to(bf16), kv_cache[i][1].to(bf16)
            k_all = torch.cat((ck, kv[:, :64].unflatten(0, (b, n))), dim=1).contiguous()
            v_all = torch.cat((cv, kv[:, 64:].unflatten(0, (b, n))), dim=1).contiguous()
            new_cache.append(torch.stack((k_all, v_all)))
            o, _ = ops.mqa_attn_fwd(q.view(b, n, H * 64), k_all, v_all, heads=H, key_mask=mask_u8, causal=True,
                                    return_lse=False, bias=bias, dropout=d_attn)
            Y = ops.gemm(o.view(M, H * 64), W["wo"])
            if d_out:
                ops.dropout_(Y, *d_out)
            R2, _, xn2, beta2, _ = ops.hc_pre_fwd(ff_hc.kernel_params(), getattr(f, "0").gamma, R_in=R, Y=Y,
                                                  beta_prev=beta, M=M, d=d)
            h = ops.gemm(xn2, W["w1"])
            gn, _ = ops.geglu_ln_fwd(h, getattr(f, "3").gamma, inner=inner, inner_pad=ip, dropout=d_ff)
            Y2 = ops.gemm(gn, W["w2"])
            if i + 1 < self.depth:
                nxt = self.layers[i + 1][0]
                R, bin_, xn, beta, _ = ops.hc_pre_fwd(nxt.kernel_params(), nxt.branch.norm.gamma, R_in=R2, Y=Y2,
                                                      beta_prev=beta2, M=M, d=d)
        out, _ = ops.hc_post_fwd(R2, Y2, beta2, self.norm.gamma, M=M, d=d)
        return out.view(b, n, d), torch.stack(new_cache)


def _wgrad_cols(dy, x_padded, out, cols):
    """weight gradient when the activation operand carries zero padding columns: out [N, cols]."""
    Mtok = dy.shape[0]
    s = best_split_k(dy.shape[1], cols, Mtok)
    ops.gemm(dy, x_padded[:, :cols], a_mn=True, b_mn=True, out=out, acc_mode=2 if s > 1 else 1, split_k=s)
