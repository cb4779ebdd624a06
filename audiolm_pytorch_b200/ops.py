"""Python faces of the C-ABI kernels (raw ops; the autograd wiring lives in transformer.py / heads.py / rel_pos.py).

Every function here launches hand-written sm_90a kernels from libalm_b200.so on the current CUDA
stream.  No function has a CPU or stock-PyTorch implementation.
"""
from __future__ import annotations

import ctypes
import functools
import math

import torch

from . import _lib

_SMS: dict[int, int] = {}


def num_sms(device=None) -> int:
    """SM count of a CUDA device (the current one by default) for the launch heuristics: 132 on an H100 SXM, 114 on
    an H100 PCIe."""
    idx = None if device is None else torch.device(device).index
    if idx is None:
        idx = torch.cuda.current_device()
    if idx not in _SMS:
        _SMS[idx] = torch.cuda.get_device_properties(idx).multi_processor_count
    return _SMS[idx]


bf16 = torch.bfloat16
f32 = torch.float32


# ---- optional in-stream kernel timing (bench.py roofline): CUDA events bracket each tagged launch -----
_PROFILE = None
PROFILE_SHAPES = False  # per-shape GEMM classes (tools/profile_step.py)


def profile_start():
    """begin collecting (start_event, end_event, work) tuples per kernel class on the current stream."""
    global _PROFILE
    _PROFILE = {}


def profile_stop():
    """-> {cls: (total_ms, total_work, launches)}; synchronises the device."""
    global _PROFILE
    prof, _PROFILE = _PROFILE, None
    torch.cuda.synchronize()
    out = {}
    for cls, recs in (prof or {}).items():
        ms = sum(a.elapsed_time(b) for a, b, _ in recs)
        out[cls] = (ms, sum(w for _, _, w in recs), len(recs))
    return out


CLASS_UNIT = {}  # kernel class -> "flop" (tensor-bound classes) or "byte" (HBM-bound classes: algorithmic bytes)


class _timed:
    def __init__(self, cls, work, unit="flop"):
        self.cls, self.work = cls, work
        CLASS_UNIT[cls] = unit

    def __enter__(self):
        if _PROFILE is not None:
            self.a = torch.cuda.Event(enable_timing=True)
            self.b = torch.cuda.Event(enable_timing=True)
            self.a.record()
        return self

    def __exit__(self, *exc):
        if _PROFILE is not None:
            self.b.record()
            _PROFILE.setdefault(self.cls, []).append((self.a, self.b, self.work))
        return False


def _check_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise _lib.AlmError("audiolm_pytorch_b200 ops need CUDA tensors (no CPU fallback)")


def gemm(a, b, *, a_mn=False, b_mn=False, out=None, out_dtype=bf16, alpha=1.0, bias=None,
         acc_mode=0, split_k=1, cls="gemm_bf16_wgmma"):
    """out[b,m,n] (op)= alpha * sum_k A(m,k) B(n,k) (+bias[n]).   bf16 operands, fp32 accumulate.

    a: [(batch,) M, K] (a_mn=False) or [(batch,) K, M] (a_mn=True); row stride must be a multiple of 8.
    b: [(batch,) N, K] (b_mn=False) or [(batch,) K, N] (b_mn=True).
    Reference counterpart: nn.Linear / einsum calls listed in include/alm_b200.h.
    """
    _check_cuda(a, b, out, bias)
    assert a.dtype == bf16 and b.dtype == bf16, "gemm operands must be bf16"
    batched = a.dim() == 3
    if not batched:
        a3, b3 = a.unsqueeze(0), b.unsqueeze(0)
    else:
        a3, b3 = a, b
    assert a3.stride(-1) == 1 and b3.stride(-1) == 1
    nb = a3.shape[0]
    assert b3.shape[0] == nb
    if a_mn:
        K, M = a3.shape[1], a3.shape[2]
    else:
        M, K = a3.shape[1], a3.shape[2]
    if b_mn:
        Kb, N = b3.shape[1], b3.shape[2]
    else:
        N, Kb = b3.shape[1], b3.shape[2]
    assert K == Kb, f"K mismatch {K} vs {Kb}"
    if out is None:
        out = torch.empty((nb, M, N) if batched else (M, N), device=a.device, dtype=out_dtype)
        assert acc_mode == 0
    o3 = out.unsqueeze(0) if out.dim() == 2 else out
    assert o3.shape == (nb, M, N) and o3.stride(-1) == 1
    assert o3.dtype in (bf16, f32)
    if bias is not None:
        assert bias.dtype == f32 and bias.numel() == N and bias.is_contiguous()
    if _PROFILE is not None and PROFILE_SHAPES:
        cls += f" M{M} N{N} K{K} b{nb} {'mn' if a_mn else 'k'}{'mn' if b_mn else 'k'} s{split_k}"
    with _timed(cls, 2.0 * M * N * K * nb):
        _lib.call(
            "alm_gemm_bf16",
            a3, int(a_mn), a3.stride(1), a3.stride(0) if nb > 1 else 0,
            b3, int(b_mn), b3.stride(1), b3.stride(0) if nb > 1 else 0,
            o3, int(o3.dtype == f32), o3.stride(1), o3.stride(0) if nb > 1 else 0,
            M, N, K, nb, float(alpha), bias, int(acc_mode), int(split_k),
        )
    return out


def _check_bias(bias, heads, n_q, n_k):
    """bias: fp32 [heads, n_q, ld] view with ld >= n_k, ld % 4 == 0 (see `pad_bias`)."""
    assert bias.dtype == f32 and bias.dim() == 3 and bias.shape[0] == heads and bias.shape[1] == n_q
    assert bias.shape[2] >= n_k and bias.stride(2) == 1 and bias.stride(1) % 4 == 0 and bias.stride(0) % 4 == 0
    return bias.stride(0), bias.stride(1)


def _ptr_array(tensors):
    import ctypes
    arr = (ctypes.c_void_p * len(tensors))(*[t.data_ptr() for t in tensors])
    return arr


def embed_gather(src, tables, d):
    """src int32 [M, 2] ((table_id << 24) | row, -1 = none), tables: list of fp32 [rows_k, d] -> fp32 [M, d]"""
    _check_cuda(src, *tables)
    assert src.dtype == torch.int32 and src.is_contiguous() and src.shape[1] == 2
    assert all(t.dtype == f32 and t.is_contiguous() and t.shape[-1] == d for t in tables)
    M = src.shape[0]
    out = torch.empty(M, d, device=src.device, dtype=f32)
    import ctypes
    _lib.call("alm_embed_gather", ctypes.cast(_ptr_array(tables), ctypes.c_void_p), len(tables), src, out, M, d)
    return out


def embed_scatter(src, grad_tables, dout):
    """backward of embed_gather: grad_tables[id][row] += dout[m] (grad tables zeroed by the caller)"""
    _check_cuda(src, dout, *grad_tables)
    M, d = dout.shape
    assert dout.dtype == f32 and dout.is_contiguous()
    import ctypes
    _lib.call("alm_embed_scatter", ctypes.cast(_ptr_array(grad_tables), ctypes.c_void_p), len(grad_tables), src, dout,
              M, d)


class PackedKeyMask:
    """key mask in the bit layout the attention kernels read (alm_pack_key_mask): uint32 [b, 4 * ceil(n_k / 128)]"""

    def __init__(self, bits, n_k):
        self.bits, self.n_k = bits, n_k


def pack_key_mask(key_mask):
    """bool / uint8 [b, n_k] (True = attend) -> PackedKeyMask; pack once per forward and hand the result to every
    layer's mqa_attn_fwd / mqa_attn_bwd."""
    if key_mask is None or isinstance(key_mask, PackedKeyMask):
        return key_mask
    _check_cuda(key_mask)
    m = key_mask.to(torch.uint8).contiguous()
    b, n_k = m.shape
    bits = torch.empty(b, (n_k + 127) // 128 * 4, device=m.device, dtype=torch.int32)
    _lib.call("alm_pack_key_mask", m, bits, b, n_k)
    return PackedKeyMask(bits, n_k)


def _drop_args(dropout):
    """(p, seed, site) or None -> the (dropout_p, seed, site) C arguments; p == 0 selects the dropout-free kernels."""
    if dropout is None:
        return 0.0, 0, 0
    p, seed, site = dropout
    if not 0.0 <= p < 1.0:
        raise ValueError(f"dropout probability must be in [0, 1), got {p}")
    return float(p), int(seed) & 0xFFFFFFFFFFFFFFFF, int(site) & 0xFFFFFFFF


def dropout_(x, p, seed, site):
    """In place: x[r, c] = keep(seed, site, r, c) ? x[r, c] / (1 - p) : 0 for a bf16 [M, C] tensor (C % 8 == 0,
    unit column stride).  The mask is a pure function of (seed, site, r, c), so calling it again on the gradient with
    the same arguments is the backward."""
    _check_cuda(x)
    assert x.dtype == bf16 and x.dim() == 2 and x.stride(1) == 1
    M, C = x.shape
    with _timed("dropout_bf16", M * C * 4, "byte"):
        _lib.call("alm_dropout_bf16", x, x.stride(0), M, C, *_drop_args((p, seed, site)))
    return x


ATTN_HEAD_WIDTHS = (32, 64, 128)


def _head_width(k):
    """dim_head of an attention call = the width of its shared key head; the kernels are built for three widths"""
    D = k.shape[-1]
    if D not in ATTN_HEAD_WIDTHS:
        raise NotImplementedError(f"the sm_90a attention kernels are built for dim_head in {ATTN_HEAD_WIDTHS}, got {D}")
    return D


def mqa_attn_fwd(q, k, v, *, heads, key_mask=None, causal=True, scale=None, return_lse=True, bias=None,
                 dropout=None):
    """Multi-query attention forward (attend.py:69-146).

    q: [b, n_q, heads*D] bf16 (last dim contiguous; may be a column slice of a wider buffer)
    k, v: [b, n_k, D] bf16 (one shared head of width D = dim_head in {32, 64, 128}, read from k);  key_mask: [b, n_k] bool/uint8 (True = attend) or None.
    Queries are right-aligned against keys (query i sees keys <= i + n_k - n_q) when causal.
    bias: optional fp32 [heads, n_q, >=n_k] additive score bias shared by the batch (attend.py:122-124).
    dropout: optional (p, seed, site): dropout on the attention probabilities (attend.py:139-140); the mask element
    of (batch, head, query i, key j) is keep(seed, site, (batch*heads + head) * n_q_pad + i, j), n_q_pad = n_q
    rounded up to 128 (the same mask at every D).  The returned lse is that of the un-dropped probabilities.
    Accepted sizes: 1 <= n_q <= n_k and b * heads * n_q_pad < 2**32 (the 32-bit dropout counter), for any batch b:
    the local attention calls this with b = batch * heads * windows, which passes 65535 on long clips.
    scale defaults to D ** -0.5.  Returns o [b, n_q, heads*D] bf16 and lse [b, heads, n_q] fp32.
    """
    _check_cuda(q, k, v, bias)
    assert q.dtype == bf16 and k.dtype == bf16 and v.dtype == bf16
    b, n_q, hd = q.shape
    n_k = k.shape[1]
    D = _head_width(k)
    assert hd == heads * D and v.shape[-1] == D, "q must be [b, n_q, heads * dim_head] and v as wide as k"
    assert q.stride(-1) == 1 and k.stride(-1) == 1 and v.stride(-1) == 1
    assert q.stride(0) == n_q * q.stride(1)
    o = torch.empty(b, n_q, hd, device=q.device, dtype=bf16)
    n_q_pad = (n_q + 127) // 128 * 128  # the backward stages lse rows with 512-B bulk copies
    lse = torch.empty(b, heads, n_q_pad, device=q.device, dtype=f32) if return_lse else None
    key_mask = pack_key_mask(key_mask)
    if key_mask is not None:
        assert key_mask.n_k == n_k and key_mask.bits.shape[0] == b
        key_mask = key_mask.bits
    if scale is None:
        scale = D ** -0.5
    # algorithmic FLOPs: QK^T + PV over the visible (lower-triangle) part only
    vis = (n_q * n_k - n_q * (n_q - 1) / 2) if causal else n_q * n_k
    bhs, brs = _check_bias(bias, heads, n_q, n_k) if bias is not None else (0, 0)
    with _timed("mqa_attn_fwd_wgmma", 4.0 * b * heads * D * vis):
        _lib.call(
            "alm_mqa_attn_fwd_dh",
            q, q.stride(1), k, k.stride(1), k.stride(0), v, v.stride(1), v.stride(0), key_mask,
            o, o.stride(1), lse, n_q_pad, bias, bhs, brs, b, heads, n_q, n_k, int(causal), float(scale),
            *_drop_args(dropout), D,
        )
    return o, lse


def mqa_attn_bwd(q, k, v, o, d_o, lse, *, heads, key_mask=None, causal=True, scale=None, bias=None, dbias=None,
                 dropout=None):
    """Backward of mqa_attn_fwd: returns dq [b,n_q,h*D], dk [b,n_k,D], dv [b,n_k,D] (bf16), D = k.shape[-1].
    dropout: the (p, seed, site) of the forward call; its mask is regenerated.

    lse is the padded [b, heads, n_q_pad] tensor returned by the forward.  With a bias, d(bias) is ACCUMULATED
    into `dbias` (fp32, same shape/strides as `bias`; the caller zeroes it once per step).
    """
    _check_cuda(q, k, v, o, d_o, lse, bias, dbias)
    b, n_q, hd = q.shape
    n_k = k.shape[1]
    n_q_pad = lse.shape[-1]
    D = _head_width(k)
    assert hd == heads * D and v.shape[-1] == D
    assert d_o.dtype == bf16 and d_o.stride(-1) == 1 and o.stride(-1) == 1
    assert d_o.stride(0) == n_q * d_o.stride(1)
    key_mask = pack_key_mask(key_mask)
    if key_mask is not None:
        assert key_mask.n_k == n_k
        key_mask = key_mask.bits
    if scale is None:
        scale = D ** -0.5
    dq = torch.empty(b, n_q, hd, device=q.device, dtype=bf16)
    delta = torch.empty(b, heads, n_q_pad, device=q.device, dtype=f32)
    dq_acc = torch.empty(b, n_q, hd, device=q.device, dtype=f32)  # fp32 dQ workspace, zeroed by alm_attn_delta
    dk = torch.empty(b, n_k, D, device=q.device, dtype=bf16)
    dv = torch.empty(b, n_k, D, device=q.device, dtype=bf16)
    bhs, brs = _check_bias(bias, heads, n_q, n_k) if bias is not None else (0, 0)
    if dbias is not None:
        assert bias is not None and dbias.dtype == f32 and dbias.shape == bias.shape and dbias.stride() == bias.stride()
    vis = (n_q * n_k - n_q * (n_q - 1) / 2) if causal else n_q * n_k
    # 5 matmuls, each executed once; the timed region also covers delta + workspace zeroing and the dq conversion
    with _timed("mqa_attn_bwd_wgmma", 10.0 * b * heads * D * vis):
        _lib.call("alm_attn_delta_dh", o, o.stride(1), d_o, d_o.stride(1), delta, n_q_pad, dq_acc, b, heads, n_q, D)
        _lib.call(
            "alm_mqa_attn_bwd_dh",
            q, q.stride(1), k, k.stride(1), k.stride(0), v, v.stride(1), v.stride(0), d_o, d_o.stride(1), key_mask,
            lse, delta, n_q_pad, dq, dq.stride(1), dq_acc, dk, dk.stride(1), dv, dv.stride(1),
            bias, dbias, bhs, brs, b, heads, n_q, n_k, int(causal), float(scale), *_drop_args(dropout), D,
        )
    return dq, dk, dv


def gemv(x, w, *, out_dtype=bf16, bias=None):
    """x [rows <= 8, K] bf16, w [N, >=K (zero padded to a multiple of 8)] bf16 -> [rows, N] (decode-step Linear)."""
    _check_cuda(x, w, bias)
    rows, K = x.shape
    N = w.shape[0]
    assert x.dtype == bf16 and w.dtype == bf16 and x.stride(1) == 1 and w.stride(1) == 1 and rows <= 8
    assert w.shape[1] >= K and w.shape[1] % 8 == 0
    out = torch.empty(rows, N, device=x.device, dtype=out_dtype)
    _lib.call("alm_gemv_bf16", x, x.stride(0), w, w.stride(0), out, int(out_dtype == f32), out.stride(0),
              None if bias is None else bias.float().contiguous(), rows, N, K)
    return out


def kv_append(kv_new, k_cache, v_cache, cache_len):
    """k_cache[b, len] = kv_new[b, :D]; v_cache[b, len] = kv_new[b, D:]  (len: int32 device scalar; D = dim_head =
    k_cache.shape[-1])."""
    _check_cuda(kv_new, k_cache, v_cache, cache_len)
    b, max_len, _ = k_cache.shape
    D = _head_width(k_cache)
    assert v_cache.shape == k_cache.shape and kv_new.shape == (b, 2 * D) and kv_new.dtype == bf16
    assert k_cache.dtype == bf16 and v_cache.dtype == bf16 and cache_len.dtype == torch.int32
    assert k_cache.stride(1) == D and v_cache.stride() == k_cache.stride() and kv_new.stride(1) == 1
    _lib.call("alm_kv_append_dh", kv_new, kv_new.stride(0), k_cache, v_cache, k_cache.stride(0), cache_len, max_len, b,
              D)


def mqa_attn_decode(q, k_cache, v_cache, cache_len, *, heads, key_mask=None, scale=None, splits=None, bias=None):
    """one new query per sequence against the static cache [b, max_len, D]: q [b, heads*D] bf16 -> o [b, heads*D] bf16.
    Attends keys 0..cache_len (inclusive: the new token has just been appended at position cache_len).
    bias: fp32 [heads, >= max_len] added to the scores of every sequence (row j of head h: bias[h, j]) or None."""
    _check_cuda(q, k_cache, v_cache, cache_len, key_mask, bias)
    b, max_len, _ = k_cache.shape
    D = _head_width(k_cache)
    assert q.shape == (b, heads * D) and q.dtype == bf16 and q.stride(1) == 1
    assert v_cache.shape == k_cache.shape and k_cache.stride(1) == D and v_cache.stride() == k_cache.stride()
    o = torch.empty(b, heads * D, device=q.device, dtype=bf16)
    if key_mask is not None:
        assert key_mask.dtype == torch.uint8 and key_mask.shape[0] == b and key_mask.shape[1] >= max_len
    if bias is not None:
        assert bias.dtype == f32 and bias.shape[0] == heads and bias.shape[1] >= max_len and bias.stride(1) == 1
    if splits is None:  # enough CTAs to spread a long cache over the SMs, fixed per cache size (static launch)
        splits = max(1, min(32, max_len // 128, num_sms(q.device) // max(1, b)))
    ws = torch.empty(b, splits, heads, D + 2, device=q.device, dtype=f32) if splits > 1 else None
    _lib.call("alm_mqa_attn_decode_dh", q, q.stride(0), k_cache, v_cache, k_cache.stride(0), cache_len, max_len, key_mask,
              0 if key_mask is None else key_mask.stride(0), bias, 0 if bias is None else bias.stride(0), o, o.stride(0),
              ws, splits, b, heads, float(D ** -0.5 if scale is None else scale), D)
    return o


def decode_bias_row(table, override, u, cls, c, cache_len, out):
    """out[h, j] (j <= L = cache_len) = (cls[L] != cls[j] or cls[L] < 0) ? override[h] : table[u[L] - u[j] + c, h].
    table fp32 [rows, H], override fp32 [H] or None (= 0), u / cls int32 [max_len], out fp32 [H, >= max_len]."""
    _check_cuda(table, override, u, cls, cache_len, out)
    rows, H = table.shape
    max_len = u.shape[0]
    assert table.dtype == f32 and table.is_contiguous() and u.dtype == torch.int32 and cls.dtype == torch.int32
    assert u.is_contiguous() and cls.is_contiguous() and cls.shape == u.shape and cache_len.dtype == torch.int32
    assert out.dtype == f32 and out.shape[0] == H and out.shape[1] >= max_len and out.stride(1) == 1
    if override is not None:
        assert override.dtype == f32 and override.is_contiguous() and override.numel() == H
    _lib.call("alm_decode_bias_row", table, rows, override, u, cls, int(c), cache_len, max_len, out, out.stride(0), H)
    return out


def head_ce_fwd(x, w, bias, labels, ignore_index):
    """fused logit head + cross entropy, forward: x [M, K] bf16, w [V, >=K] bf16 (+ bias [V] fp32), labels [M] int64
    -> (lse [M] fp32, loss_rows [M] fp32 = lse - logit[label], 0 where label == ignore_index).  No logits in HBM."""
    _check_cuda(x, w, bias, labels)
    M, K = x.shape
    V = w.shape[0]
    assert x.dtype == bf16 and w.dtype == bf16 and x.stride(1) == 1 and w.stride(1) == 1 and w.shape[1] >= K
    assert labels.dtype == torch.int64 and labels.is_contiguous() and labels.numel() == M
    tiles = int(_lib.load().alm_gemm_head_ce_tiles(V))
    part = torch.empty(M, tiles, 2, device=x.device, dtype=f32)
    lab = torch.empty(M, device=x.device, dtype=f32)
    lse = torch.empty(M, device=x.device, dtype=f32)
    rows = torch.empty(M, device=x.device, dtype=f32)
    with _timed("gemm_head_ce_fused", 2.0 * M * V * K):
        _lib.call("alm_gemm_head_ce", x, x.stride(0), w, w.stride(0), bias, labels, int(ignore_index), 1, part, lab, None,
                  None, None, None, 0, M, V, K)
    _lib.call("alm_ce_finish", part, tiles, lab, labels, int(ignore_index), lse, rows, M)
    return lse, rows


def head_ce_bwd(x, w, bias, labels, ignore_index, lse, scale_num, scale_den, dlogits):
    """fused logit head + cross entropy, backward: recomputes the logits tile by tile and writes
    dlogits [M, >=V] bf16 = (softmax - onehot) * scale_num / scale_den (device scalars), zero rows where ignored."""
    _check_cuda(x, w, bias, labels, lse, scale_num, scale_den, dlogits)
    M, K = x.shape
    V = w.shape[0]
    assert dlogits.dtype == bf16 and dlogits.shape[0] == M and dlogits.shape[1] >= V and dlogits.stride(1) == 1
    assert scale_num.dtype == f32 and scale_den.dtype == f32 and lse.dtype == f32
    # the recomputation is executed work, not algorithmic work: timed in the fused-head class with 0 algorithmic FLOPs
    with _timed("gemm_head_ce_fused", 0.0):
        _lib.call("alm_gemm_head_ce", x, x.stride(0), w, w.stride(0), bias, labels, int(ignore_index), 2, None, None, lse,
                  scale_num, scale_den, dlogits, dlogits.stride(0), M, V, K)
    return dlogits


DECODE_STEP_MAX_ROWS = 4


def decode_stack_scratch(b, d, heads, inner, device):
    """workspace of alm_decode_stack_step (barrier counter + error flag + the vectors that cross its barriers)."""
    n = int(_lib.load().alm_decode_stack_scratch_bytes(b, d, heads, inner))
    if n <= 0:
        raise _lib.AlmError(f"alm_decode_stack_step does not take b={b}, d={d}, heads={heads}, inner={inner}")
    return torch.zeros(n, device=device, dtype=torch.uint8)


def decode_stack_grid():
    """CTAs of the one-kernel decode step (= SMs); the engine regroups its operands for this count."""
    return int(_lib.load().alm_decode_stack_grid())


@functools.lru_cache(maxsize=None)
def decode_stack_plan(b, d, heads, inner, n_layers, dim_head=64):
    """None if alm_decode_stack_step refuses this shape on the current device (it is built for dim_head 64 alone), else
    for phases A, C, D, E (q|kv, out, W1, W2 projections) whether the weight rows are staged in shared memory (True)
    or read from L2 (False)."""
    staged = (ctypes.c_int32 * 4)()
    if _lib.load().alm_decode_stack_plan_dh(b, d, heads, inner, n_layers, dim_head, staged) != 0:
        return None
    return tuple(bool(s) for s in staged)


def regroup_rows(w, grid):
    """[N, K] -> [grid * pc, K] with row (c * pc + l) = w[c + l * grid] (zeros past N): CTA c's rows become contiguous."""
    N, K = w.shape
    pc = -(-N // grid)
    wp = torch.zeros(pc * grid, K, device=w.device, dtype=w.dtype)
    wp[:N] = w
    return wp.view(pc, grid, K).transpose(0, 1).contiguous().view(grid * pc, K)


def decode_stack_step(table, x, out, final_gamma, cache_len, k_cache, key_mask, scratch, *, heads, inner, grid,
                      value_residual=True, scale=None):
    """the whole hyper-connection stack for ONE new token per sequence in one cooperative kernel.
    table: int64 [L, 24] device pointers (see include/alm_b200.h); x fp32 [b, d]; out bf16 [b, d];
    k_cache: [L, b, max_len, 64] (only its strides / max_len are read here; the table holds the per-layer bases).
    Increments cache_len on the device."""
    _check_cuda(table, x, out, final_gamma, cache_len, key_mask, scratch)
    L, b, max_len, dh = k_cache.shape
    d = x.shape[1]
    assert table.dtype == torch.int64 and table.shape == (L, 24) and table.is_contiguous()
    assert x.dtype == f32 and x.is_contiguous() and out.dtype == bf16 and out.is_contiguous() and x.shape == (b, d)
    assert dh == 64 and k_cache.stride(2) == 64 and cache_len.dtype == torch.int32 and final_gamma.dtype == f32
    if key_mask is not None:
        assert key_mask.dtype == torch.uint8 and key_mask.shape[0] == b and key_mask.shape[1] >= max_len
    _lib.call("alm_decode_stack_step", table, L, x, out, final_gamma, cache_len, max_len, k_cache.stride(1), key_mask,
              0 if key_mask is None else key_mask.stride(0), scratch, scratch.numel(), b, d, heads, inner,
              int(bool(value_residual)), float(64 ** -0.5 if scale is None else scale), grid)
    return out


def bias_gather_fwd(table, idx, override, *, ld=None):
    """table [P, H] fp32, idx [n_q, n_k] int32 (-1 = override), override [H] fp32 or None -> bias [H, n_q, ld] fp32."""
    _check_cuda(table, idx, override)
    assert table.dtype == f32 and table.is_contiguous() and idx.dtype == torch.int32 and idx.is_contiguous()
    H = table.shape[1]
    n_q, n_k = idx.shape
    ld = (n_k + 3) // 4 * 4 if ld is None else ld
    out = torch.empty(H, n_q, ld, device=table.device, dtype=f32)
    _lib.call("alm_bias_gather_fwd", table, idx, None if override is None else override.contiguous(), out, H, n_q,
              n_k, ld)
    return out


def bias_gather_bwd(dbias, idx, table_rows, *, want_override):
    """scatter-add of d(bias) [H, n_q, ld] back to the table rows / the per-head override scalar."""
    _check_cuda(dbias, idx)
    assert dbias.dtype == f32 and dbias.is_contiguous()
    H, n_q, ld = dbias.shape
    n_k = idx.shape[1]
    dtable = torch.zeros(table_rows, H, device=dbias.device, dtype=f32)
    dover = torch.zeros(H, device=dbias.device, dtype=f32) if want_override else None
    _lib.call("alm_bias_gather_bwd", dbias, idx, dtable, dover, H, n_q, n_k, ld)
    return dtable, dover


HC_MIN_STREAMS, HC_MAX_STREAMS = 2, 8  # stream counts the hyper-connection kernels are built for


def hc_aux_floats(streams):
    """floats of per-token state kept for the backward (csrc/hyper_conn_v2.cuh: aux_floats): ta[S(S+1)] tb[S] inv[S]
    z[S(S+1)+S] pad mean rstd, rounded up to a multiple of 4 so that one bulk copy stages a row"""
    return (2 * streams * (streams + 1) + 3 * streams + 4 + 3) // 4 * 4


HC_AUX = hc_aux_floats(4)


def _hc_param_ptrs(hc, ln_gamma):
    return (hc["gamma"], hc["dyn_alpha"], hc["dyn_beta"], hc["static_alpha"], hc["static_beta"],
            hc["alpha_scale"], hc["beta_scale"], ln_gamma)


def hc_pre_fwd(hc, ln_gamma, *, R_in=None, Y=None, beta_prev=None, x_expand=None, M, d, streams=4, want_bin=True):
    """depth(prev branch) + width(this branch) + pre-LayerNorm.  hc: dict of fp32 HC params.

    Returns R_out [M,S,d] bf16, bin [M,d] bf16 (None unless want_bin), xn [M,d] bf16, beta [M,S] f32,
    aux [M, hc_aux_floats(S)] f32.
    """
    dev = ln_gamma.device
    R_out = torch.empty(M, streams, d, device=dev, dtype=bf16)
    bin_ = torch.empty(M, d, device=dev, dtype=bf16) if want_bin else None
    xn = torch.empty(M, d, device=dev, dtype=bf16)
    beta = torch.empty(M, streams, device=dev, dtype=f32)
    aux = torch.empty(M, hc_aux_floats(streams), device=dev, dtype=f32)
    rs = 2 * streams  # bytes per channel of the bf16 [S, d] residual
    with _timed("hc_pre_fwd", M * d * ((4 if x_expand is not None else rs + 2) + rs + 2 + (2 if want_bin else 0)),
                "byte"):
        _lib.call("alm_hc_pre_fwd", R_in, Y, beta_prev, x_expand, *_hc_param_ptrs(hc, ln_gamma),
                  R_out, bin_, xn, beta, aux, M, d, streams)
    return R_out, bin_, xn, beta, aux


def hc_pre_bwd(hc, ln_gamma, grads, g_ln_gamma, aux, dR_out, dxn, dbeta, *, dbin_extra=None, R_in=None, Y=None,
               beta_prev=None, x_expand=None, dx_scale=1.0, M, d, streams=4):
    """Backward of hc_pre_fwd.  `grads`: dict of fp32 accumulators shaped like `hc` (atomically added to, as is
    g_ln_gamma).

    Returns (dR_in, dY, dbeta_prev) or dx_expand [M,d] f32 when the op expanded the streams.
    """
    dev = ln_gamma.device
    if x_expand is not None:
        dx = torch.empty(M, d, device=dev, dtype=f32)
        dR_in = dY = dbp = None
    else:
        dx = None
        dR_in = torch.empty(M, streams, d, device=dev, dtype=bf16)
        dY = torch.empty(M, d, device=dev, dtype=bf16)
        dbp = torch.empty(M, streams, device=dev, dtype=f32)
    rs = 2 * streams
    nbytes = M * d * ((4 + rs + 2 + 4 if x_expand is not None else rs + 2 + rs + 2 + rs + 2)
                      + (2 if dbin_extra is not None else 0))
    with _timed("hc_pre_bwd", nbytes, "byte"):
        _lib.call("alm_hc_pre_bwd", R_in, Y, beta_prev, x_expand, *_hc_param_ptrs(hc, ln_gamma), aux, dR_out, dxn,
                  dbin_extra, dbeta, dR_in, dY, dbp, dx, float(dx_scale),
                  grads["gamma"], grads["dyn_alpha"], grads["dyn_beta"], grads["static_alpha"], grads["static_beta"],
                  grads["alpha_scale"], grads["beta_scale"], g_ln_gamma, M, d, streams)
    return dx if x_expand is not None else (dR_in, dY, dbp)


def hc_post_fwd(R_in, Y, beta_prev, ln_gamma, *, M, d, streams=4):
    out = torch.empty(M, d, device=R_in.device, dtype=bf16)
    stats = torch.empty(M, 2, device=R_in.device, dtype=f32)
    _lib.call("alm_hc_post_fwd", R_in, Y, beta_prev, ln_gamma, out, stats, M, d, streams)
    return out, stats


def hc_post_bwd(R_in, Y, beta_prev, ln_gamma, stats, dout, g_ln_gamma, *, M, d, streams=4):
    dR_in = torch.empty(M, streams, d, device=R_in.device, dtype=bf16)
    dY = torch.empty(M, d, device=R_in.device, dtype=bf16)
    dbp = torch.empty(M, streams, device=R_in.device, dtype=f32)
    _lib.call("alm_hc_post_bwd", R_in, Y, beta_prev, ln_gamma, stats, dout, dR_in, dY, dbp, g_ln_gamma, M, d, streams)
    return dR_in, dY, dbp


def geglu_ln_fwd(h, gamma, *, inner, inner_pad, dropout=None):
    """h [M, 2*inner_pad] bf16 (a | gate) -> gn [M, inner_pad] bf16 = LN(gelu(gate)*a)*gamma, stats [M,2].
    dropout: optional (p, seed, site): gn is returned dropped, mask keep(seed, site, row, channel)."""
    M = h.shape[0]
    gn = torch.empty(M, inner_pad, device=h.device, dtype=bf16)
    stats = torch.empty(M, 2, device=h.device, dtype=f32)
    with _timed("geglu_ln_fwd", M * inner_pad * 6, "byte"):
        _lib.call("alm_geglu_ln_fwd", h, h.stride(0), inner_pad, gamma, gn, gn.stride(0), stats, M, inner, inner_pad,
                  *_drop_args(dropout))
    return gn, stats


def geglu_ln_bwd(h, gamma, stats, dgn, g_gamma, *, inner, inner_pad, dropout=None):
    """dropout: the (p, seed, site) of the forward; the mask is applied to dgn first."""
    M = h.shape[0]
    dh = torch.empty_like(h)
    assert dh.stride(0) == h.stride(0)
    with _timed("geglu_ln_bwd", M * inner_pad * 10, "byte"):
        _lib.call("alm_geglu_ln_bwd", h, h.stride(0), inner_pad, gamma, stats, dgn, dgn.stride(0), dh, g_gamma, M,
                  inner, inner_pad, *_drop_args(dropout))
    return dh


def ce_fwd_bwd(logits, labels, *, ignore_index=-1, scale_num=None, scale_den=None, want_grad=True):
    """logits [R, V] f32 (row stride free), labels [R] int64 -> loss_rows [R] f32, dlogits [R, Vpad] bf16."""
    R, V = logits.shape
    Vpad = (V + 7) // 8 * 8
    loss_rows = torch.empty(R, device=logits.device, dtype=f32)
    dlogits = torch.empty(R, Vpad, device=logits.device, dtype=bf16) if want_grad else None
    _lib.call("alm_ce_fwd_bwd", logits, logits.stride(0), labels, int(ignore_index), loss_rows, dlogits,
              Vpad, scale_num, scale_den, R, V, Vpad)
    return loss_rows, dlogits


def axpby(x, alpha, y, beta, out=None):
    """out = alpha*x + beta*y on 2-D bf16 views (last dim contiguous)."""
    rows, cols = x.shape
    if out is None:
        out = torch.empty(rows, cols, device=x.device, dtype=bf16)
    _lib.call("alm_axpby_bf16", x, x.stride(0), float(alpha), y, y.stride(0) if y is not None else 0, float(beta),
              out, out.stride(0), rows, cols)
    return out


def cast_pad(src, cols_pad=None, out=None):
    """fp32 [R, C] (last dim contiguous) -> bf16 [R, cols_pad] zero padded."""
    rows, cols = src.shape
    cols_pad = cols if cols_pad is None else cols_pad
    if out is None:
        out = torch.empty(rows, cols_pad, device=src.device, dtype=bf16)
    _lib.call("alm_cast_pad_bf16", src, src.stride(0), out, out.stride(0), rows, cols, cols_pad)
    return out


def cast_pad_multi(desc):
    """desc: device int64 [n, 7] rows {src ptr, dst ptr, rows, cols, cols_pad, lds, ldd}: all casts in one launch"""
    _check_cuda(desc)
    assert desc.dtype == torch.int64 and desc.is_contiguous() and desc.shape[1] == 7
    _lib.call("alm_cast_pad_multi", desc, desc.shape[0])


def scale_by_scalar(x, s):
    _lib.call("alm_scale_by_scalar_bf16", x, s, x.numel())
    return x


# ---- SoundStream codec -------------------------------------------------------------------------------
PAD_MODES = {"reflect": 0, "constant": 1, "zeros": 1, "replicate": 2}


# (K, stride, dilation) shapes with a register-tiled specialisation (csrc/conv_tiled.cuh)
CONV_TILED_SHAPES = {(7, 1, 1), (7, 1, 3), (7, 1, 9), (1, 1, 1), (3, 1, 1), (4, 2, 1), (6, 3, 1), (8, 4, 1), (10, 5, 1),
                     (16, 8, 1)}


def causal_conv1d(x, weight, bias=None, *, stride=1, dilation=1, pad_mode="reflect", elu=False, residual=None,
                  weight_packed=None):
    """CausalConv1d forward (soundstream.py:332-345) with optional fused ELU and skip add. fp32 [B,C,T].

    weight [Cout, Cin, K] (torch layout); weight_packed: optional cached copy [Cin, K, Cout] (weight.permute(1, 2, 0))
    that lets the register-tiled kernel stage weights with coalesced loads."""
    _check_cuda(x, weight, bias, residual, weight_packed)
    assert x.dtype == f32 and weight.dtype == f32
    x = x.contiguous()
    B, Cin, T = x.shape
    Cout, Cin_w, K = weight.shape
    assert Cin_w == Cin, "groups != 1 is not supported"
    pad = dilation * (K - 1) + 1 - stride
    Tout = (T + pad - dilation * (K - 1) - 1) // stride + 1
    y = torch.empty(B, Cout, Tout, device=x.device, dtype=f32)
    if residual is not None:
        residual = residual.contiguous()
        assert residual.shape == y.shape
    packed = weight_packed is not None and (K, stride, dilation) in CONV_TILED_SHAPES
    if packed:
        assert weight_packed.shape == (Cin, K, Cout) and weight_packed.is_contiguous() and weight_packed.dtype == f32
    cls = "causal_conv1d"
    if _PROFILE is not None and PROFILE_SHAPES:
        cls += f" Cin{Cin} Cout{Cout} K{K} s{stride} d{dilation} T{T}"
    with _timed(cls, 2.0 * B * Cout * Tout * Cin * K):
        _lib.call("alm_causal_conv1d_fwd", x, weight_packed if packed else weight.contiguous(),
                  None if bias is None else bias.contiguous(), residual, y, B, Cin, Cout, T, K, stride, dilation,
                  PAD_MODES[pad_mode], int(elu), int(packed))
    return y


RU_FUSED_CHANNELS = {32, 64, 128, 256}
RU_FUSED_DILATIONS = {1, 3, 9}


def residual_unit(x, w7_packed, b7, w1_packed, b1, *, dilation, pad_mode="reflect"):
    """fused ResidualUnit forward (soundstream.py:362-369); packed weights [C,7,C] / [C,1,C], fp32 [B,C,T]."""
    _check_cuda(x, w7_packed, b7, w1_packed, b1)
    x = x.contiguous()
    B, C, T = x.shape
    assert w7_packed.shape == (C, 7, C) and w1_packed.shape == (C, 1, C) and x.dtype == f32
    y = torch.empty_like(x)
    with _timed("residual_unit_fused", 2.0 * B * C * T * C * 8):
        _lib.call("alm_residual_unit_fwd", x, w7_packed, b7.contiguous(), w1_packed, b1.contiguous(), y, B, C, T,
                  dilation, PAD_MODES[pad_mode])
    return y


def se_fold_weight(w1):
    """SqueezeExcite's first 1x1 conv [Ci, C, 1] with the reference's cumulative mean folded in -> fp32 [Ci, C].

    SqueezeExcite.forward (soundstream.py:156-169) receives [B, C, T] but cumsums dim -2, so its "cumulative mean" runs
    over channels: m[c] = mean_{c' <= c} y[c'].  That is linear, so W1 m = W1' y with
    W1'[i, c'] = sum_{c >= c'} W1[i, c] / (c + 1), computed here in fp64."""
    w = w1.detach()[..., 0].double()
    C = w.shape[1]
    scaled = w / torch.arange(1, C + 1, device=w.device, dtype=torch.float64)
    return scaled.flip(-1).cumsum(-1).flip(-1).float().contiguous()


def codec_se_fp32(y, x, w1_folded, b1, w2, b2):
    """SqueezeExcite residual tail out = x + y * gate(y) on fp32 [B, C, T] (csrc/codec.cu); w1_folded from
    se_fold_weight, w2 [C, Ci(, 1)]."""
    _check_cuda(y, x, w1_folded, b1, w2, b2)
    y, x = y.contiguous(), x.contiguous()
    B, C, T = y.shape
    Ci = w1_folded.shape[0]
    assert x.shape == y.shape and y.dtype == f32 and x.dtype == f32 and w1_folded.shape == (Ci, C)
    w2 = w2.detach().reshape(C, Ci).float().contiguous()
    out = torch.empty_like(y)
    with _timed("codec_se_fp32", 2.0 * B * T * 2 * C * Ci):
        _lib.call("alm_codec_se_fp32", y, x, w1_folded, b1.detach().float().contiguous(), w2,
                  b2.detach().float().contiguous(), out, B, C, Ci, T)
    return out


def causal_conv_transpose1d(x, weight, bias=None, *, stride):
    """CausalConvTranspose1d forward (soundstream.py:347-360): weight [Cin, Cout, 2*stride]."""
    _check_cuda(x, weight, bias)
    x = x.contiguous()
    B, Cin, n = x.shape
    Cin_w, Cout, K = weight.shape
    assert Cin_w == Cin and K == 2 * stride
    y = torch.empty(B, Cout, n * stride, device=x.device, dtype=f32)
    _lib.call("alm_causal_convT1d_fwd", x, weight.contiguous(), None if bias is None else bias.contiguous(), y, B,
              Cin, Cout, n, stride)
    return y


# ---- SoundStream encoder on the tensor cores (csrc/codec_tc.cu) ---------------------------------------
def c8s_pack(x, phases=1):
    """fp32 [B, C, T] -> C8S bf16 [B, 2C/8, P, T/P, 8] (torch ops; boundaries and tests only)."""
    B, C, T = x.shape
    assert C % 8 == 0 and T % phases == 0
    hi = x.to(bf16)
    lo = (x - hi.float()).to(bf16)

    def arr(t):
        return t.reshape(B, C // 8, 8, T // phases, phases).permute(0, 1, 4, 3, 2)

    return torch.cat((arr(hi), arr(lo)), dim=1).contiguous()


def c8s_unpack(a):
    """C8S bf16 [B, 2C/8, P, T/P, 8] -> fp32 [B, C, T]."""
    B, nch2, P, Tp, _ = a.shape
    nch = nch2 // 2
    v = a[:, :nch].float() + a[:, nch:].float()
    return v.permute(0, 1, 4, 3, 2).reshape(B, nch * 8, Tp * P)


def _split_units(w, bn=None):
    """w fp32 [Cout, Cin, K] -> bf16 [K, Cin/16, 2 (hi, lo), 2, Cout, 8] (optionally tiled over Cout by bn)."""
    Cout, Cin, K = w.shape
    assert Cin % 16 == 0
    hi = w.to(bf16)
    lo = (w - hi.float()).to(bf16)

    def arr(t):
        return t.permute(2, 1, 0).reshape(K, Cin // 16, 2, 8, Cout).permute(0, 1, 2, 4, 3)

    st = torch.stack((arr(hi), arr(lo)), dim=2)                      # [K, kk, part, cc, Cout, 8]
    if bn is not None:
        st = st.reshape(K, Cin // 16, 2, 2, Cout // bn, bn, 8).permute(4, 0, 1, 2, 3, 5, 6)
    return st.contiguous()


def pack_ru_weights(w7, w1):
    """ResidualUnit weights [C, C, 7], [C, C, 1] -> the unit layout alm_codec_ru_tc streams (tap 7 = the 1x1 conv)."""
    return _split_units(torch.cat((w7.detach().float(), w1.detach().float()), dim=2))


def se_inner_pad(C):
    """inner width of the tensor-core SqueezeExcite GEMMs: the reference's max(8, C // 4), zero-padded to >= 32"""
    return max(32, C // 4)


def pack_ru_se_weights(w7, w1, se_w1, se_w2):
    """ResidualUnit(squeeze_excite=True) weights -> the unit layout alm_codec_ru_se_tc streams: pack_ru_weights, then the
    folded first SE conv (se_fold_weight) as [C/16] k-steps with NS rows and the second SE conv as [NS/16] k-steps with C
    rows, NS = se_inner_pad(C), zero-padded."""
    C = w7.shape[0]
    Ci = se_w1.shape[0]
    ns = se_inner_pad(C)
    assert se_w1.shape[:2] == (Ci, C) and se_w2.shape[:2] == (C, Ci) and Ci <= ns
    w1f = torch.zeros(ns, C, 1, device=w7.device, dtype=f32)
    w1f[:Ci, :, 0] = se_fold_weight(se_w1)
    w2p = torch.zeros(C, ns, 1, device=w7.device, dtype=f32)
    w2p[:, :Ci, 0] = se_w2.detach().reshape(C, Ci).float()
    return torch.cat((pack_ru_weights(w7, w1).flatten(), _split_units(w1f).flatten(), _split_units(w2p).flatten()))


def conv_tc_bn(cout):
    return 256 if cout % 256 == 0 else (128 if cout % 128 == 0 else 64)


def pack_conv_weights(w):
    return _split_units(w.detach().float(), bn=conv_tc_bn(w.shape[0]))


def pack_convT_weights(w, stride):
    """CausalConvTranspose1d weight [Cin, Cout, 2s] -> (units for alm_codec_conv_tc, Cout' = s * Cout): the transposed conv
    is the 2-tap causal conv  out[i, (r, o)] = W[c, o, r + s] x[i - 1, c] + W[c, o, r] x[i, c]  (soundstream.py:347-360)."""
    cin, cout, k = w.shape
    assert k == 2 * stride
    wf = w.detach().float()
    taps = torch.stack((wf[..., stride:], wf[..., :stride]), dim=-1)          # [c, o, r, j]: j = 0 -> x[i-1], 1 -> x[i]
    wp = taps.permute(2, 1, 0, 3).reshape(stride * cout, cin, 2)               # [(r, o), c, j]
    return pack_conv_weights(wp)


def codec_pack_c8s(x):
    """fp32 channels-last [B, n, C] -> C8S [B, 2C/8, 1, n, 8] (entry of the tensor-core decoder)."""
    _check_cuda(x)
    B, n, C = x.shape
    x = x.to(f32).contiguous()
    y = torch.empty(B, 2 * C // 8, 1, n, 8, device=x.device, dtype=bf16)
    _lib.call("alm_codec_pack_c8s", x, y, B, n, C)
    return y


def codec_last_conv(x, weight, bias, *, pad_mode="reflect"):
    """CausalConv1d(Cin, 1, K) on C8S (P = 1) -> fp32 [B, 1, T] (soundstream.py:626)."""
    _check_cuda(x, weight, bias)
    B, nch2, P, T, _ = x.shape
    assert P == 1 and weight.shape[0] == 1 and weight.shape[1] == nch2 * 4
    y = torch.empty(B, 1, T, device=x.device, dtype=f32)
    with _timed("codec_last_conv", 4.0 * B * T * (nch2 * 4 + 1), "byte"):
        _lib.call("alm_codec_last_conv", x, weight.detach().contiguous(),
                  None if bias is None else bias.detach().contiguous(), y, B, T, nch2 * 4, weight.shape[2],
                  PAD_MODES[pad_mode])
    return y


def codec_first_conv(wave, weight, bias, *, pad_mode="reflect"):
    """CausalConv1d(1, Cout, K) on fp32 [B, T] -> C8S [B, 2Cout/8, 1, T, 8] (soundstream.py:520)."""
    _check_cuda(wave, weight, bias)
    B, T = wave.shape
    Cout, cin, K = weight.shape
    assert cin == 1 and wave.dtype == f32
    y = torch.empty(B, 2 * Cout // 8, 1, T, 8, device=wave.device, dtype=bf16)
    with _timed("codec_first_conv", (B * T * 4 + B * Cout * T * 4), "byte"):
        _lib.call("alm_codec_first_conv", wave.contiguous(), weight.detach().contiguous(),
                  None if bias is None else bias.detach().contiguous(), y, B, T, Cout, K, PAD_MODES[pad_mode])
    return y


def codec_ru_tc(x, w_units, b7, b1, *, dilation, pad_mode="reflect", out_phases=1):
    """fused ResidualUnit on C8S activations (P = 1 in, `out_phases` planes out)."""
    _check_cuda(x, w_units, b7, b1)
    B, nch2, P, T, _ = x.shape
    C = nch2 * 4
    assert P == 1 and x.dtype == bf16 and x.is_contiguous() and w_units.dtype == bf16 and w_units.is_contiguous()
    assert w_units.numel() == 8 * (C // 16) * 2 * 2 * C * 8
    y = torch.empty(B, nch2, out_phases, T // out_phases, 8, device=x.device, dtype=bf16)
    cls = "codec_ru_tc"
    if _PROFILE is not None and PROFILE_SHAPES:
        cls += f" C{C} T{T} d{dilation} P{out_phases}"
    with _timed(cls, 2.0 * B * C * T * 4, "byte"):
        _lib.call("alm_codec_ru_tc", x, y, w_units, b7, b1, B, C, T, int(dilation), PAD_MODES[pad_mode],
                  int(out_phases))
    return y


def codec_ru_se_tc(x, w_units, b7, b1, se_b1, se_b2, *, dilation, pad_mode="reflect", out_phases=1):
    """fused ResidualUnit with SqueezeExcite on C8S activations; w_units from pack_ru_se_weights."""
    _check_cuda(x, w_units, b7, b1, se_b1, se_b2)
    B, nch2, P, T, _ = x.shape
    C = nch2 * 4
    ns = se_inner_pad(C)
    assert P == 1 and x.dtype == bf16 and x.is_contiguous() and w_units.dtype == bf16 and w_units.is_contiguous()
    assert w_units.numel() == (8 * (C // 16) * C + (C // 16) * ns + (ns // 16) * C) * 2 * 2 * 8
    se_b1, se_b2 = se_b1.detach().float().contiguous(), se_b2.detach().float().contiguous()
    assert se_b2.numel() == C and 1 <= se_b1.numel() <= ns
    y = torch.empty(B, nch2, out_phases, T // out_phases, 8, device=x.device, dtype=bf16)
    cls = "codec_ru_se_tc"
    if _PROFILE is not None and PROFILE_SHAPES:
        cls += f" C{C} T{T} d{dilation} P{out_phases}"
    with _timed(cls, 2.0 * B * C * T * 4, "byte"):
        _lib.call("alm_codec_ru_se_tc", x, y, w_units, b7, b1, se_b1, se_b2, B, C, se_b1.numel(), T, int(dilation),
                  PAD_MODES[pad_mode], int(out_phases))
    return y


def codec_conv_tc(x, w_units, bias, *, cout, kernel_size, stride, pad_mode="reflect", out_phases=1, out_fp32=False,
                  upsample=1):
    """CausalConv1d(Cin, cout, kernel_size, stride) on C8S activations with P = stride planes.  upsample = s > 1: the
    transposed-conv form (see pack_convT_weights): cout = s * C' columns become s time steps of C' channels."""
    _check_cuda(x, w_units, bias)
    B, nch2, P, Tp, _ = x.shape
    Cin, Tin = nch2 * 4, P * Tp
    assert P == stride and x.is_contiguous() and w_units.is_contiguous()
    n_out = Tin // stride
    if out_fp32:
        y = torch.empty(B, n_out, cout, device=x.device, dtype=f32)
    elif upsample > 1:
        y = torch.empty(B, 2 * (cout // upsample) // 8, 1, n_out * upsample, 8, device=x.device, dtype=bf16)
    else:
        y = torch.empty(B, 2 * cout // 8, out_phases, n_out // out_phases, 8, device=x.device, dtype=bf16)
    cls = "codec_conv_tc"
    if _PROFILE is not None and PROFILE_SHAPES:
        cls += f" Cin{Cin} Cout{cout} K{kernel_size} s{stride} T{Tin}"
    with _timed(cls, 4.0 * B * (Cin * Tin + cout * n_out), "byte"):
        _lib.call("alm_codec_conv_tc", x, y, w_units, bias, B, Cin, cout, Tin, int(kernel_size), int(stride),
                  PAD_MODES[pad_mode], int(out_phases), int(out_fp32), int(upsample))
    return y



# ---- gate-loop layer (csrc/codec_gate_loop.cu) --------------------------------------------------------
def gate_loop_fold_weight(w, gamma):
    """SimpleGateLoopLayer's to_qkva weight [3C, C] with its RMSNorm scale sqrt(C) * gamma folded into the columns ->
    fp32 [3C, C], computed in fp64.  The norm's 1 / max(||u||, 1e-12) is per time step and stays in the kernel."""
    w = w.detach().double()
    C = w.shape[1]
    return (w * (gamma.detach().double() * math.sqrt(C))[None, :]).float().contiguous()


def gate_loop_slice(C):
    """channels per CTA of alm_codec_gate_loop_tc (its q, kv and a are three m64nNSk16 accumulators)"""
    return min(C, 64)


def pack_gate_loop_weights(w_folded):
    """folded [3C, C] -> the units alm_codec_gate_loop_tc streams: per channel slice of NS = gate_loop_slice(C), its q, kv
    and a rows (3 NS) in the split-bf16 conv layout, bf16 [C/NS][C/16][hi, lo][2][3 NS][8]"""
    C = w_folded.shape[1]
    ns = gate_loop_slice(C)
    rows = w_folded.detach().float().reshape(3, C // ns, ns, C).permute(1, 0, 2, 3).reshape(3 * C, C, 1)
    return _split_units(rows, bn=3 * ns).reshape(C // ns, C // 16, 2, 2, 3 * ns, 8).contiguous()


def _gate_loop_workspace(B, C, T, device, tc):
    n = int(_lib.load().alm_codec_gate_loop_workspace(B, C, T, int(tc)))
    return torch.empty(n, device=device, dtype=f32) if n else None


def codec_gate_loop_fp32(x, w_folded):
    """Residual(ChannelTranspose(SimpleGateLoopLayer)) on fp32 [B, C, T]: y = 2x + q * h.  The projection is
    causal_conv1d with K = 1 on the folded weight; the norm, the gates and the scan are alm_codec_gate_loop_fp32."""
    _check_cuda(x, w_folded)
    x = x.contiguous()
    B, C, T = x.shape
    assert x.dtype == f32 and w_folded.shape == (3 * C, C)
    proj = causal_conv1d(x, w_folded[:, :, None])
    y = torch.empty_like(x)
    with _timed("codec_gate_loop_fp32", 4.0 * B * T * 5 * C, "byte"):
        _lib.call("alm_codec_gate_loop_fp32", x, proj, y, _gate_loop_workspace(B, C, T, x.device, False), B, C, T)
    return y


def codec_gate_loop_tc(x, w_units):
    """Residual(ChannelTranspose(SimpleGateLoopLayer)) on C8S activations (P = 1 in and out), one fused kernel pair:
    the split-bf16 projection on the tensor cores, the norm, the gates and the scan (alm_codec_gate_loop_tc);
    w_units from pack_gate_loop_weights."""
    _check_cuda(x, w_units)
    B, nch2, P, T, _ = x.shape
    C = nch2 * 4
    ns = gate_loop_slice(C)
    assert P == 1 and x.dtype == bf16 and x.is_contiguous()
    assert w_units.dtype == bf16 and w_units.is_contiguous() and w_units.shape == (C // ns, C // 16, 2, 2, 3 * ns, 8)
    y = torch.empty_like(x)
    cls = "codec_gate_loop_tc"
    if _PROFILE is not None and PROFILE_SHAPES:
        cls += f" C{C} T{T}"
    with _timed(cls, 8.0 * B * T * C, "byte"):
        _lib.call("alm_codec_gate_loop_tc", x, w_units, y, _gate_loop_workspace(B, C, T, x.device, True), B, C, T)
    return y

def rvq_encode(x, codebooks):
    """x [N, D] fp32, codebooks [Q, C, D] fp32 -> (quantized [N, D] fp32, indices [N, Q] int64)."""
    _check_cuda(x, codebooks)
    assert x.dtype == f32 and codebooks.dtype == f32 and x.stride(-1) == 1
    N, D = x.shape
    Q, C, D2 = codebooks.shape
    assert D == D2
    codebooks = codebooks.contiguous()
    quant = torch.empty(N, D, device=x.device, dtype=f32)
    idx = torch.empty(N, Q, device=x.device, dtype=torch.int64)
    ws = torch.empty(Q * C, device=x.device, dtype=f32)
    with _timed("rvq_encode", 2.0 * N * Q * C * D):
        _lib.call("alm_rvq_encode", x, x.stride(0), codebooks, ws, quant, D, idx, Q, N, D, C, Q)
    return quant, idx


def rvq_search_width(D):
    """width the tensor-core search runs at: D rounded up to a multiple of 8 (the score GEMM's row pitch 3D must be
    one).  The extra columns are zero in the codebooks and in the residual, so they add exact zeros to every norm and
    dot product and the fp32 argmin is that of width D."""
    return -(-D // 8) * 8


def rvq_pack_codebooks(codebooks):
    """codebooks fp32 [Q, C, D] -> (codebooks fp32 [Q, C, Dp], packed bf16 [Q, C, 3Dp] = [hi | hi | lo], e2 fp32 [Q, C])
    for rvq_encode_tc, zero-padded to Dp = rvq_search_width(D)."""
    _check_cuda(codebooks)
    Q, C, D = codebooks.shape
    Dp = rvq_search_width(D)
    cb = codebooks.to(f32).contiguous()
    if Dp != D:
        cb = torch.nn.functional.pad(cb, (0, Dp - D))
    packed, e2 = _split_pack(cb.view(Q * C, Dp))
    return cb, packed.view(Q, C, 3 * Dp), e2.view(Q, C)


def _split_pack(rows):
    """fp32 [R, K] contiguous -> (bf16 [R, 3K] = [hi | hi | lo], fp32 |row|^2 [R])"""
    R, K = rows.shape
    packed = torch.empty(R, 3 * K, device=rows.device, dtype=bf16)
    e2 = torch.empty(R, device=rows.device, dtype=f32)
    _lib.call("alm_rvq_pack_codebooks", rows, packed, e2, R, K)
    return packed, e2


RVQ_METRICS = {"euclid": ("alm_rvq_prepare", "alm_rvq_select"), "cosine": ("alm_rvq_prepare_cos", "alm_rvq_select_cos")}


def rvq_encode_tc(x, packed_codebooks, *, metric="euclid"):
    """x [N, D] fp32 -> (quantized [N, D] fp32, indices [N, Q] int64); distance GEMMs on the tensor cores, the
    winner of every stage chosen by exact fp32 re-evaluation of the candidates (csrc/rvq_tc.cu).  Any D: the search
    runs at the padded width of rvq_pack_codebooks.  metric "euclid": argmin of the Euclidean distance; "cosine":
    argmax of F.normalize(r) . e_c (VectorQuantize(use_cosine_sim=True)); both lowest index on ties."""
    prepare, select = RVQ_METRICS[metric]
    cb, packed, e2 = packed_codebooks
    _check_cuda(x, cb)
    assert x.dtype == f32 and x.stride(-1) == 1
    N, D = x.shape
    Q, C, Dp = cb.shape
    assert Dp == rvq_search_width(D), f"codebooks packed for width {Dp}, x has {D}"
    dev = x.device
    r = torch.empty(N, Dp, device=dev, dtype=f32)
    quant = torch.empty(N, Dp, device=dev, dtype=f32)
    rp = torch.empty(N, 3 * Dp, device=dev, dtype=bf16)
    scores = torch.empty(N, C, device=dev, dtype=f32)
    idx = torch.empty(N, Q, device=dev, dtype=torch.int64)
    with _timed("rvq_encode_tc" if metric == "euclid" else f"rvq_encode_tc_{metric}", 2.0 * N * Q * C * D):
        _lib.call(prepare, x, x.stride(0), r, quant, Dp, rp, N, D, Dp)
        for q in range(Q):
            gemm(rp, packed[q], out=scores, cls="rvq_score_gemm")
            _lib.call(select, scores, C, e2[q], cb[q], r, quant, Dp, rp, idx[:, q:], Q, N, Dp, C,
                      int(q + 1 < Q))
    return (quant if Dp == D else quant[:, :D].contiguous()), idx


def split_rows(x):
    """fp32 [N, D] (unit column stride) -> bf16 [N, 3D] = [x_hi | x_lo | x_hi], the activation operand of split_gemm"""
    _check_cuda(x)
    assert x.dtype == f32 and x.stride(-1) == 1
    N, D = x.shape
    out = torch.empty(N, 3 * D, device=x.device, dtype=bf16)
    _lib.call("alm_split_rows", x, x.stride(0), out, N, D)
    return out


def split_linear(x, w_packed, bias):
    """nn.Linear on fp32 rows x [N, K] in split bf16: x @ w^T + bias -> fp32 [N, Nout], w_packed = pack_split_weight(w),
    the bias added in the GEMM's epilogue"""
    return split_gemm(split_rows(x), w_packed, bias, cls="split_linear")


def nearest_centroid(x, packed_centroids):
    """cluster assignment of HubertWithKmeans.forward (hubert_kmeans.py:114-116: `(-torch.cdist(embed, centers)).argmax(-1)`):
    x [N, D] fp32, packed_centroids = rvq_pack_codebooks(centers[None]) -> ids [N] int64.  Same kernels as one RVQ stage:
    the distance GEMM on the tensor cores, then the exact fp32 re-rank (lowest index on ties, as argmax does)."""
    _, idx = rvq_encode_tc(x, packed_centroids)
    return idx[:, 0]


def rvq_decode(indices, codebooks):
    """indices [N, Q] int64 (-1 = dropped) -> sum of selected codes [N, D] fp32."""
    _check_cuda(indices, codebooks)
    indices = indices.to(torch.int64).contiguous()
    N, Q = indices.shape
    Qc, C, D = codebooks.shape
    assert Q <= Qc
    out = torch.empty(N, D, device=indices.device, dtype=f32)
    _lib.call("alm_rvq_decode", indices, Q, codebooks.contiguous(), out, D, N, D, C, Q)
    return out


# ---- EnCodec 24 kHz (csrc/encodec.cu) -----------------------------------------------------------------
def encodec_conv(x, weight, bias, *, stride=1, weight_packed=None):
    """EnCodec's causal Conv1d (kernel K, stride s, dilation 1) on fp32 [B, Cin, L] -> [B, Cout, ceil(L / s)]:
    reflect padding of K - s on the left and ceil(L / s) * s - L on the right.  The common case (no right padding,
    L > K - s) is the SoundStream conv's own reflect halo; otherwise the row is padded first (alm_encodec_pad1d)
    and the conv runs on it unpadded, dropping the outputs of its own (zero) halo."""
    _check_cuda(x, weight, bias)
    B, Cin, L = x.shape
    K = weight.shape[-1]
    pl, pr = K - stride, -L % stride
    if pr == 0 and L > pl:
        return causal_conv1d(x, weight, bias, stride=stride, pad_mode="reflect", weight_packed=weight_packed)
    x = x.contiguous()
    xp = torch.empty(B, Cin, pl + L + pr, device=x.device, dtype=f32)
    _lib.call("alm_encodec_pad1d", x, xp, B * Cin, L, pl, pr)
    y = causal_conv1d(xp, weight, bias, stride=stride, pad_mode="constant", weight_packed=weight_packed)
    return y[..., pl // stride:].contiguous()


def encodec_resblock(x, w3, b3, w1, ws, b_out, *, elu_out):
    """SEANet resnet block on fp32 [B, C, T]: Ws x + W1 ELU(W3 * ELU(x) + b3) + b_out, ELU'd when elu_out.
    w3 [C/2, C, 3], w1 [C, C/2], ws [C, C] and b_out = b1 + bs, all fp32 contiguous."""
    _check_cuda(x, w3, b3, w1, ws, b_out)
    x = x.contiguous()
    B, C, T = x.shape
    assert x.dtype == f32 and w3.shape == (C // 2, C, 3) and w1.shape == (C, C // 2) and ws.shape == (C, C)
    y = torch.empty_like(x)
    with _timed("encodec_resblock", 2.0 * B * T * (3 * C * C // 2 + C * C // 2 + C * C)):
        _lib.call("alm_encodec_resblock_fp32", x, w3, b3, w1, ws, b_out, y, B, C, T, int(elu_out))
    return y


ENCODEC_LSTM_H = 512
ENCODEC_LSTM_UNITS = 4  # hidden units per CTA (csrc/encodec.cu)


def encodec_lstm_pack(w_ih, w_hh, b_ih, b_hh):
    """two layers' torch.nn.LSTM parameters (lists of [4H, H] / [4H]) -> (w [H/4, 32, 2H], bias [H/4, 32]) fp32:
    CTA k's row (layer l, gate g, unit u) at (l * 4 + g) * 4 + u is [W_ih_l | W_hh_l] of hidden unit 4k + u; the two
    biases are added in fp64."""
    H, U = ENCODEC_LSTM_H, ENCODEC_LSTM_UNITS
    w = torch.stack([torch.cat((wi, wh), dim=1).reshape(4, H // U, U, 2 * H) for wi, wh in zip(w_ih, w_hh)])
    b = torch.stack([(bi.double() + bh.double()).reshape(4, H // U, U) for bi, bh in zip(b_ih, b_hh)])
    w = w.permute(2, 0, 1, 3, 4).reshape(H // U, 32, 2 * H)  # [cta][layer][gate][unit][K]
    b = b.permute(2, 0, 1, 3).reshape(H // U, 32)
    return w.float().contiguous(), b.float().contiguous()


def encodec_lstm(x, packed, *, elu_out, check=False):
    """EnCodec's LSTM block y = LSTM2(LSTM1(x)) + x (ELU'd when elu_out) on fp32 [B, 512, T] or on C8S
    [B, 128, 1, T, 8] (bf16, the tensor-core codec layout); packed from encodec_lstm_pack.  One persistent cooperative
    kernel (csrc/encodec.cu).  check=True synchronises and raises if a device-wide barrier of the kernel timed out."""
    w, b = packed
    _check_cuda(x, w, b)
    x = x.contiguous()
    c8s = x.dtype == bf16
    if c8s:
        B, nch2, P, T, _ = x.shape
        assert nch2 * 4 == ENCODEC_LSTM_H and P == 1
    else:
        B, H, T = x.shape
        assert H == ENCODEC_LSTM_H and x.dtype == f32
    y = torch.empty_like(x)
    ws = torch.empty(int(_lib.load().alm_encodec_lstm_workspace(B, T)), device=x.device, dtype=torch.uint8)
    H = ENCODEC_LSTM_H
    with _timed("encodec_lstm", 2.0 * B * T * 2 * 4 * H * 2 * H):
        _lib.call("alm_encodec_lstm", x, w, b, y, ws, B, T, int(elu_out), int(c8s))
    if check and int(ws[-12:-8].view(torch.int32).item()) != 0:
        raise _lib.AlmError("alm_encodec_lstm: a device-wide barrier timed out (the output is not valid)")
    return y


def pack_encodec_resblock(w3, w1, ws):
    """resnet-block weights w3 [C/2, C, 3], w1 [C, C/2], ws [C, C] (fp32) -> the 5-tap unit layout of
    alm_encodec_resblock_tc: W3's taps with rows zero-padded to C, W1 with columns zero-padded to C, then Ws."""
    C = ws.shape[0]
    w = torch.zeros(C, C, 5, device=ws.device, dtype=f32)
    w[: C // 2, :, :3] = w3.detach().float()
    w[:, : C // 2, 3] = w1.detach().float()
    w[:, :, 4] = ws.detach().float()
    return _split_units(w)


def encodec_resblock_tc(x, w_units, b3_pad, b_out, *, elu_out, out_phases=1):
    """the resnet block on C8S activations (P = 1 in, `out_phases` planes out) on the tensor cores; w_units from
    pack_encodec_resblock, b3_pad = b3 zero-padded to C."""
    _check_cuda(x, w_units, b3_pad, b_out)
    B, nch2, P, T, _ = x.shape
    C = nch2 * 4
    assert P == 1 and x.dtype == bf16 and x.is_contiguous() and w_units.dtype == bf16 and w_units.is_contiguous()
    assert w_units.numel() == 5 * (C // 16) * 2 * 2 * C * 8 and b3_pad.numel() == C and b_out.numel() == C
    y = torch.empty(B, nch2, out_phases, T // out_phases, 8, device=x.device, dtype=bf16)
    with _timed("encodec_resblock_tc", 2.0 * B * T * 5 * C * C):
        _lib.call("alm_encodec_resblock_tc", x, y, w_units, b3_pad, b_out, B, C, T, int(elu_out), int(out_phases))
    return y



SQ_MODES = {"fsq": 0, "lfq": 1}


def fsq_constants(levels, num_quantizers):
    """per-dimension constants of residual FSQ as vector-quantize-pytorch computes them, in torch fp32 on the CPU:
    (consts fp32 [4 + Q, dc] = half_l, offset, shift, L // 2, then scale[q] = (L - 1) ** -q; ints int32 [2, dc] =
    levels, basis = cumprod([1, L_0, ..., L_{dc-2}])).  The kernels take these as they are, so the rounding boundaries
    they quantize against are bit-identical to the quantizer's."""
    lv = torch.tensor(levels, dtype=torch.int32)
    half_l = (lv - 1) * (1 + 1e-3) / 2
    offset = torch.where(lv % 2 == 0, 0.5, 0.0)
    shift = (offset / half_l).atanh()
    scales = torch.stack([(torch.tensor(levels, dtype=f32) - 1) ** -q for q in range(num_quantizers)])
    basis = torch.cumprod(torch.tensor([1] + list(levels[:-1])), dim=0, dtype=torch.int32)
    consts = torch.cat((torch.stack((half_l, offset, shift, (lv // 2).to(f32))), scales)).to(f32).contiguous()
    return consts, torch.stack((lv, basis)).contiguous()


def lfq_constants(codebook_dim, num_quantizers):
    """the same layout for residual LFQ: scale[q] = 2 ** -q in every dimension, basis_j = 2 ** (dc - 1 - j) (most
    significant bit first); the FSQ rows are unused (zero) and every level is 2."""
    dc = codebook_dim
    scales = torch.tensor([2.0 ** -q for q in range(num_quantizers)], dtype=f32)[:, None].expand(-1, dc)
    consts = torch.cat((torch.zeros(4, dc, dtype=f32), scales)).contiguous()
    basis = 2 ** torch.arange(dc - 1, -1, -1, dtype=torch.int32)
    return consts, torch.stack((torch.full((dc,), 2, dtype=torch.int32), basis)).contiguous()


def _sq_args(mode, groups, Dg, weights, consts, ints):
    assert mode in SQ_MODES and consts.dtype == f32 and ints.dtype == torch.int32
    dc, Q = consts.shape[1], consts.shape[0] - 4
    assert weights is not None or Dg == dc, "the projections (Dg != dc) need their weights"
    w_in, b_in, w_out_t, b_out = weights if Dg != dc else (None,) * 4
    return dc, Q, w_in, b_in, w_out_t, b_out


def sq_encode(x, *, mode, groups, weights, consts, ints, index_dtype):
    """residual FSQ / LFQ (csrc/scalar_quant.cu): x [N, groups * Dg] fp32 (row stride free) -> (quantized [N, groups * Dg]
    fp32, indices [groups, N, Q] of index_dtype, int32 or int64).  consts / ints from fsq_constants / lfq_constants on
    x's device; weights = (w_in [g, dc, Dg], b_in [g, dc], w_out_t [g, dc, Dg], b_out [g, Dg]) fp32 contiguous, ignored
    when Dg == dc (identity projections)."""
    _check_cuda(x, consts, ints)
    assert x.dtype == f32 and x.stride(-1) == 1 and x.shape[1] % groups == 0 and index_dtype in (torch.int32, torch.int64)
    N, D = x.shape
    Dg = D // groups
    dc, Q, w_in, b_in, w_out_t, b_out = _sq_args(mode, groups, Dg, weights, consts, ints)
    quant = torch.empty(N, D, device=x.device, dtype=f32)
    idx = torch.empty(groups, N, Q, device=x.device, dtype=index_dtype)
    with _timed("sq_encode", 4.0 * N * D * dc if Dg != dc else 0.0):
        _lib.call("alm_sq_encode", x, x.stride(0), N, groups, Dg, SQ_MODES[mode], w_in, b_in, w_out_t, b_out, consts,
                  ints, dc, Q, quant, D, idx, int(index_dtype == torch.int64))
    return quant, idx


def sq_decode(indices, *, mode, Dg, weights, consts, ints):
    """get_output_from_indices of sq_encode's quantizer: indices [groups, N, q'] int32 / int64, q' <= Q, -1 = dropped
    -> fp32 [N, groups * Dg] = project_out(sum of the codes).  Bit-identical to sq_encode's quantized on its own
    indices."""
    _check_cuda(indices, consts, ints)
    assert indices.dtype in (torch.int32, torch.int64)
    indices = indices.contiguous()
    groups, N, Qi = indices.shape
    dc, Q, _, _, w_out_t, b_out = _sq_args(mode, groups, Dg, weights, consts, ints)
    out = torch.empty(N, groups * Dg, device=indices.device, dtype=f32)
    _lib.call("alm_sq_decode", indices, int(indices.dtype == torch.int64), Qi, N, groups, Dg, SQ_MODES[mode], w_out_t,
              b_out, consts, ints, dc, Q, out, groups * Dg)
    return out


def topk_gumbel_sample(logits, uniform, *, k, temperature=1.0):
    """ids [R] = Gumbel-max sample over the k largest logits of each row (noise supplied by the caller)."""
    _check_cuda(logits, uniform)
    assert logits.dtype == f32 and uniform.dtype == f32 and logits.shape == uniform.shape
    assert logits.stride(-1) == 1 and uniform.stride(-1) == 1
    R, V = logits.shape
    ids = torch.empty(R, device=logits.device, dtype=torch.int64)
    _lib.call("alm_topk_gumbel_sample", logits, logits.stride(0), uniform, uniform.stride(0), ids, R, V, int(k),
              float(temperature))
    return ids


def resid_ln_fwd(r, y, gamma, *, want_r_new=True, want_raw=False):
    """plain residual + LayerNorm (num_residual_streams == 1).  r [M,d] fp32, y [M,d] bf16 or None.

    Returns r_new [M,d] fp32 (== r when y is None and want_r_new False), xn bf16, raw bf16 copy (optional), stats."""
    M, d = r.shape
    r_new = torch.empty_like(r) if (want_r_new and y is not None) else None
    xn = torch.empty(M, d, device=r.device, dtype=bf16)
    raw = torch.empty(M, d, device=r.device, dtype=bf16) if want_raw else None
    stats = torch.empty(M, 2, device=r.device, dtype=f32)
    _lib.call("alm_resid_ln_fwd", r, y, gamma, r_new, xn, raw, stats, M, d)
    return (r_new if r_new is not None else r), xn, raw, stats


def resid_ln_bwd(r_new, gamma, stats, dr_out, dxn, dextra, g_gamma, *, out_scale=1.0, want_bf16=True):
    """dr = out_scale * (dr_out + LN_bwd(dxn) + dextra) as fp32 (and bf16 for the next GEMMs)."""
    M, d = r_new.shape
    dr = torch.empty(M, d, device=r_new.device, dtype=f32)
    dr_b = torch.empty(M, d, device=r_new.device, dtype=bf16) if want_bf16 else None
    _lib.call("alm_resid_ln_bwd", r_new, gamma, stats, dr_out, dxn, dextra, dr, dr_b, g_gamma, float(out_scale), M, d)
    return dr, dr_b


# ---- HuBERT feature path (csrc/hubert.cu; the network itself is audiolm_pytorch_b200/hubert.py) ----------------------
def pack_split_weight(w):
    """fp32 weight [N, K] -> bf16 [N, 3K] = [w_hi | w_hi | w_lo], the B operand of a split-bf16 GEMM against activation
    rows [x_hi | x_lo | x_hi] (the packing of rvq_pack_codebooks, without its padding)"""
    _check_cuda(w)
    return _split_pack(w.to(f32).contiguous())[0]


def pack_split_conv_weight(w):
    """conv weight [Cout, Cin, k] -> bf16 [Cout, k * 3 Cin]: per output channel, the k taps' packed rows in tap order,
    matching a window of k split rows of the input"""
    Cout, Cin, k = w.shape
    return pack_split_weight(w.permute(0, 2, 1).reshape(Cout * k, Cin)).view(Cout, k * 3 * Cin)


def split_gemm(xs, w_packed, bias=None, cls="hubert_gemm"):
    """fp32 [..., N] = x @ w^T (+ bias) for x in the split layout xs [..., 3K] and w_packed = pack_split_weight(w)"""
    lead = xs.shape[:-1]
    out = gemm(xs.reshape(-1, xs.shape[-1]), w_packed, out_dtype=f32, bias=bias, cls=cls)
    return out.view(*lead, w_packed.shape[0])


def hubert_conv_gemm(xs, w_packed, bias, *, kernel_size, stride, cls="hubert_conv_gemm"):
    """strided conv over the split layout xs [B, T, 3C] -> fp32 [B, T_out, Cout], one GEMM per clip whose A rows
    overlap: output row t reads the kernel_size * 3C elements from row t * stride.  w_packed = pack_split_conv_weight(w).
    (Clips run as separate GEMMs because every clip shares the weight, which the batched GEMM would need as a stride-0
    operand.)"""
    B, T, C3 = xs.shape
    assert xs.is_contiguous()
    T_out = (T - kernel_size) // stride + 1
    a = xs.as_strided((B, T_out, kernel_size * C3), (T * C3, stride * C3, 1))
    out = torch.empty(B, T_out, w_packed.shape[0], device=xs.device, dtype=f32)
    for b in range(B):
        gemm(a[b], w_packed, out=out[b], bias=bias, cls=cls)
    return out


def hubert_pos_conv(x, w_packed, *, kernel_size, cls="hubert_pos_gemm"):
    """grouped positional conv (padding kernel_size // 2, the first T outputs kept) of x fp32 [B, T, D], without its
    bias: per clip one GEMM batched over the groups, from the zero-padded group-major split copy (alm_hubert_pos_pack)
    with overlapping A rows.  w_packed: [groups, D / groups, kernel_size * 3 D / groups] (per group
    pack_split_conv_weight).  -> fp32 [B, groups, T, D / groups]"""
    _check_cuda(x, w_packed)
    B, T, D = x.shape
    G, Dg, Kp = w_packed.shape
    k = kernel_size
    Tp = T + k - 1
    xp = torch.empty(B, G, Tp, 3 * Dg, device=x.device, dtype=bf16)
    _lib.call("alm_hubert_pos_pack", x, xp, B, T, D, G, k // 2, Tp)
    out = torch.empty(B, G, T, Dg, device=x.device, dtype=f32)
    for b in range(B):
        a = xp[b].as_strided((G, T, Kp), (Tp * 3 * Dg, 3 * Dg, 1))
        gemm(a, w_packed, out=out[b], cls=cls)
    return out


def hubert_conv0(wave, w, bias, *, stride):
    """first conv of the feature extractor: wave fp32 [B, T], w [C, 1, K] (+ bias [C]) -> fp32 [B, T1, C]"""
    _check_cuda(wave, w, bias)
    B, T = wave.shape
    C, _, K = w.shape
    y = torch.empty(B, (T - K) // stride + 1, C, device=wave.device, dtype=f32)
    _lib.call("alm_hubert_conv0", wave, w, bias, y, B, T, C, K, stride)
    return y


def hubert_chan_stats(y):
    """GroupNorm(C, C) statistics of y fp32 [B, T, C] over time -> fp32 [B, C, 2] = {mean, 1 / sqrt(var + 1e-5)}"""
    B, T, C = y.shape
    stats = torch.empty(B, C, 2, device=y.device, dtype=f32)
    _lib.call("alm_hubert_chan_stats", y, stats, B, T, C)
    return stats


def hubert_norm_act(y, *, bias=None, stats=None, ln=False, gamma=None, beta=None, gelu=False, want_out=False,
                    want_split=True):
    """per row of y fp32 [..., C]: (+ bias), GroupNorm (stats from hubert_chan_stats, y [B, T, C]) or LayerNorm (ln),
    gamma / beta, GELU -> (fp32 [..., C] or None, split bf16 [..., 3C] or None)"""
    _check_cuda(y, bias, stats, gamma, beta)
    C = y.shape[-1]
    M = y.numel() // C
    mode = 1 if stats is not None else 2 if ln else 0
    want_out = want_out or (mode == 2 and bias is not None)
    out = torch.empty_like(y) if want_out else None
    split = torch.empty(*y.shape[:-1], 3 * C, device=y.device, dtype=bf16) if want_split else None
    _lib.call("alm_hubert_norm_act", y, bias, mode, stats, y.shape[1] if mode == 1 else 0, gamma, beta, int(gelu), out,
              split, M, C)
    return out, split


def hubert_add_ln(r, y=None, *, T, groups=1, y_bias=None, y_gelu=False, gamma=None, beta=None, keep_ln=False,
                  want_split=True):
    """in place on the residual stream r fp32 [B * T, D] (or [B, T, D]): r_new = r + act(y + y_bias); with gamma,
    LayerNorm(r_new) gamma + beta goes to the returned split bf16 [..., 3D] and, if keep_ln, into r"""
    _check_cuda(r, y, y_bias, gamma, beta)
    D = r.shape[-1]
    split = torch.empty(*r.shape[:-1], 3 * D, device=r.device, dtype=bf16) if (want_split and gamma is not None) else None
    _lib.call("alm_hubert_add_ln", r, y, groups, T, y_bias, int(y_gelu), gamma, beta, int(keep_ln), r, split,
              r.numel() // D, D)
    return split


def hubert_attention(qkv, *, heads):
    """multi-head self-attention (no mask, not causal) on the bf16 attention kernel: qkv fp32 [B, T, 3D] (q | k | v,
    biases included) -> the merged heads in the split layout bf16 [B, T, 3D], for the output projection"""
    _check_cuda(qkv)
    B, T, D3 = qkv.shape
    D = D3 // 3
    dh = D // heads
    q, k, v = (torch.empty(B * heads, T, dh, device=qkv.device, dtype=bf16) for _ in range(3))
    _lib.call("alm_hubert_qkv_heads", qkv, q, k, v, B, T, D, heads)
    o, _ = mqa_attn_fwd(q, k, v, heads=1, causal=False, scale=dh ** -0.5, return_lse=False)
    split = torch.empty(B, T, 3 * D, device=qkv.device, dtype=bf16)
    _lib.call("alm_hubert_merge_heads", o, split, B, T, D, heads)
    return split


# ---- vq-wav2vec feature path (csrc/vq_wav2vec.cu; the network itself is audiolm_pytorch_b200/vq_wav2vec.py) ----------
W2V_STATS_ROWS = 64  # ALM_W2V_STATS_ROWS: rows per fp64 partial of alm_w2v_group_stats
W2V_ACT = {None: 0, "relu": 1, "gelu": 2}


def w2v_group_stats(y, groups=1):
    """GroupNorm(groups, C) statistics of y fp32 [B, T, C] over the (C / groups) x T elements of each group ->
    fp32 [B, groups, 2] = {mean, 1 / sqrt(var + 1e-5)}; fixed-order fp64 partial sums, so batch-independent"""
    _check_cuda(y)
    assert y.dtype == f32 and y.is_contiguous()
    B, T, C = y.shape
    stats = torch.empty(B, groups, 2, device=y.device, dtype=f32)
    work = torch.empty(B * groups * -(-T // W2V_STATS_ROWS) * 2, device=y.device, dtype=torch.float64)
    _lib.call("alm_w2v_group_stats", y, stats, work, B, T, C, groups)
    return stats


def w2v_norm_act(y, stats, *, gamma=None, beta=None, act=None, residual=None, step=1, residual_scale=1.0,
                 log_compress=False, want_out=False, want_split=True):
    """per element of y fp32 [B, T, C]: GroupNorm with stats [B, G, 2] (w2v_group_stats), the optional per-channel
    gamma / beta, act (None, "relu" or "gelu"); with residual fp32 [B, Tr, C]:
    (v + residual[:, ::step][:, :T]) * residual_scale; log(|v| + 1) if log_compress
    -> (fp32 [B, T, C] or None, split bf16 [B, T, 3C] or None)"""
    _check_cuda(y, stats, gamma, beta, residual)
    assert y.dtype == f32 and y.is_contiguous() and (residual is None or residual.is_contiguous())
    B, T, C = y.shape
    out = torch.empty_like(y) if want_out else None
    split = torch.empty(B, T, 3 * C, device=y.device, dtype=bf16) if want_split else None
    Tr = residual.shape[1] if residual is not None else 0
    _lib.call("alm_w2v_norm_act", y, stats, gamma, beta, W2V_ACT[act], residual, Tr, int(step), float(residual_scale),
              int(log_compress), out, split, B, T, C, stats.shape[1])
    return out, split


# ---- band-limited resampling (csrc/resample.cu) ----------------------------------------------------------------------
RESAMPLE_ZEROS = 6        # torchaudio's lowpass_filter_width, the reference never changes it
RESAMPLE_ROLLOFF = 0.99   # torchaudio's rolloff, likewise


def resample_rates(orig_hz, new_hz):
    """the rates reduced by their gcd, (o, n); ValueError for a non-positive or non-integer rate, as torchaudio"""
    for r in (orig_hz, new_hz):
        if not r > 0:
            raise ValueError(f"resample: sample rates must be positive, got {orig_hz} -> {new_hz}")
        if int(r) != r:
            raise ValueError(f"resample: sample rates must be integers, got {orig_hz} -> {new_hz}")
    o, n = int(orig_hz), int(new_hz)
    g = math.gcd(o, n)
    return o // g, n // g


def resample_length(L, orig_hz, new_hz):
    """samples torchaudio.functional.resample makes of L input samples: ceil(n L / o)"""
    o, n = resample_rates(orig_hz, new_hz)
    return -(-n * L // o)


@functools.lru_cache(maxsize=None)
def resample_table(o, n):
    """compact polyphase filter of the reduced rates o -> n (o != n), in fp64: (taps [n, T], first [n], counts [n]).

    torchaudio's dense filter is K[p, m] = (base / o) sinc(pi t) cos^2(pi t / 12), m < 2 width + o, with
    t = clamp(base ((m - width) / o - p / n), -6, 6), base = 0.99 min(o, n), width = ceil(6 o / base).  Phase p keeps
    the taps with |t| < 6 before the clamp, a run of counts[p] taps from input offset first[p] relative to k o: at
    |t| = 6 the window is cos^2(pi / 2), so every dropped tap is below 1e-48.  t is formed with the same fp64 operations
    as torchaudio, so the kept taps are torchaudio's fp64 taps.  Row p of taps holds the run, zero-padded to
    T = max(counts)."""
    assert o > 0 and n > 0 and o != n and math.gcd(o, n) == 1
    f64 = torch.float64
    base = min(o, n) * RESAMPLE_ROLLOFF
    width = math.ceil(RESAMPLE_ZEROS * o / base)
    # t rises by base / o <= 0.99 per tap: the run of |t| < 6 is at most 12 o / base + 1 taps long and starts after
    # m = width + o (p / n - 6 / base); evaluate two taps of margin on each side
    span = math.floor(2 * RESAMPLE_ZEROS * o / base) + 6
    p = torch.arange(n, dtype=f64)
    m = torch.floor(width + o * (p / n - RESAMPLE_ZEROS / base)).long()[:, None] - 2 + torch.arange(span)
    t = ((-p / n)[:, None] + (m - width).to(f64) / o) * base
    assert bool((t[:, 0] <= -RESAMPLE_ZEROS).all() and (t[:, -1] >= RESAMPLE_ZEROS).all())
    keep = (t.abs() < RESAMPLE_ZEROS) & (m >= 0) & (m < 2 * width + o)
    counts = keep.sum(1)
    lead = keep.long().argmax(1)
    T = int(counts.max())
    i = torch.arange(T)
    valid = i[None] < counts[:, None]
    col = (lead[:, None] + i).clamp(max=span - 1)
    tk = t.gather(1, col)
    window = torch.cos(tk * math.pi / RESAMPLE_ZEROS / 2) ** 2
    tk = tk * math.pi
    taps = torch.where(tk == 0, torch.ones_like(tk), tk.sin() / tk) * (window * (base / o))
    taps = torch.where(valid, taps, torch.zeros_like(taps))
    first = m.gather(1, lead[:, None])[:, 0] - width
    return taps, first, counts


_RESAMPLE_DEVICE_TABLES: dict = {}


def _resample_device_table(o, n, device):
    key = (o, n, device)
    if key not in _RESAMPLE_DEVICE_TABLES:
        taps, first, _ = resample_table(o, n)
        _RESAMPLE_DEVICE_TABLES[key] = (taps.t().to(f32).contiguous().to(device),
                                        first.to(torch.int32).to(device), taps.shape[1])
    return _RESAMPLE_DEVICE_TABLES[key]


def resample(x, orig_hz, new_hz, *, start=0, count=None):
    """torchaudio.functional.resample(x, orig_hz, new_hz) with its defaults (Hann-windowed sinc, 6 zero crossings,
    rolloff 0.99) on the compact polyphase filter, one launch: x CUDA [..., L], any float dtype -> fp32 [..., count],
    the output samples [start, start + count) of the ceil(n L / o) torchaudio makes (count=None: up to the end).

    Computes in fp32; a row's output is bitwise the same alone or in a batch.  orig_hz == new_hz returns the input
    unchanged (sliced to the window), as torchaudio does.  No autograd.  Rates must be positive integers (ValueError)."""
    o, n = resample_rates(orig_hz, new_hz)
    L = x.shape[-1]
    total = -(-n * L // o)
    if count is None:
        count = total - start
    if not (0 <= start and 0 <= count and start + count <= total):
        raise ValueError(f"resample: window [{start}, {start} + {count}) is outside the {total} output samples")
    if o == n:
        return x if (start, count) == (0, L) else x[..., start:start + count]
    _check_cuda(x)
    lead = x.shape[:-1]
    y = torch.empty(*lead, count, device=x.device, dtype=f32)
    rows = y.numel() // count if count else 0
    if rows == 0 or L == 0:
        return y.zero_()
    x2 = x.detach().reshape(rows, L)
    if x2.dtype != f32 or x2.stride(1) != 1 or (rows > 1 and x2.stride(0) < L):
        x2 = x2.to(f32).contiguous()
    taps, first, T = _resample_device_table(o, n, x.device)
    with _timed("resample", 4.0 * rows * (L + count), unit="byte"):
        _lib.call("alm_resample", x2, x2.stride(0) if rows > 1 else L, L, y, start, count, rows, taps, first, T, o, n)
    return y
