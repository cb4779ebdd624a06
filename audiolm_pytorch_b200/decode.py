"""CUDA-graph decode engine for the KV-cache sampling loops (config C5; audiolm_pytorch.py:1406-1511,
1608-1740, 1896-2039).

The reference (and `Transformer.forward` with a `kv_cache`) re-concatenate the per-layer cache with `torch.cat` every step
and launch ~60 kernels + as many torch ops per token from Python, so a token costs host and launch overhead rather
than GPU work.  Here one decode step

    embed(last token) -> 6 x [hyper-connection pre, q/kv GEMMs, kv append, decode attention, out GEMM,
                              hyper-connection pre, W1 GEMM, GEGLU+LN, W2 GEMM] -> post + LN -> head -> top-k Gumbel

works on STATIC buffers: the K/V cache is a preallocated [depth, b, max_len, dim_head] pair whose fill level lives in
a device int32 (`alm_kv_append`, `alm_mqa_attn_decode` read it at run time), the token goes in and out through a
device buffer.  The step is therefore captured ONCE per sampling position class in a CUDA graph and replayed per
token; the host only replays the graph and polls for EOS.

Every stack `Transformer` accepts runs here: the plain residual (num_residual_streams=1) takes resid_ln steps
instead of the hyper-connection ones, and a model with an additive attention bias (flash_attn=False: relative
position bias, the coarse cross bias, the fine 2-D bias) hands the engine a per-position description of it
(`StackDecoder.set_bias`); each step writes the new token's bias row once (`alm_decode_bias_row`) and every layer's
decode attention adds it to its scores.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from . import ops
from .transformer import Transformer, _pad8

bf16 = torch.bfloat16
f32 = torch.float32


# on = one persistent kernel per token (csrc/decode_step.cu) instead of ~11 launches per layer; off = the multi-kernel
# step replayed from a CUDA graph.  Off by default: on the H100 the one-kernel step measured slower (486 vs 401 us per
# token at batch 1, 600 cached positions; DESIGN.md §4.3).  Both paths are tested against each other.
FUSED_STACK_STEP = False


class StackDecoder:
    """One-token incremental forward of a `Transformer` stack against a static KV cache."""

    def __init__(self, tr: Transformer, batch: int, max_len: int):
        dev = next(tr.parameters()).device
        self.tr, self.b, self.max_len = tr, batch, max_len
        self.kc = torch.zeros(tr.depth, batch, max_len, tr.dim_head, device=dev, dtype=bf16)
        self.vc = torch.zeros_like(self.kc)
        self.len = torch.zeros(1, device=dev, dtype=torch.int32)
        # key mask (1 = attend): a STATIC buffer so that captured graphs keep pointing at it; all ones by default
        self.mask = torch.ones(batch, max_len, device=dev, dtype=torch.uint8)
        self.host_len = 0  # host mirror of `len` (graph replays advance it too): a full cache is an error, not a drop
        self._fused = None  # (signature, pointer table, scratch, out) of the one-kernel step
        self.bias = None    # static (table, override, u, cls, c, row) of the attention bias, see set_bias

    def _fused_state(self):
        """device pointer table + per-CTA regrouped operand copies of alm_decode_stack_step; rebuilt only when a
        parameter / packed copy changed (never during graph capture: the warm-up steps of GraphedStep build it)."""
        tr = self.tr
        Ws = [tr._weights(i) for i in range(tr.depth)]   # refreshes the packed bf16 copies if a weight moved
        small = []
        for attn_hc, _, ff_hc in tr.layers:
            f = ff_hc.branch
            small.append([*attn_hc.kernel_params().values(), attn_hc.branch.norm.gamma,
                          *ff_hc.kernel_params().values(), getattr(f, "0").gamma, getattr(f, "3").gamma])
        sig = (tuple(t.data_ptr() for ts in small for t in ts), tuple(w.data_ptr() for W in Ws for w in W.values()),
               tr.__dict__.get("_pack_ver"), tr._packed.generation)
        if self._fused is None or self._fused[0] != sig:
            dev = self.kc.device
            f0 = tr.layers[0][2].branch
            G = ops.decode_stack_grid()
            with torch.inference_mode(False), torch.no_grad():
                rows, keep = [], []
                for i, W in enumerate(Ws):
                    ts = small[i]
                    for t in ts:
                        assert t.dtype == f32 and t.is_contiguous()
                    wa = ops.regroup_rows(torch.cat((W["wq"], W["wkv"]), dim=0), G)
                    wc, wd, we = (ops.regroup_rows(W[k], G) for k in ("wo", "w1", "w2"))
                    keep.append((wa, wc, wd, we))
                    rows.append([t.data_ptr() for t in ts[:16]] + [wa.data_ptr(), 0, wc.data_ptr(), wd.data_ptr(),
                                we.data_ptr(), ts[16].data_ptr(), self.kc[i].data_ptr(), self.vc[i].data_ptr()])
                table = torch.tensor(rows, dtype=torch.int64, device=dev)
                scratch = ops.decode_stack_scratch(self.b, tr.dim, tr.heads, f0.inner, dev)
                out = torch.empty(self.b, tr.dim, device=dev, dtype=bf16)
            self._fused = (sig, table, scratch, out, keep, G)
        return self._fused

    def fused_ok(self):
        """the one-kernel step covers the 4-stream stack of head width 64 without an attention bias, at the sizes its
        kernel takes (ops.decode_stack_plan); everything else runs the multi-kernel step"""
        tr = self.tr
        return (FUSED_STACK_STEP and self.b <= ops.DECODE_STEP_MAX_ROWS and tr.num_residual_streams == 4
                and self.bias is None
                and ops.decode_stack_plan(self.b, tr.dim, tr.heads, tr.layers[0][2].branch.inner, tr.depth,
                                          dim_head=tr.dim_head) is not None)

    def barrier_timeouts(self) -> int:
        """sticky error flag of the one-kernel step (a device-wide barrier gave up waiting); 0 when healthy"""
        if self._fused is None:
            return 0
        return int(self._fused[2][256:260].view(torch.int32).item())

    def load_cache(self, kv):
        """kv: [depth, 2, b, n, dim_head] as returned by Transformer(..., return_kv_cache=True)"""
        n = kv.shape[-2]
        assert n <= self.max_len and kv.shape[2] == self.b
        self.kc[:, :, :n] = kv[:, 0].to(bf16)
        self.vc[:, :, :n] = kv[:, 1].to(bf16)
        self.len.fill_(n)
        self.host_len = n

    def set_key_mask(self, mask=None):
        """mask: bool [b, n] (True = attend) or None; positions past n (tokens still to be generated) are attended"""
        self.mask.fill_(1)
        if mask is not None:
            self.mask[:, :mask.shape[1]] = mask.to(torch.uint8)

    def set_bias(self, table, override, u, cls, c):
        """The additive attention bias shared by every layer and sequence, as the rule of `alm_decode_bias_row`:
        for the token at cache position L and keys j <= L,
            bias[h, j] = (cls[L] != cls[j] or cls[L] < 0) ? override[h] : table[u[L] - u[j] + c, h]
        table fp32 [P, H], override [H] or None, u / cls int32 [max_len] (the models' `decode_bias`).
        The first call allocates STATIC buffers that captured graphs keep pointing at; later calls rewrite them in
        place, so the table size, the presence of an override and c must not change (the engine cache keys on them)."""
        H = self.tr.heads
        assert table.dim() == 2 and table.shape[1] == H and u.shape == (self.max_len,) and cls.shape == (self.max_len,)
        if self.bias is None:
            dev = self.kc.device
            self.bias = (torch.empty(table.shape, device=dev, dtype=f32),
                         None if override is None else torch.empty(H, device=dev, dtype=f32),
                         torch.empty(self.max_len, device=dev, dtype=torch.int32),
                         torch.empty(self.max_len, device=dev, dtype=torch.int32), int(c),
                         torch.zeros(H, self.max_len, device=dev, dtype=f32))
        bt, bo, bu, bc, c0, _ = self.bias
        assert bt.shape == table.shape and (bo is None) == (override is None) and c0 == int(c), \
            "the bias table's size, override and c are fixed once set"
        bt.copy_(table.detach())
        if bo is not None:
            bo.copy_(override.detach().reshape(H))
        bu.copy_(u)
        bc.copy_(cls)

    @torch.no_grad()
    def step(self, x):
        """x [b, d] (embedding of the new token) -> normed output [b, d] bf16; appends to the cache, len += 1."""
        tr = self.tr
        b, d, H, D = self.b, tr.dim, tr.heads, tr.dim_head
        if tr.rel_pos_bias is not None and self.bias is None:
            raise ops._lib.AlmError("this stack has a relative position bias: set it with StackDecoder.set_bias "
                                    "(the models' decode_bias) before decoding")
        x2 = x.reshape(b, d).to(f32).contiguous()
        if self.fused_ok():
            _, table, scratch, out, _, G = self._fused_state()
            f0 = tr.layers[0][2].branch
            ops.decode_stack_step(table, x2, out, tr.norm.gamma, self.len, self.kc, self.mask, scratch, heads=H,
                                  inner=f0.inner, grid=G, value_residual=tr.add_value_residual)
            return out   # (the kernel advanced self.len)
        # a few rows: every Linear is a weight-read-bound matrix-vector product (alm_gemv_bf16 over all SMs)
        mm = (lambda a, w: ops.gemv(a, w)) if b <= 8 else (lambda a, w: ops.gemm(a, w))
        brow = None
        if self.bias is not None:   # the new token's bias row, read by every layer
            table, over, u, cls, c, brow = self.bias
            ops.decode_bias_row(table, over, u, cls, c, self.len, brow)
        # the residual stream as in Transformer._walk_forward: fp32 r (plain, resid_ln) or bf16 R [b, S, d]
        # (hyper-connections); `bin_` (the un-normalised branch input) feeds to_kv
        S = tr.num_residual_streams
        plain = S == 1
        hc0 = tr.layers[0][0]
        if plain:
            r, xn, bin_, _ = ops.resid_ln_fwd(x2, None, hc0.branch.norm.gamma, want_raw=True)
        else:
            R, bin_, xn, beta, _ = ops.hc_pre_fwd(hc0.kernel_params(), hc0.branch.norm.gamma, x_expand=x2, M=b, d=d,
                                                 streams=S)
        v_first = None
        for i, (attn_hc, _, ff_hc) in enumerate(tr.layers):
            W = tr._weights(i)
            f = ff_hc.branch
            inner, ip = f.inner, _pad8(f.inner)
            q = mm(xn, W["wq"])                      # [b, H*D]
            kv = mm(bin_, W["wkv"])                  # [b, 2*D]
            if tr.add_value_residual and v_first is not None:
                ops.axpby(kv[:, D:], 0.5, v_first, 0.5, out=kv[:, D:])
            elif tr.add_value_residual:
                v_first = kv[:, D:].clone()
            ops.kv_append(kv, self.kc[i], self.vc[i], self.len)
            o = ops.mqa_attn_decode(q, self.kc[i], self.vc[i], self.len, heads=H, key_mask=self.mask, bias=brow)
            Y = mm(o, W["wo"])
            if plain:
                r, xn2, _, _ = ops.resid_ln_fwd(r, Y, getattr(f, "0").gamma)
            else:
                R2, _, xn2, beta2, _ = ops.hc_pre_fwd(ff_hc.kernel_params(), getattr(f, "0").gamma, R_in=R, Y=Y,
                                                      beta_prev=beta, M=b, d=d, streams=S)
            h = mm(xn2, W["w1"])
            gn, _ = ops.geglu_ln_fwd(h, getattr(f, "3").gamma, inner=inner, inner_pad=ip)
            Y2 = mm(gn, W["w2"])
            if i + 1 < tr.depth:
                nxt = tr.layers[i + 1][0]
                if plain:
                    r, xn, bin_, _ = ops.resid_ln_fwd(r, Y2, nxt.branch.norm.gamma, want_raw=True)
                else:
                    R, bin_, xn, beta, _ = ops.hc_pre_fwd(nxt.kernel_params(), nxt.branch.norm.gamma, R_in=R2, Y=Y2,
                                                          beta_prev=beta2, M=b, d=d, streams=S)
        if plain:
            out = ops.resid_ln_fwd(r, Y2, tr.norm.gamma)[1]
        else:
            out, _ = ops.hc_post_fwd(R2, Y2, beta2, tr.norm.gamma, M=b, d=d, streams=S)
        self.len.add_(1)
        return out


class GraphedStep:
    """Capture `fn()` (which must only touch static buffers) in a CUDA graph after a warm-up on a side stream.
    `state` lists (tensor, ...) whose contents are restored after warm-up so the warm-up steps leave no trace."""

    def __init__(self, fn, state):
        saved = [t.clone() for t in state]
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(2):  # lazy weight packing, cudaFuncSetAttribute, allocator warm-up
                fn()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        for t, s in zip(state, saved):
            t.copy_(s)
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            fn()
        for t, s in zip(state, saved):  # capture does not execute, but keep the contract explicit
            t.copy_(s)

    def __call__(self):
        self.graph.replay()


class TokenDecoder:
    """Sampling loop state shared by the three wrappers: static token / sequence buffers + graphed steps.

    embed_fn(tok [b] int64, key) -> [b, d] embedding of the token just sampled
    logits_fn(out [b, d] bf16, key) -> fp32 logits [b, V] for the NEXT token (already EOS-masked if needed)
    `key` selects the sampling position class (quantizer index); one graph is captured per key."""

    def __init__(self, stack: StackDecoder, embed_fn, logits_fn, *, filter_thres, temperature, use_graph=True):
        dev = stack.kc.device
        self.stack, self.embed_fn, self.logits_fn = stack, embed_fn, logits_fn
        self.filter_thres, self.temperature = filter_thres, temperature
        self.tok = torch.zeros(stack.b, device=dev, dtype=torch.long)
        self.use_graph = use_graph
        self._graphs = {}

    def _step(self, key):
        out = self.stack.step(self.embed_fn(self.tok, key))
        logits = self.logits_fn(out, key).float().contiguous()
        k = max(int((1 - self.filter_thres) * logits.shape[-1]), 1)
        noise = torch.zeros_like(logits).uniform_(0, 1)
        self.tok.copy_(ops.topk_gumbel_sample(logits, noise, k=k, temperature=self.temperature))

    def advance(self, key=0):
        """consume self.tok (the token sampled last), append it to the cache, sample the next one into self.tok"""
        st = self.stack
        if st.host_len >= st.max_len:
            raise ops._lib.AlmError(f"decode KV cache is full ({st.max_len} positions); build the engine with a larger max_len")
        st.host_len += 1
        if not self.use_graph:
            return self._step(key)
        g = self._graphs.get(key)
        if g is None:
            g = self._graphs[key] = GraphedStep(lambda: self._step(key), [self.tok, self.stack.len])
        g()
