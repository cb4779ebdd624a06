"""Functional fp32 / fp64 CPU oracle of SoundStream(use_gate_loop_layers=True) — TEST INFRASTRUCTURE ONLY.

The reference imports `SimpleGateLoopLayer` from gateloop-transformer (soundstream.py:29), which is not vendored and
cannot be installed offline.  `SimpleGateLoopLayer` below restates the published layer's eval path (PARITY UNPINNED
against the package, as for hyper-connections and local-attention); oracle/make_golden_gate_loop.py runs the
reference's own soundstream.py on top of it.  oracle/ref_import.py still stubs `gateloop_transformer` with `_Absent`,
so a script that builds the reference with `use_gate_loop_layers=True` must first bind the reference module's `GateLoop`
name to `SimpleGateLoopLayer`, as make_golden_gate_loop.main() does (SoundStream.__init__ looks the name up at
construction).  The functional encoder / decoder mirror oracle/codec_se.py layer by layer, with a gate-loop layer after
every block (soundstream.py:522-525, 618-621).

On x [b, C, n] the reference computes Residual(ChannelTranspose(GateLoop(C)))(x), u_t = x[:, :, t]:
    x^_t = u_t / max(||u_t||, 1e-12) * sqrt(C) * gamma,   [q; kv; a]_t = W x^_t,   W = to_qkva.0.weight [3C, C]
    h_t = sigmoid(a_t) h_{t-1} + kv_t  (h_{-1} = 0),      out_t = 2 u_t + q_t h_t
The factor 2 is a reference quirk: ChannelTranspose.forward returns fn(x) + x and Residual adds x once more.  The
encoder's `use_heinsen=False` and the decoder's package default evaluate the same recurrence.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F
from torch import nn

from . import codec as oc
from . import codec_se as ose
from .transformer import sub


def linear_scan(a, kv):
    """h_t = a_t h_{t-1} + kv_t along the last dim, h_{-1} = 0: a Hillis-Steele scan of (A, H) pairs, log2(n) steps."""
    A, H = a.clone(), kv.clone()
    n, d = a.shape[-1], 1
    while d < n:
        H = torch.cat((H[..., :d], torch.addcmul(H[..., d:], A[..., d:], H[..., :-d])), dim=-1)
        A = torch.cat((A[..., :d], A[..., d:] * A[..., :-d]), dim=-1)
        d *= 2
    return H


def gate_loop(st, x):
    """GateLoop(C) (SimpleGateLoopLayer) on x [b, C, n] -> q * h [b, C, n]; keys norm.gamma, to_qkva.0.weight"""
    C = x.shape[-2]
    xn = F.normalize(x, dim=-2) * math.sqrt(C) * st["norm.gamma"][:, None]
    q, kv, a = torch.einsum("oc,bcn->bon", st["to_qkva.0.weight"], xn).split(C, dim=-2)
    return q * linear_scan(torch.sigmoid(a), kv)


def gate_loop_block(st, x):
    """Residual(ChannelTranspose(GateLoop(C))) on x [b, C, n]; keys fn.fn.*"""
    return 2 * x + gate_loop(sub(st, "fn.fn"), x)


class SimpleGateLoopLayer(nn.Module):
    """gateloop-transformer's SimpleGateLoopLayer, eval path on x [b, n, dim] -> q * h.  Keys `norm.gamma`,
    `to_qkva.0.weight`; the `cache` / `return_cache` streaming arguments are not restated (soundstream.py never passes
    them)."""

    def __init__(self, dim, prenorm=True, use_heinsen=False, use_jax_associative_scan=False, post_ln=False,
                 reverse=False):
        super().__init__()
        assert prenorm and not post_ln and not reverse, "only the configuration soundstream.py builds is restated"
        self.norm = nn.Module()
        self.norm.gamma = nn.Parameter(torch.ones(dim))
        self.to_qkva = nn.Sequential(nn.Linear(dim, 3 * dim, bias=False))

    def forward(self, x):
        st = {"norm.gamma": self.norm.gamma, "to_qkva.0.weight": self.to_qkva[0].weight}
        return gate_loop(st, x.transpose(1, 2)).transpose(1, 2)


def _has_gate_loops(st):
    return "2.fn.fn.norm.gamma" in st


def encoder(st, x, strides=(2, 4, 5, 8), dilations=(1, 3, 9), pad_mode="reflect"):
    """SoundStream.encoder (soundstream.py:519-531) with a gate-loop layer after each block: [b, 1, T] -> [b, D, n]."""
    assert _has_gate_loops(st)
    x = oc.causal_conv1d(x, st["0.conv.weight"], st["0.conv.bias"], pad_mode=pad_mode)
    for i, s in enumerate(strides):
        blk = sub(st, f"{2 * i + 1}")
        for ri, d in enumerate(dilations):
            x = ose.residual_unit(sub(blk, f"{ri}"), x, d, pad_mode)
        # the reference's EncoderBlock builds its strided conv without pad_mode: always reflect
        x = oc.causal_conv1d(x, blk["3.conv.weight"], blk["3.conv.bias"], stride=s)
        x = gate_loop_block(sub(st, f"{2 * i + 2}"), x)
    last = 2 * len(strides) + 1
    return oc.causal_conv1d(x, st[f"{last}.conv.weight"], st[f"{last}.conv.bias"], pad_mode=pad_mode)


def decoder(st, x, strides=(2, 4, 5, 8), dilations=(1, 3, 9), pad_mode="reflect"):
    """SoundStream.decoder (soundstream.py:615-627) with a gate-loop layer after each block: [b, D, n] -> [b, 1, T]."""
    assert _has_gate_loops(st)
    x = oc.causal_conv1d(x, st["0.conv.weight"], st["0.conv.bias"], pad_mode=pad_mode)
    for i, s in enumerate(reversed(strides)):
        blk = sub(st, f"{2 * i + 1}")
        x = oc.causal_conv_transpose1d(x, blk["0.conv.weight"], blk["0.conv.bias"], s)
        for ri, d in enumerate(dilations, start=1):
            x = ose.residual_unit(sub(blk, f"{ri}"), x, d, pad_mode)
        x = gate_loop_block(sub(st, f"{2 * i + 2}"), x)
    last = 2 * len(strides) + 1
    return oc.causal_conv1d(x, st[f"{last}.conv.weight"], st[f"{last}.conv.bias"], pad_mode=pad_mode)


def soundstream_tokenize(st, wave, strides=(2, 4, 5, 8)):
    """forward(..., return_encoded=True) without local attention, one RVQ group: wave [b, T] -> (quantized, indices)"""
    x = encoder(sub(st, "encoder"), wave[:, None, :], strides).transpose(1, 2)
    b, n, D = x.shape
    q, i = oc.rvq_encode(x.reshape(b * n, D), oc.codebooks_of(st))
    return q.reshape(b, n, D), i.reshape(b, n, -1)


def soundstream_decode_indices(st, indices, strides=(2, 4, 5, 8)):
    """decode_from_codebook_indices, one RVQ group: indices [b, n, q] -> wave [b, 1, T]"""
    b, n, q = indices.shape
    x = oc.rvq_decode(indices.reshape(b * n, q), oc.codebooks_of(st)).reshape(b, n, -1).transpose(1, 2)
    return decoder(sub(st, "decoder"), x, strides)
