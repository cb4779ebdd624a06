"""Functional fp32 CPU oracle of SoundStream(squeeze_excite=True) — TEST INFRASTRUCTURE ONLY.

Restates /root/reference/audiolm_pytorch/soundstream.py:145-169 (SqueezeExcite) and :362-369 (ResidualUnit with
`squeeze_excite=True`, the SE module at Sequential index 4 once the reference's `Sequential` drops the None) on top of
oracle/codec.py, whose SE-free encoder / decoder this mirrors layer by layer.  Pinned against the reference by
oracle/make_golden_codec_options.py.

Reference quirk reproduced on purpose: SqueezeExcite.forward receives [B, C, T] but takes `seq = x.shape[-2]` and
cumsums dim -2, so its "cumulative mean" runs over CHANNELS (m[c, t] = mean_{c' <= c} y[c', t]), not over time.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from . import codec as oc
from .transformer import sub


def squeeze_excite(st, y):
    """SqueezeExcite(C) on y [b, C, t] with keys net.0.{weight,bias} [Ci, C, 1], net.2.{weight,bias} [C, Ci, 1]."""
    C = y.shape[-2]
    m = y.cumsum(dim=-2) / torch.arange(1, C + 1, dtype=y.dtype, device=y.device)[:, None]  # mean over channels 0..c
    s = F.silu(torch.einsum("ic,bct->bit", st["net.0.weight"][..., 0], m) + st["net.0.bias"][:, None])
    gate = torch.sigmoid(torch.einsum("ci,bit->bct", st["net.2.weight"][..., 0], s) + st["net.2.bias"][:, None])
    return y * gate


def residual_unit(st, x, dilation, pad_mode="reflect"):
    """x + SE(ELU(conv1(ELU(conv7_dil(x))))); the SE term only when the unit has keys fn.4.*"""
    h = F.elu(oc.causal_conv1d(x, st["fn.0.conv.weight"], st["fn.0.conv.bias"], dilation=dilation, pad_mode=pad_mode))
    h = F.elu(oc.causal_conv1d(h, st["fn.2.conv.weight"], st["fn.2.conv.bias"], pad_mode=pad_mode))
    if "fn.4.net.0.weight" in st:
        h = squeeze_excite(sub(st, "fn.4"), h)
    return x + h


def encoder(st, x, strides=(2, 4, 5, 8), dilations=(1, 3, 9), pad_mode="reflect"):
    """SoundStream.encoder (soundstream.py:519-531) with SE residual units: [b, c_in, T] -> [b, D, T/prod(strides)]."""
    x = oc.causal_conv1d(x, st["0.conv.weight"], st["0.conv.bias"], pad_mode=pad_mode)
    for bi, s in enumerate(strides, start=1):
        for ri, d in enumerate(dilations):
            x = residual_unit(sub(st, f"{bi}.{ri}"), x, d, pad_mode)
        # the reference's EncoderBlock builds its strided conv without pad_mode: always reflect
        x = oc.causal_conv1d(x, st[f"{bi}.3.conv.weight"], st[f"{bi}.3.conv.bias"], stride=s)
    last = len(strides) + 1
    return oc.causal_conv1d(x, st[f"{last}.conv.weight"], st[f"{last}.conv.bias"], pad_mode=pad_mode)


def decoder(st, x, strides=(2, 4, 5, 8), dilations=(1, 3, 9), pad_mode="reflect"):
    """SoundStream.decoder (soundstream.py:615-627) with SE residual units: [b, D, n] -> [b, c_in, n*prod(strides)]."""
    x = oc.causal_conv1d(x, st["0.conv.weight"], st["0.conv.bias"], pad_mode=pad_mode)
    for bi, s in enumerate(reversed(strides), start=1):
        x = oc.causal_conv_transpose1d(x, st[f"{bi}.0.conv.weight"], st[f"{bi}.0.conv.bias"], s)
        for ri, d in enumerate(dilations, start=1):
            x = residual_unit(sub(st, f"{bi}.{ri}"), x, d, pad_mode)
    last = len(strides) + 1
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
