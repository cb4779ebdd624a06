"""Functional fp32 CPU oracle of the SoundStream codec hot path — TEST INFRASTRUCTURE ONLY.

Restates /root/reference/audiolm_pytorch/soundstream.py:332-395 (causal convs, residual units, encoder /
decoder blocks), :691-709 (decode_from_codebook_indices / decode), :797-866 (forward / tokenize) with
explicit index arithmetic (not F.pad + nn.Conv1d), plus the RVQ eval path of vector-quantize-pytorch
(PARITY UNPINNED upstream, see oracle/third_party.py).  Pinned by oracle/make_golden.py.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from .third_party import euclid_nearest
from .transformer import sub


def causal_pad(x, pad, mode="reflect"):
    """left padding of CausalConv1d (soundstream.py:339,344): reflect excludes the edge sample."""
    if pad == 0:
        return x
    if mode == "reflect":
        left = x[..., 1:pad + 1].flip(-1)
    elif mode == "replicate":
        left = x[..., :1].expand(*x.shape[:-1], pad)
    elif mode == "constant":
        left = x.new_zeros(*x.shape[:-1], pad)
    else:
        raise ValueError(mode)
    return torch.cat((left, x), dim=-1)


def causal_conv1d(x, weight, bias, stride=1, dilation=1, pad_mode="reflect"):
    """CausalConv1d (soundstream.py:332-345): y[o,t] = b[o] + sum_c sum_j W[o,c,j] xp[c, t*s + j*d]."""
    k = weight.shape[-1]
    pad = dilation * (k - 1) + 1 - stride
    xp = causal_pad(x, pad, pad_mode)
    t_out = (xp.shape[-1] - dilation * (k - 1) - 1) // stride + 1
    y = bias[None, :, None].expand(x.shape[0], -1, t_out).clone()
    for j in range(k):
        taps = xp[..., j * dilation: j * dilation + (t_out - 1) * stride + 1: stride]  # [b, c, t_out]
        y = y + torch.einsum("oc,bct->bot", weight[:, :, j], taps)
    return y


def causal_conv_transpose1d(x, weight, bias, stride):
    """CausalConvTranspose1d (soundstream.py:347-360): weight [c_in, c_out, 2s]; keep first n*s samples.

    y[o, i*s + r] = b[o] + sum_c W[c,o,r] x[c,i] + W[c,o,r+s] x[c,i-1]
    """
    b, c, n = x.shape
    s = stride
    assert weight.shape[-1] == 2 * s
    cur = torch.einsum("cor,bci->boir", weight[..., :s], x)            # taps r
    prev = torch.einsum("cor,bci->boir", weight[..., s:], F.pad(x, (1, 0))[..., :n])  # taps r+s on x[i-1]
    y = (cur + prev).reshape(b, -1, n * s)
    return y + bias[None, :, None]


def residual_unit(st, x, dilation, pad_mode="reflect"):
    """x + ELU(conv1(ELU(conv7_dil(x)))) (soundstream.py:362-369); keys fn.0.conv.*, fn.2.conv.*"""
    h = F.elu(causal_conv1d(x, st["fn.0.conv.weight"], st["fn.0.conv.bias"], dilation=dilation, pad_mode=pad_mode))
    h = F.elu(causal_conv1d(h, st["fn.2.conv.weight"], st["fn.2.conv.bias"], pad_mode=pad_mode))
    return x + h


def encoder(st, x, strides=(2, 4, 5, 8), dilations=(1, 3, 9), pad_mode="reflect"):
    """SoundStream.encoder (soundstream.py:519-531): x [b, c_in, T] -> [b, codebook_dim, T/prod(strides)]."""
    x = causal_conv1d(x, st["0.conv.weight"], st["0.conv.bias"], pad_mode=pad_mode)
    for bi, s in enumerate(strides, start=1):
        for ri, d in enumerate(dilations):
            x = residual_unit(sub(st, f"{bi}.{ri}"), x, d, pad_mode)
        # the reference's EncoderBlock builds its strided conv without pad_mode: always reflect
        x = causal_conv1d(x, st[f"{bi}.3.conv.weight"], st[f"{bi}.3.conv.bias"], stride=s)
    last = len(strides) + 1
    return causal_conv1d(x, st[f"{last}.conv.weight"], st[f"{last}.conv.bias"], pad_mode=pad_mode)


def decoder(st, x, strides=(2, 4, 5, 8), dilations=(1, 3, 9), pad_mode="reflect"):
    """SoundStream.decoder (soundstream.py:615-627): x [b, codebook_dim, n] -> [b, c_in, n*prod(strides)]."""
    x = causal_conv1d(x, st["0.conv.weight"], st["0.conv.bias"], pad_mode=pad_mode)
    for bi, s in enumerate(reversed(strides), start=1):
        x = causal_conv_transpose1d(x, st[f"{bi}.0.conv.weight"], st[f"{bi}.0.conv.bias"], s)
        for ri, d in enumerate(dilations, start=1):
            x = residual_unit(sub(st, f"{bi}.{ri}"), x, d, pad_mode)
    last = len(strides) + 1
    return causal_conv1d(x, st[f"{last}.conv.weight"], st[f"{last}.conv.bias"], pad_mode=pad_mode)


def codebooks_of(st, group=0):
    """[q, c, d] fp32 codebooks from rq.rvqs.{g}.layers.{q}._codebook.embed (shape (1,c,d))."""
    qs = sorted({int(k.split(".")[4]) for k in st if k.startswith(f"rq.rvqs.{group}.layers.")})
    return torch.stack([st[f"rq.rvqs.{group}.layers.{q}._codebook.embed"][0] for q in qs])


def rvq_encode(x, codebooks):
    """ResidualVQ eval forward: x [N, d], codebooks [q, c, d] -> (quantized [N, d], indices [N, q] int64)."""
    residual = x.float()
    out = torch.zeros_like(residual)
    idxs = []
    for cb in codebooks:
        idx = euclid_nearest(residual, cb)
        quant = cb[idx]
        residual = residual - quant
        out = out + quant
        idxs.append(idx)
    return out, torch.stack(idxs, dim=-1)


def rvq_decode(indices, codebooks):
    """get_output_from_indices: indices [N, q] (-1 = dropped) -> sum_q codebooks[q][idx] [N, d]."""
    out = 0
    for q in range(indices.shape[-1]):
        idx = indices[..., q]
        out = out + codebooks[q][idx.clamp(min=0)].masked_fill((idx < 0)[..., None], 0.0)
    return out


def rvq_margin(x, codebooks):
    """smallest gap between best and second-best distance over all stages (for bit-exactness claims)."""
    residual = x.float()
    worst = torch.full((x.shape[0],), float("inf"))
    for cb in codebooks:
        d = torch.cdist(residual.double(), cb.double())
        top2 = d.topk(2, dim=-1, largest=False)
        worst = torch.minimum(worst, (top2.values[:, 1] - top2.values[:, 0]).float())
        residual = residual - cb[top2.indices[:, 0]]
    return worst


def soundstream_tokenize(st, wave, strides=(2, 4, 5, 8), groups=1):
    """SoundStream.forward(..., return_encoded=True) without local attention (soundstream.py:802-852).

    wave [b, T] -> (quantized [b, n, D], indices [b, n, g*q] int64)
    """
    x = encoder(sub(st, "encoder"), wave[:, None, :], strides).transpose(1, 2)  # b n c
    b, n, D = x.shape
    outs, idxs = [], []
    for g, chunk in enumerate(x.chunk(groups, dim=-1)):
        o, i = rvq_encode(chunk.reshape(b * n, -1), codebooks_of(st, g))
        outs.append(o.reshape(b, n, -1))
        idxs.append(i.reshape(b, n, -1))
    return torch.cat(outs, -1), torch.cat(idxs, -1)


def soundstream_decode_indices(st, indices, strides=(2, 4, 5, 8), groups=1):
    """decode_from_codebook_indices (soundstream.py:691-709): indices [b, n, g*q] -> wave [b, 1, T]."""
    b, n, gq = indices.shape
    q = gq // groups
    parts = [rvq_decode(indices[..., g * q:(g + 1) * q].reshape(b * n, q), codebooks_of(st, g)).reshape(b, n, -1)
             for g in range(groups)]
    x = torch.cat(parts, -1).transpose(1, 2)
    return decoder(sub(st, "decoder"), x, strides)
