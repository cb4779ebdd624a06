"""CPU restatement of fairseq's vq-wav2vec as called by the reference's FairseqVQWav2Vec (vq_wav2vec.py:75-76):
`model.feature_extractor(wav)` (wav2vec's ConvFeatureExtractionModel), then `model.vector_quantizer.forward_idx(...)`
(KmeansVectorQuantizer).

Pure torch on fairseq-layout state dicts, any dtype (tests run it in fp64).  It restates fairseq's published source
(models/wav2vec/wav2vec.py, modules/kmeans_vector_quantizer.py, modules/fp32_group_norm.py); fairseq is not
installable offline, so parity with fairseq itself is unpinned.  The points it restates, one by one:

1. Input: x = wav.unsqueeze(1), shape [B, 1, T].
2. Conv blocks: each is Sequential(Conv1d(n_in, n_out, k, stride, bias=False), Dropout, Fp32GroupNorm(1, n_out,
   affine=not non_affine_group_norm), activation), the activation ReLU or GELU (exact erf) from `activation`.
   Keys: feature_extractor.conv_layers.{i}.0.weight, plus .2.weight / .2.bias when the norm is affine.
   GroupNorm(1, C) takes one mean and one biased variance per clip over all C x T, eps 1e-5, then the per-channel
   affine.
3. Skip connections (skip_connections_feat): after a block whose output has as many channels as its input,
   x = (x + residual[..., ::r_tsz // tsz][..., :tsz]) * sqrt(residual_scale), residual being the previous block's
   output after its own skip.  The subsampling step r_tsz // tsz is not the stride on short clips (k 8, s 4,
   r_tsz 12: tsz 2, step 6).
4. Log compression (log_compression): x = log(|x| + 1) after the last block.
5. k-means quantizer, KmeansVectorQuantizer(dim, num_vars, groups, combine_groups, vq_dim):
   projection = Sequential(Conv1d(dim, dim, 1, groups=groups, bias=False), Fp32GroupNorm(groups, dim)), the
   GroupNorm affine; ze is viewed as [B, T, G, var_dim] with var_dim = vq_dim // groups (so only vq_dim == dim runs);
   embedding has shape [num_vars, 1 if combine_groups else G, var_dim], expanded across the groups when combined;
   idx[b, t, g] = argmin_v ||ze[b, t, g] - e[v, g]||_2, the lowest index on ties.
"""
from __future__ import annotations

import argparse
import enum
import math
import sys
import types

import torch
import torch.nn.functional as F

from .hubert import parse_conv_layers

EPS = 1e-5
EMBEDDING = "vector_quantizer.embedding"
PROJ = "vector_quantizer.projection."


def conv_layers(arch):
    return parse_conv_layers(arch["conv_feature_layers"])


def features(st, arch, wave):
    """ConvFeatureExtractionModel (points 1-4): wave [B, T] -> [B, T', C] (channels last)"""
    x = wave[:, None, :]  # 1
    for i, (_, _, s) in enumerate(conv_layers(arch)):
        p = f"feature_extractor.conv_layers.{i}."
        residual = x
        x = F.conv1d(x, st[p + "0.weight"], stride=s)  # 2: no bias; Dropout is the identity at inference
        x = F.group_norm(x, 1, st.get(p + "2.weight"), st.get(p + "2.bias"), EPS)
        x = F.gelu(x) if arch["activation"] == "gelu" else F.relu(x)
        if arch["skip_connections_feat"] and x.shape[1] == residual.shape[1]:  # 3
            tsz, r_tsz = x.shape[2], residual.shape[2]
            x = (x + residual[..., ::r_tsz // tsz][..., :tsz]) * math.sqrt(arch["residual_scale"])
    if arch["log_compression"]:  # 4
        x = (x.abs() + 1).log()
    return x.transpose(1, 2)


def project(st, x):
    """the quantizer's projection (point 5): features [B, T, C] -> ze [B, T, G, var_dim]"""
    w = st[PROJ + "0.weight"]
    C = w.shape[0]
    G = C // w.shape[1]
    y = F.conv1d(x.transpose(1, 2), w, groups=G)
    y = F.group_norm(y, G, st[PROJ + "1.weight"], st[PROJ + "1.bias"], EPS)
    B, _, T = y.shape
    return y.view(B, G, C // G, T).permute(0, 3, 1, 2)


def codewords(st, groups):
    """embedding expanded to [num_vars, G, var_dim] (combine_groups shares one codebook across the groups)"""
    e = st[EMBEDDING]
    return e.expand(e.shape[0], groups, e.shape[2])


def distances(ze, e):
    """||ze[b, t, g] - e[v, g]||_2 -> [B, T, G, V], by direct differences (no |x|^2 - 2 x.e + |e|^2 expansion)"""
    B, T, G, vd = ze.shape
    d = [torch.cdist(ze[:, :, g].reshape(1, B * T, vd), e[:, g][None].to(ze.dtype),
                     compute_mode="donot_use_mm_for_euclid_dist")[0] for g in range(G)]
    return torch.stack(d, dim=1).view(B, T, G, -1)


def ids(ze, e):
    """idx [B, T, G] int64: the nearest codeword per group, the lowest index on ties"""
    return distances(ze, e).argmin(-1)


def margins(ze, e):
    """distance gap between the nearest and the runner-up codeword, per frame and group [B, T, G]"""
    two = distances(ze, e).topk(2, dim=-1, largest=False).values
    return two[..., 1] - two[..., 0]


def block_diagonal(w):
    """grouped 1x1 conv weight [C, C / G, 1] -> the dense [C, C] weight it applies (zeros off the diagonal blocks)"""
    C, Cg, _ = w.shape
    return torch.block_diag(*w[:, :, 0].view(C // Cg, Cg, Cg))


def random_state(arch, *, seed, groups, num_vars, combine_groups, affine=True):
    """seeded random weights in the fairseq checkpoint layout (a few unused tensors of the wav2vec model included),
    scaled so activations keep unit size"""
    g = torch.Generator().manual_seed(seed)

    def rn(*shape, scale):
        return torch.randn(*shape, generator=g) * scale

    st, cin = {}, 1
    for i, (c, k, _) in enumerate(conv_layers(arch)):
        p = f"feature_extractor.conv_layers.{i}."
        st[p + "0.weight"] = rn(c, cin, k, scale=(cin * k) ** -0.5)
        if affine:
            st[p + "2.weight"] = 1 + rn(c, scale=0.1)
            st[p + "2.bias"] = rn(c, scale=0.1)
        cin = c
    vd = cin // groups
    st[PROJ + "0.weight"] = rn(cin, vd, 1, scale=vd ** -0.5)
    st[PROJ + "1.weight"] = 1 + rn(cin, scale=0.1)
    st[PROJ + "1.bias"] = rn(cin, scale=0.1)
    st[EMBEDDING] = rn(num_vars, 1 if combine_groups else groups, vd, scale=1.0)
    st["feature_aggregator.conv_layers.0.0.weight"] = rn(cin, cin, 2, scale=(2 * cin) ** -0.5)
    st["wav2vec_predictions.project_to_steps.weight"] = rn(cin, cin, 1, 2, scale=cin ** -0.5)
    return st


PUBLISHED = dict(conv_feature_layers="[(512, 10, 5), (512, 8, 4), (512, 4, 2), (512, 4, 2), (512, 4, 2), "
                                     "(512, 1, 1), (512, 1, 1), (512, 1, 1)]",
                 activation="relu", log_compression=True, skip_connections_feat=True, residual_scale=0.5,
                 vq_type="kmeans", vq_vars=320, vq_groups=2, combine_groups=False, vq_dim=0,
                 non_affine_group_norm=False)


# ---- checkpoints in fairseq's formats, for tests ---------------------------------------------------------------------
FAKE_ENUM_MODULE = "fairseq.dataclass.utils"


def write_checkpoint(path, st, arch, form="cfg"):
    """a fairseq-layout checkpoint: form "cfg" stores cfg = {"model": arch} with `activation` as a member of a fake
    fairseq ChoiceEnum (the fake module is removed again afterwards), form "args" stores arch as an
    argparse.Namespace"""
    if form == "args":
        torch.save({"model": st, "args": argparse.Namespace(**arch)}, path)
        return
    added = [n for n in ("fairseq", "fairseq.dataclass", FAKE_ENUM_MODULE) if n not in sys.modules]
    for n in added:
        sys.modules[n] = types.ModuleType(n)
    try:
        choice = enum.Enum("Choices", {"relu": "relu", "gelu": "gelu"}, module=FAKE_ENUM_MODULE)
        sys.modules[FAKE_ENUM_MODULE].Choices = choice
        model = dict(arch)
        if "activation" in model and model["activation"] in ("relu", "gelu"):
            model["activation"] = choice(model["activation"])
        torch.save({"model": st, "cfg": {"model": model}}, path)
    finally:
        for n in added:
            sys.modules.pop(n, None)
