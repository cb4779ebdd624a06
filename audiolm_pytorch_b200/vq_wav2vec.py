"""FairseqVQWav2Vec (vq_wav2vec.py:19-81): semantic tokens from raw audio - vq-wav2vec's conv features, then the
nearest codeword of its k-means quantizer in every group - on the sm_90a kernels, loading fairseq checkpoints without
fairseq (through hubert.load_checkpoint).

The network is fairseq's wav2vec `feature_extractor` followed by `vector_quantizer.forward_idx`:
  1. conv blocks: Conv1d without bias, GroupNorm(1, C) over the whole clip (affine unless non_affine_group_norm),
     ReLU or GELU; with skip_connections_feat, a block whose input and output widths agree adds its input subsampled
     by r_tsz // tsz and scales by sqrt(residual_scale); with log_compression, log(|x| + 1) after the last block;
  2. the quantizer's grouped 1x1 projection and GroupNorm(G, C);
  3. per group, the nearest codeword of `embedding` (one codebook shared by the groups with combine_groups).
Precision: conv 0 runs on fp32 CUDA cores (ops.hubert_conv0); every other conv and the projection run on the wgmma
GEMM in split bf16 (x_hi w_hi + x_lo w_hi + x_hi w_lo, fp32 accumulation); norms, activations, skips and the log are
fp32 (csrc/vq_wav2vec.cu); the codeword search is the RVQ stage of rvq_tc.cu (ops.nearest_centroid).  There is no CPU
path: CPU inputs raise AlmError.

Envelope (NotImplementedError at construction otherwise): conv widths and var_dim multiples of 8; vq_dim == dim (the
only case fairseq's quantizer runs); activation "relu" or "gelu".  The published vq-wav2vec k-means model (eight
512-wide convs, 2 groups of 320 codewords) is inside it.  A clip must be at least one frame long (465 samples for the
published extractor).
"""
from __future__ import annotations

import argparse
import math
from pathlib import Path

import torch
from torch import nn

from . import _lib, ops
from .hubert import (_conv_flops, _Node, _plain, _register, curtail_to_multiple, getattr_path, load_checkpoint,
                     parse_conv_layers, receptive_field, resample_curtailed)
from .soundstream import SoundStream

f32 = torch.float32

ARCH_KEYS = ("conv_feature_layers", "activation", "log_compression", "skip_connections_feat", "residual_scale",
             "vq_type")
OPTIONAL_KEYS = ("vq_vars", "vq_groups", "combine_groups", "vq_dim", "non_affine_group_norm")
INVALID = "the vq wav2vec model does not seem to be valid"  # the reference's assertion message (vq_wav2vec.py:47)
EMBEDDING = "vector_quantizer.embedding"
PROJ = "vector_quantizer.projection."


def read_arch(ckpt):
    """the architecture fields of a fairseq wav2vec checkpoint, from cfg["model"] or, in older checkpoints, args.
    No field has a default: fairseq's argparse and dataclass defaults disagree (log_compression)."""
    src = None
    cfg = _plain(ckpt.get("cfg")) if isinstance(ckpt, dict) else None
    if isinstance(cfg, dict) and isinstance(cfg.get("model"), dict):
        src = cfg["model"]
    elif isinstance(ckpt, dict) and ckpt.get("args") is not None:
        args = ckpt["args"]
        src = vars(args) if isinstance(args, argparse.Namespace) else _plain(args)
    if not isinstance(src, dict):
        raise ValueError("cannot read the vq-wav2vec architecture: the checkpoint has neither a cfg['model'] dict nor "
                         "args")
    missing = [k for k in ARCH_KEYS if k not in src]
    if missing:
        raise ValueError(f"cannot read the vq-wav2vec architecture: the checkpoint's config lacks {', '.join(missing)}")
    arch = {k: _plain(src[k]) for k in ARCH_KEYS + OPTIONAL_KEYS if k in src}
    arch["activation"] = str(arch["activation"])
    arch["vq_type"] = str(arch["vq_type"])
    return arch


def read_geometry(arch, st):
    """what the tensors determine: per conv (width, kernel, stride) and whether its norm is affine, the quantizer's
    groups, num_vars, var_dim and combine_groups.  ValueError where the tensors and the config disagree."""
    layers = parse_conv_layers(arch["conv_feature_layers"])
    n = sum(1 for k in st if k.startswith("feature_extractor.conv_layers.") and k.endswith(".0.weight"))
    if n != len(layers):
        raise ValueError(f"conv_feature_layers lists {len(layers)} convs, the checkpoint holds {n}")
    cin, affine = 1, []
    for i, (c, k, _) in enumerate(layers):
        w = st[f"feature_extractor.conv_layers.{i}.0.weight"]
        if tuple(w.shape) != (c, cin, k):
            raise ValueError(f"conv {i}: weight shape {tuple(w.shape)}, conv_feature_layers says {(c, cin, k)}")
        affine.append(f"feature_extractor.conv_layers.{i}.2.weight" in st)
        cin = c
    if "non_affine_group_norm" in arch and any(a == bool(arch["non_affine_group_norm"]) for a in affine):
        raise ValueError(f"non_affine_group_norm={arch['non_affine_group_norm']} disagrees with the norms' tensors")
    for key in (PROJ + "0.weight", PROJ + "1.weight", PROJ + "1.bias"):
        if key not in st:
            raise ValueError(f"the checkpoint lacks {key}")
    w, e = st[PROJ + "0.weight"], st[EMBEDDING]
    if w.dim() != 3 or w.shape[0] != cin or w.shape[2] != 1 or cin % w.shape[1]:
        raise ValueError(f"vector_quantizer.projection.0.weight has shape {tuple(w.shape)}; the features are {cin} wide")
    groups = cin // w.shape[1]
    if e.dim() != 3 or e.shape[1] not in (1, groups):
        raise ValueError(f"vector_quantizer.embedding has shape {tuple(e.shape)}; the projection has {groups} groups")
    geo = dict(layers=layers, affine=affine, dim=cin, groups=groups, num_vars=e.shape[0], var_dim=e.shape[2],
               combine_groups=e.shape[1] == 1)
    for key, name in (("vq_groups", "groups"), ("vq_vars", "num_vars")):
        if key in arch and int(arch[key]) != geo[name]:
            raise ValueError(f"{key}={arch[key]} disagrees with the tensors ({name} {geo[name]})")
    if "combine_groups" in arch and groups > 1 and bool(arch["combine_groups"]) != geo["combine_groups"]:
        raise ValueError(f"combine_groups={arch['combine_groups']} disagrees with vector_quantizer.embedding "
                         f"{tuple(e.shape)}")
    return geo


def check_envelope(arch, geo):
    """NotImplementedError naming the first field outside what the kernels are built for"""
    if arch["activation"] not in ("relu", "gelu"):
        raise NotImplementedError(f"activation {arch['activation']!r} (built: 'relu', 'gelu')")
    for c, k, s in geo["layers"]:
        if c % 8 or k < 1 or s < 1:
            raise NotImplementedError(f"conv_feature_layers ({c}, {k}, {s}): widths must be multiples of 8")
    vq_dim = int(arch.get("vq_dim") or 0) or geo["dim"]
    if vq_dim != geo["dim"] or geo["var_dim"] * geo["groups"] != geo["dim"]:
        raise NotImplementedError(f"vq_dim {vq_dim} with var_dim {geo['var_dim']} x {geo['groups']} groups: only "
                                  f"vq_dim == dim ({geo['dim']}) is built")
    if geo["var_dim"] % 8:
        raise NotImplementedError(f"var_dim {geo['var_dim']} must be a multiple of 8")


def block_diagonal_weight(w):
    """grouped 1x1 conv weight [C, C / G, 1] -> the dense block-diagonal [C, C] weight of the same map, so the grouped
    projection is one GEMM (its zero blocks add exact zeros)"""
    C, Cg, _ = w.shape
    return torch.block_diag(*w[:, :, 0].reshape(C // Cg, Cg, Cg))


class FairseqVQWav2Vec(nn.Module):
    """checkpoint as published at https://github.com/facebookresearch/fairseq/blob/main/examples/wav2vec/README.md
    (vq-wav2vec_kmeans.pt, or your own k-means vq-wav2vec); see the module docstring for what runs where"""

    def __init__(self, checkpoint_path, target_sample_hz=24000, seq_len_multiple_of=None):
        super().__init__()
        self.target_sample_hz = target_sample_hz
        self.seq_len_multiple_of = seq_len_multiple_of
        assert Path(checkpoint_path).exists(), f"path {checkpoint_path} does not exist"
        ckpt = load_checkpoint(checkpoint_path)
        self.arch = read_arch(ckpt)
        st = ckpt["model"]
        if self.arch["vq_type"] != "kmeans" or EMBEDDING not in st:
            raise AssertionError(INVALID)
        self.geo = read_geometry(self.arch, st)
        check_envelope(self.arch, self.geo)
        self.model = _Node()
        for k, v in st.items():
            _register(self.model, k, v)

    @property
    def groups(self):
        return self.geo["groups"]

    @property
    def codebook_size(self):
        return self.geo["num_vars"]

    @property
    def downsample_factor(self):
        return 80  # the reference's constant (vq_wav2vec.py:53-56); the published extractor's hop is 160

    # ---- weights in the GEMM layouts, rebuilt when a tensor changes -------------------------------------------------
    def _packed(self):
        st = dict(self.model.state_dict(keep_vars=True))
        return SoundStream._cached(self, "_packed_weights", list(st.values()), lambda: self._pack(st))

    def _pack(self, st):
        P = {}
        for i, (_, k, s) in enumerate(self.geo["layers"]):
            w = st[f"feature_extractor.conv_layers.{i}.0.weight"].float()
            if i == 0:
                P["conv0"] = w.contiguous()
            elif k == 1 and s == 1:
                P[f"conv{i}"] = ops.pack_split_weight(w[:, :, 0].contiguous())
            else:
                P[f"conv{i}"] = ops.pack_split_conv_weight(w)
        P["proj"] = ops.pack_split_weight(block_diagonal_weight(st[PROJ + "0.weight"].float()).contiguous())
        e = st[EMBEDDING].float()
        if self.geo["combine_groups"]:
            P["codes"] = ops.rvq_pack_codebooks(e[:, 0][None])
        else:
            cb, packed, e2 = ops.rvq_pack_codebooks(e.permute(1, 0, 2))
            P["codes"] = [(cb[g:g + 1], packed[g:g + 1], e2[g:g + 1]) for g in range(self.groups)]
        return P

    def _vec(self, name):
        t = getattr_path(self.model, name)
        return t if t.dtype == f32 else t.float()

    # ---- forward -----------------------------------------------------------------------------------------------------
    def _features(self, wave):
        """fp32 wave [B, T] on the GPU -> (features fp32 [B, n, C], the same in the split layout)"""
        a, P, layers = self.arch, self._packed(), self.geo["layers"]
        if wave.shape[-1] < receptive_field(layers):
            raise ValueError(f"a clip of {wave.shape[-1]} samples is shorter than one frame "
                             f"({receptive_field(layers)} samples)")
        wave = wave.to(f32).contiguous()
        B = wave.shape[0]
        skip, act = bool(a["skip_connections_feat"]), a["activation"]
        scale = math.sqrt(float(a["residual_scale"]))
        n = len(layers)
        with ops._timed("w2v_conv_extractor", _conv_flops(layers, B, wave.shape[-1])):
            x, xs, c_in = None, None, 1
            for i, (c, k, s) in enumerate(layers):
                if i == 0:
                    y = ops.hubert_conv0(wave, P["conv0"], None, stride=s)
                elif k == 1 and s == 1:
                    y = ops.split_gemm(xs, P[f"conv{i}"], cls="w2v_conv_gemm")
                else:
                    y = ops.hubert_conv_gemm(xs, P[f"conv{i}"], None, kernel_size=k, stride=s, cls="w2v_conv_gemm")
                norm = f"feature_extractor.conv_layers.{i}.2"
                aff = self.geo["affine"][i]
                res = x if skip and c == c_in else None
                last = i == n - 1
                x, xs = ops.w2v_norm_act(y, ops.w2v_group_stats(y), gamma=self._vec(norm + ".weight") if aff else None,
                                         beta=self._vec(norm + ".bias") if aff else None, act=act, residual=res,
                                         step=res.shape[1] // y.shape[1] if res is not None else 1,
                                         residual_scale=scale, log_compress=last and bool(a["log_compression"]),
                                         want_out=last or (skip and layers[i + 1][0] == c))
                c_in = c
        return x, xs

    def extract_features(self, wave):
        """fp32 wave [B, T] on the GPU -> the feature extractor's output fp32 [B, n, C] (channels last)"""
        return self._features(wave)[0]

    def _ze(self, xs):
        B, n, C3 = xs.shape
        C, G = C3 // 3, self.groups
        with ops._timed("w2v_projection", 2.0 * B * n * C * C / G):
            y = ops.split_gemm(xs, self._packed()["proj"], cls="w2v_proj_gemm")
            ze, _ = ops.w2v_norm_act(y, ops.w2v_group_stats(y, G), gamma=self._vec(PROJ + "1.weight"),
                                     beta=self._vec(PROJ + "1.bias"), want_out=True, want_split=False)
        return ze.view(B, n, G, C // G)

    def quantizer_input(self, wave):
        """ze fp32 [B, n, G, var_dim]: the projected, group-normalised features the codeword search runs on"""
        return self._ze(self._features(wave)[1])

    def assign(self, ze):
        """nearest codeword of every frame and group: ze fp32 [B, n, G, var_dim] -> int64 [B, n, G]"""
        B, n, G, vd = ze.shape
        codes = self._packed()["codes"]
        with ops._timed("w2v_assignment", 2.0 * B * n * G * self.codebook_size * vd):
            if self.geo["combine_groups"]:
                return ops.nearest_centroid(ze.reshape(B * n * G, vd), codes).view(B, n, G)
            rows = ze.reshape(B * n, G * vd)
            return torch.stack([ops.nearest_centroid(rows[:, g * vd:(g + 1) * vd], codes[g]) for g in range(G)],
                               dim=-1).view(B, n, G)

    @torch.inference_mode()
    def forward(self, wav_input, flatten=True, input_sample_hz=None):
        if not wav_input.is_cuda:
            raise _lib.AlmError("FairseqVQWav2Vec runs on the GPU only (no CPU fallback); move the module and the "
                                "wave to a CUDA device")
        wav_input = resample_curtailed(wav_input, input_sample_hz, self.target_sample_hz, self.seq_len_multiple_of)
        if self.seq_len_multiple_of is not None:
            wav_input = curtail_to_multiple(wav_input, self.seq_len_multiple_of)
        idx = self.assign(self.quantizer_input(wav_input))
        if not flatten:
            return idx
        return idx.reshape(idx.shape[0], -1)

