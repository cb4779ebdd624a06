"""SoundStream codec inference path on libalm_b200 (sm_90a): causal conv encoder -> residual quantizer -> decoder.

Drop-in surface of /root/reference/audiolm_pytorch/soundstream.py:314-395, 451-866 for the calls the AudioLM
hot path makes: `forward(x, return_encoded=True | return_codes_only=True | return_recons_only=True)`,
`tokenize`, `decode_from_codebook_indices`, `decode`, with the reference's constructor kwargs and
state_dict keys for `encoder.*`, `decoder.*`, `rq.*` (including the gate-loop layers of `use_gate_loop_layers`).  The quantizer is the residual VQ
(Euclidean or cosine-similarity codebooks, optionally behind `codebook_dim` projections), residual FSQ
(`use_finite_scalar_quantizer`) or residual LFQ (`use_lookup_free_quantizer`), eval path only.  GAN / mel training
losses, quantizer training and FiLM denoising are outside this build; the local-attention bottleneck lives in
local_attn.py.
"""
from __future__ import annotations

import functools
import math
import pickle
from itertools import cycle
from pathlib import Path

import torch
from torch import nn

from . import ops
from .local_attn import LocalTransformer

f32 = torch.float32


FUSE_RESIDUAL_UNITS = True  # False: conv7 + conv1 as two launches (A/B tests)
RVQ_ON_TENSOR_CORES = True      # False: fp32 CUDA-core search kernel (A/B tests)
ENCODER_ON_TENSOR_CORES = True  # False: fp32 CUDA-core conv kernels for the whole encoder (A/B tests)
GATE_LOOP_TC_CHANNELS = (32, 64, 128, 256, 512)  # widths alm_codec_gate_loop_tc takes


def exists(v):
    return v is not None


def curtail_window(total, mult, from_left=False):
    """(start, count) of the samples the reference's curtail_to_multiple (utils.py:8-12) keeps of `total`.  From the
    left it slices [-keep:], which keeps everything when keep is 0."""
    keep = total // mult * mult
    if from_left and keep:
        return total - keep, keep
    return 0, total if from_left else keep


class CausalConv1d(nn.Module):
    """soundstream.py:332-345; parameters live in `.conv` (nn.Conv1d) for state_dict compatibility."""

    def __init__(self, chan_in, chan_out, kernel_size, pad_mode="reflect", **kwargs):
        super().__init__()
        self.dilation = kwargs.get("dilation", 1)
        self.stride = kwargs.get("stride", 1)
        self.pad_mode = pad_mode
        self.causal_padding = self.dilation * (kernel_size - 1) + (1 - self.stride)
        self.conv = nn.Conv1d(chan_in, chan_out, kernel_size, **kwargs)
        self._packed = (None, None)  # (weight version key, [Cin, K, Cout] copy for the register-tiled kernel)

    def _packed_weight(self):
        w = self.conv.weight
        key = (w.data_ptr(), w._version, w.device)
        if self._packed[0] != key:
            with torch.no_grad():
                self._packed = (key, w.detach().permute(1, 2, 0).contiguous())
        return self._packed[1]

    def forward(self, x, elu=False, residual=None):
        k = self.conv.kernel_size[0]
        wp = self._packed_weight() if (k, self.stride, self.dilation) in ops.CONV_TILED_SHAPES else None
        return ops.causal_conv1d(x, self.conv.weight, self.conv.bias, stride=self.stride, dilation=self.dilation,
                                 pad_mode=self.pad_mode, elu=elu, residual=residual, weight_packed=wp)


class CausalConvTranspose1d(nn.Module):
    """soundstream.py:347-360."""

    def __init__(self, chan_in, chan_out, kernel_size, stride, **kwargs):
        super().__init__()
        assert kernel_size == 2 * stride
        self.upsample_factor = stride
        self.conv = nn.ConvTranspose1d(chan_in, chan_out, kernel_size, stride, **kwargs)

    def forward(self, x):
        return ops.causal_conv_transpose1d(x, self.conv.weight, self.conv.bias, stride=self.upsample_factor)


class SqueezeExcite(nn.Module):
    """soundstream.py:145-169: y * sigmoid(W2 SiLU(W1 m + b1) + b2), m the cumulative mean over CHANNELS (the reference
    cumsums dim -2 of [B, C, T]); keys `net.0.*` [Ci, C, 1] and `net.2.*` [C, Ci, 1], Ci = max(8, C // 4).  Applied by
    ResidualUnit, which adds the skip input in the same kernel."""

    def __init__(self, dim, reduction_factor=4, dim_minimum=8):
        super().__init__()
        inner = max(dim_minimum, dim // reduction_factor)
        self.net = nn.Sequential(nn.Conv1d(dim, inner, 1), nn.SiLU(), nn.Conv1d(inner, dim, 1), nn.Sigmoid())

    def folded_weight(self):
        """[Ci, C] first-conv weight with the cumulative mean folded in (ops.se_fold_weight), cached per weight version"""
        return SoundStream._cached(self, "_folded", [self.net[0].weight], lambda: ops.se_fold_weight(self.net[0].weight))

    def residual(self, y, x):
        """x + SqueezeExcite(y) on fp32 [B, C, T] (csrc/codec.cu)"""
        return ops.codec_se_fp32(y, x, self.folded_weight(), self.net[0].bias, self.net[2].weight, self.net[2].bias)


class _RUBody(nn.Module):
    """holds the two convs under the reference's Sequential indices 0 and 2 (1, 3 are ELUs) and, with squeeze_excite,
    the SqueezeExcite under index 4."""

    def __init__(self, chan_in, chan_out, dilation, kernel_size, pad_mode, squeeze_excite=False):
        super().__init__()
        self.add_module("0", CausalConv1d(chan_in, chan_out, kernel_size, dilation=dilation, pad_mode=pad_mode))
        self.add_module("2", CausalConv1d(chan_out, chan_out, 1, pad_mode=pad_mode))
        if squeeze_excite:
            self.add_module("4", SqueezeExcite(chan_out))


def _se_of(ru):
    return getattr(ru.fn, "4", None)


class ResidualUnit(nn.Module):
    """x + SE(ELU(conv1(ELU(conv7_dil(x))))) (soundstream.py:362-369), SE = identity unless squeeze_excite; keys
    `fn.{0,2}.conv.*` (and `fn.4.net.{0,2}.*`).  Two fused launches without SE, three with it."""

    def __init__(self, chan_in, chan_out, dilation, kernel_size=7, squeeze_excite=False, pad_mode="reflect"):
        super().__init__()
        self.fn = _RUBody(chan_in, chan_out, dilation, kernel_size, pad_mode, squeeze_excite)

    def forward(self, x):
        c7, c1 = getattr(self.fn, "0"), getattr(self.fn, "2")
        se = _se_of(self)
        if se is not None:
            return se.residual(c1(c7(x, elu=True), elu=True), x)
        C = x.shape[1]
        if (FUSE_RESIDUAL_UNITS and C in ops.RU_FUSED_CHANNELS and c7.dilation in ops.RU_FUSED_DILATIONS
                and c7.conv.kernel_size[0] == 7 and c1.conv.kernel_size[0] == 1 and c7.conv.out_channels == C
                and x.shape[-1] > 6 * c7.dilation):
            return ops.residual_unit(x, c7._packed_weight(), c7.conv.bias, c1._packed_weight(), c1.conv.bias,
                                     dilation=c7.dilation, pad_mode=c7.pad_mode)
        h = c7(x, elu=True)
        return c1(h, elu=True, residual=x)


def EncoderBlock(chan_in, chan_out, stride, cycle_dilations=(1, 3, 9), squeeze_excite=False, pad_mode="reflect"):
    it = cycle(cycle_dilations)
    return nn.Sequential(*[ResidualUnit(chan_in, chan_in, next(it), squeeze_excite=squeeze_excite, pad_mode=pad_mode)
                           for _ in range(3)],
                         CausalConv1d(chan_in, chan_out, 2 * stride, stride=stride))


def DecoderBlock(chan_in, chan_out, stride, cycle_dilations=(1, 3, 9), squeeze_excite=False, pad_mode="reflect"):
    it = cycle(cycle_dilations)
    return nn.Sequential(CausalConvTranspose1d(chan_in, chan_out, 2 * stride, stride=stride),
                         *[ResidualUnit(chan_out, chan_out, next(it), squeeze_excite=squeeze_excite, pad_mode=pad_mode)
                           for _ in range(3)])


class _RMSNorm(nn.Module):
    """gateloop-transformer's RMSNorm: F.normalize(x, dim=-1) * sqrt(dim) * gamma; key `gamma` [dim]."""

    def __init__(self, dim):
        super().__init__()
        self.gamma = nn.Parameter(torch.ones(dim))


class GateLoop(nn.Module):
    """SimpleGateLoopLayer(dim) of gateloop-transformer as the reference builds it (soundstream.py:29, 524-525, 620-621),
    eval path: on u_t = x[:, :, t],  [q; kv; a]_t = W RMSNorm(u_t),  h_t = sigmoid(a_t) * h_{t-1} + kv_t,  out_t = q_t * h_t.
    Keys `norm.gamma` [C] and `to_qkva.0.weight` [3C, C] (rows q, kv, a).  Runs only inside Residual(ChannelTranspose(.)),
    whose two skip adds the kernels fuse: the block computes 2 x + q * h."""

    def __init__(self, dim):
        super().__init__()
        self.norm = _RMSNorm(dim)
        self.to_qkva = nn.Sequential(nn.Linear(dim, 3 * dim, bias=False))

    def folded_weight(self):
        """[3C, C] projection with sqrt(C) * gamma folded in (ops.gate_loop_fold_weight), cached per weight version"""
        w = self.to_qkva[0].weight
        return SoundStream._cached(self, "_folded", [w, self.norm.gamma],
                                   lambda: ops.gate_loop_fold_weight(w, self.norm.gamma))

    def block_fp32(self, x):
        """Residual(ChannelTranspose(self)) on fp32 [B, C, T] (csrc/codec_gate_loop.cu)"""
        return ops.codec_gate_loop_fp32(x.to(f32), self.folded_weight())

    def block_tc(self, h):
        """Residual(ChannelTranspose(self)) on C8S activations (P = 1), projection on the tensor cores"""
        w = self.to_qkva[0].weight
        units = SoundStream._cached(self, "_tc_units", [w, self.norm.gamma],
                                    lambda: ops.pack_gate_loop_weights(ops.gate_loop_fold_weight(w, self.norm.gamma)))
        return ops.codec_gate_loop_tc(h, units)


class ChannelTranspose(nn.Module):
    """soundstream.py:322-330 around a GateLoop: holds it under `fn`; its skip add runs in the gate-loop kernel."""

    def __init__(self, fn):
        super().__init__()
        self.fn = fn


class Residual(nn.Module):
    """soundstream.py:314-320 around ChannelTranspose(GateLoop): keys `fn.fn.*`.  With ChannelTranspose's own skip add,
    x enters the output twice (a reference quirk kept on purpose): Residual(ChannelTranspose(g))(x) = 2 x + g(x)."""

    def __init__(self, fn):
        super().__init__()
        self.fn = fn

    def forward(self, x):
        return self.fn.fn.block_fp32(x)


def _gate_loop_of(m):
    return m.fn.fn if isinstance(m, Residual) else None


# ---- residual VQ containers (state_dict keys of vector-quantize-pytorch) ---------------------------
class _Codebook(nn.Module):
    def __init__(self, dim, codebook_size):
        super().__init__()
        self.register_buffer("initted", torch.Tensor([False]))
        self.register_buffer("cluster_size", torch.ones(1, codebook_size))
        self.register_buffer("embed_avg", torch.zeros(1, codebook_size, dim))
        self.register_buffer("embed", torch.zeros(1, codebook_size, dim))


class _VQLayer(nn.Module):
    def __init__(self, dim, codebook_size):
        super().__init__()
        self._codebook = _Codebook(dim, codebook_size)


# VectorQuantize / ResidualVQ kwargs that only shape training (EMA, k-means init, dead-code expiry, losses, sampling,
# gradient estimators, quantize dropout); eval computes the same with or without them
_VQ_TRAINING_KWARGS = {"decay", "eps", "commitment_weight", "kmeans_init", "kmeans_iters", "sync_kmeans",
                       "threshold_ema_dead_code", "stochastic_sample_codes", "sample_codebook_temp", "straight_through",
                       "rotation_trick", "reinmax", "sync_codebook", "ema_update", "learnable_codebook",
                       "commitment_use_cross_entropy_loss"}
_VQ_TRAINING_PREFIXES = ("orthogonal_reg_", "codebook_diversity_", "quantize_dropout")


def _check_vq_kwargs(kwargs):
    unknown = sorted(k for k in kwargs if k not in _VQ_TRAINING_KWARGS and not k.startswith(_VQ_TRAINING_PREFIXES))
    if unknown:
        raise NotImplementedError(f"ResidualVQ: rq_kwargs {unknown} are outside this build")


class ResidualVQ(nn.Module):
    """vector-quantize-pytorch ResidualVQ, eval path: r = project_in(x); per stage the nearest code (Euclidean, or the
    largest cosine similarity with use_cosine_sim) is subtracted from r and added to the output; project_out(output).
    The projections are Linear(dim, codebook_dim) / Linear(codebook_dim, dim) with bias, absent when the widths agree;
    they and the cosine search run on the tensor cores only."""

    def __init__(self, *, dim, num_quantizers, codebook_size, codebook_dim=None, use_cosine_sim=False, **kwargs):
        super().__init__()
        _check_vq_kwargs(kwargs)
        if not isinstance(codebook_size, int):
            raise NotImplementedError(f"ResidualVQ: codebook_size={codebook_size!r} is outside this build (one int)")
        dc = dim if codebook_dim is None else codebook_dim
        self.projected = dc != dim
        if self.projected and (dim % 8 or dc % 8):
            raise NotImplementedError(f"ResidualVQ: projection {dim} -> {dc} is outside this build (dim per group and "
                                      "codebook_dim multiples of 8)")
        self.use_cosine_sim = bool(use_cosine_sim)
        self.codebook_dim = dc
        self.project_in = nn.Linear(dim, dc) if self.projected else nn.Identity()
        self.project_out = nn.Linear(dc, dim) if self.projected else nn.Identity()
        self.layers = nn.ModuleList([_VQLayer(dc, codebook_size) for _ in range(num_quantizers)])

    def codebooks(self):
        return torch.stack([l._codebook.embed[0] for l in self.layers]).to(f32)

    def _projections(self):
        """(w_in packed, b_in, w_out packed, b_out) for ops.split_linear, cached per weight version"""
        mods = (self.project_in, self.project_out)
        params = [p_ for m in mods for p_ in (m.weight, m.bias)]
        return SoundStream._cached(self, "_proj", params, lambda: tuple(
            t for m in mods for t in (ops.pack_split_weight(m.weight.detach()), m.bias.detach().float().contiguous())))

    def _project(self, x, side):
        if not self.projected:
            return x
        w_in, b_in, w_out, b_out = self._projections()
        return ops.split_linear(x, *((w_in, b_in) if side == "in" else (w_out, b_out)))

    def _check_tensor_cores(self):
        if not RVQ_ON_TENSOR_CORES and (self.use_cosine_sim or self.projected):
            raise NotImplementedError("ResidualVQ: cosine-similarity and projected codebooks run on the tensor-core "
                                      "search only (RVQ_ON_TENSOR_CORES = True)")

    def forward(self, x):
        if self.training:
            raise NotImplementedError("RVQ training (EMA / k-means / commitment loss) is outside this build")
        if not all(bool(l._codebook.initted.item()) for l in self.layers):
            raise RuntimeError("codebooks are not initialised (load a checkpoint; k-means init is not built)")
        self._check_tensor_cores()
        b, n, d = x.shape
        flat = self._project(x.reshape(b * n, d).to(f32).contiguous(), "in")
        if RVQ_ON_TENSOR_CORES:   # any width: rvq_encode_tc zero-pads to a multiple of 8
            embeds = [l._codebook.embed for l in self.layers]
            key = tuple((e.data_ptr(), e._version) for e in embeds)
            if self.__dict__.get("_tc_key") != key:
                with torch.inference_mode(False), torch.no_grad():
                    self.__dict__["_tc_pack"] = ops.rvq_pack_codebooks(self.codebooks())
                self.__dict__["_tc_key"] = key
            quant, idx = ops.rvq_encode_tc(flat, self.__dict__["_tc_pack"],
                                           metric="cosine" if self.use_cosine_sim else "euclid")
        else:
            quant, idx = ops.rvq_encode(flat, self.codebooks())
        quant = self._project(quant, "out")
        return quant.view(b, n, d), idx.view(b, n, -1), torch.zeros(1, len(self.layers), device=x.device)

    def get_output_from_indices(self, indices):
        b, n, q = indices.shape
        out = self._project(ops.rvq_decode(indices.reshape(b * n, q), self.codebooks()), "out")
        return out.view(b, n, -1)


class GroupedResidualVQ(nn.Module):
    """channels split into `groups`, one ResidualVQ each (soundstream.py:592-607)."""

    def __init__(self, *, dim, groups=1, **kwargs):
        super().__init__()
        assert dim % groups == 0
        self.groups = groups
        self.rvqs = nn.ModuleList([ResidualVQ(dim=dim // groups, **kwargs) for _ in range(groups)])

    def forward(self, x):
        outs = [rvq(c) for rvq, c in zip(self.rvqs, x.chunk(self.groups, dim=-1))]
        return (torch.cat([o[0] for o in outs], dim=-1), torch.stack([o[1] for o in outs]),
                torch.stack([o[2] for o in outs]))

    def get_output_from_indices(self, indices):  # g b n q
        return torch.cat([rvq.get_output_from_indices(i) for rvq, i in zip(self.rvqs, indices)], dim=-1)


# ---- residual FSQ / LFQ (vector-quantize-pytorch GroupedResidualFSQ / GroupedResidualLFQ, eval path) -----------------
# rq_kwargs that only shape training (quantize dropout, the LFQ losses); anything else changes what eval computes
_SQ_TRAINING_KWARGS = {"quantize_dropout", "quantize_dropout_cutoff_index", "quantize_dropout_multiple_of"}
_LFQ_TRAINING_KWARGS = _SQ_TRAINING_KWARGS | {"entropy_loss_weight", "commitment_loss_weight", "diversity_gamma"}


class _ScalarQuantizerGroup(nn.Module):
    """one group's ResidualFSQ / ResidualLFQ: `project_in` Linear(Dg, dc) and `project_out` Linear(dc, Dg), both
    identities when Dg == dc.  They are its only persistent state."""

    def __init__(self, dim, codebook_dim):
        super().__init__()
        proj = dim != codebook_dim
        self.project_in = nn.Linear(dim, codebook_dim) if proj else nn.Identity()
        self.project_out = nn.Linear(codebook_dim, dim) if proj else nn.Identity()


class _GroupedScalarQuantizer(nn.Module):
    """channels split into `groups`, each r = project_in(x); Q residual per-dimension quantizer stages; project_out.
    All groups and stages run in one launch (ops.sq_encode, csrc/scalar_quant.cu)."""

    mode = None
    index_dtype = None

    def __init__(self, *, dim, groups, num_quantizers, codebook_dim, constants, kwargs, allowed_kwargs):
        super().__init__()
        unknown = sorted(set(kwargs) - allowed_kwargs)
        if unknown:
            raise NotImplementedError(f"{type(self).__name__}: rq_kwargs {unknown} are outside this build")
        if groups not in (1, 2, 4) or dim % groups:
            raise NotImplementedError(f"{type(self).__name__}: groups={groups} with dim={dim} is outside this build "
                                      "(groups 1, 2 or 4 dividing dim)")
        if not 1 <= num_quantizers <= 32:
            raise NotImplementedError(f"{type(self).__name__}: num_quantizers={num_quantizers} is outside this build (1..32)")
        dg = dim // groups
        if not (dg == codebook_dim or (dg % 4 == 0 and dg <= 1024)):
            raise NotImplementedError(f"{type(self).__name__}: dim per group {dg} is outside this build (equal to the "
                                      f"codebook dim {codebook_dim}, or a multiple of 4 up to 1024)")
        self.groups = groups
        self.num_quantizers = num_quantizers
        self.codebook_dim = codebook_dim
        self.dim_per_group = dg
        self.rvqs = nn.ModuleList([_ScalarQuantizerGroup(dg, codebook_dim) for _ in range(groups)])
        consts, ints = constants
        self.register_buffer("sq_consts", consts, persistent=False)
        self.register_buffer("sq_ints", ints, persistent=False)

    def _weights(self):
        """(w_in [g, dc, Dg], b_in [g, dc], w_out_t [g, dc, Dg], b_out [g, Dg]) fp32, cached per weight version"""
        if self.dim_per_group == self.codebook_dim:
            return None
        params = [p_ for r in self.rvqs for p_ in (*r.project_in.parameters(), *r.project_out.parameters())]

        def pack():
            ins, outs = [r.project_in for r in self.rvqs], [r.project_out for r in self.rvqs]
            return (torch.stack([m.weight.detach() for m in ins]).float().contiguous(),
                    torch.stack([m.bias.detach() for m in ins]).float().contiguous(),
                    torch.stack([m.weight.detach().t() for m in outs]).float().contiguous(),
                    torch.stack([m.bias.detach() for m in outs]).float().contiguous())
        return SoundStream._cached(self, "_sq_weights", params, pack)

    def _encode(self, x):
        if self.training:
            raise NotImplementedError(f"{type(self).__name__} training (quantize dropout, aux losses) is outside this build")
        b, n, d = x.shape
        quant, idx = ops.sq_encode(x.reshape(b * n, d).to(f32), mode=self.mode, groups=self.groups,
                                   weights=self._weights(), consts=self.sq_consts, ints=self.sq_ints,
                                   index_dtype=self.index_dtype)
        return quant.view(b, n, d), idx.view(self.groups, b, n, self.num_quantizers)

    def get_output_from_indices(self, indices):
        """indices [g, b, n, q'] (q' <= num_quantizers leading stages, -1 = dropped) -> [b, n, dim]"""
        g, b, n, q = indices.shape
        out = ops.sq_decode(indices.reshape(g, b * n, q), mode=self.mode, Dg=self.dim_per_group,
                            weights=self._weights(), consts=self.sq_consts, ints=self.sq_ints)
        return out.view(b, n, -1)


class GroupedResidualFSQ(_GroupedScalarQuantizer):
    """residual finite scalar quantization (arXiv 2309.15505) as soundstream.py:576-587 builds it; forward returns
    (quantized, indices int32 [g, b, n, Q]), no loss.  codebook_size = prod(levels)."""

    mode = "fsq"
    index_dtype = torch.int32

    def __init__(self, *, dim, levels, num_quantizers, groups=1, **kwargs):
        levels = [int(l_) for l_ in levels]
        if not 1 <= len(levels) <= 16 or min(levels) < 2 or math.prod(levels) >= 2 ** 31:
            raise NotImplementedError(f"GroupedResidualFSQ: levels={levels} are outside this build (1 to 16 levels, each "
                                      ">= 2, product below 2^31)")
        super().__init__(dim=dim, groups=groups, num_quantizers=num_quantizers, codebook_dim=len(levels),
                         constants=ops.fsq_constants(levels, num_quantizers), kwargs=kwargs,
                         allowed_kwargs=_SQ_TRAINING_KWARGS)
        self.levels = levels
        self.codebook_size = math.prod(levels)

    def forward(self, x):
        return self._encode(x)


class GroupedResidualLFQ(_GroupedScalarQuantizer):
    """residual lookup-free quantization (arXiv 2310.05737) as soundstream.py:561-572 builds it; forward returns
    (quantized, indices int64 [g, b, n, Q], aux losses [g, Q], zero in eval)."""

    mode = "lfq"
    index_dtype = torch.int64

    def __init__(self, *, dim, num_quantizers, codebook_size, groups=1, **kwargs):
        dc = int(codebook_size).bit_length() - 1
        if codebook_size != 2 ** dc or not 1 <= dc <= 16:
            raise NotImplementedError(f"GroupedResidualLFQ: codebook_size={codebook_size} is outside this build (a power "
                                      "of two from 2 to 2^16)")
        super().__init__(dim=dim, groups=groups, num_quantizers=num_quantizers, codebook_dim=dc,
                         constants=ops.lfq_constants(dc, num_quantizers), kwargs=kwargs,
                         allowed_kwargs=_LFQ_TRAINING_KWARGS)
        self.codebook_size = codebook_size

    def forward(self, x):
        quant, idx = self._encode(x)
        return quant, idx, torch.zeros(self.groups, self.num_quantizers, device=x.device)


class SoundStream(nn.Module):
    """soundstream.py:451-866 (inference path)."""

    def __init__(self, *, channels=32, strides=(2, 4, 5, 8), channel_mults=(2, 4, 8, 16), codebook_dim=512,
                 codebook_size=None, finite_scalar_quantizer_levels=None, rq_num_quantizers=8,
                 rq_commitment_weight=1.0, rq_ema_decay=0.95, rq_quantize_dropout_multiple_of=1, rq_groups=1,
                 rq_stochastic_sample_codes=False, rq_rotation_trick=True, rq_kwargs: dict = {},
                 use_lookup_free_quantizer=False, use_finite_scalar_quantizer=False, input_channels=1,
                 discr_multi_scales=(1, 0.5, 0.25), stft_normalized=False, enc_cycle_dilations=(1, 3, 9),
                 dec_cycle_dilations=(1, 3, 9), multi_spectral_window_powers_of_two=tuple(range(6, 12)),
                 multi_spectral_n_ffts=512, multi_spectral_n_mels=64, recon_loss_weight=1.0,
                 multi_spectral_recon_loss_weight=1e-5, adversarial_loss_weight=1.0, feature_loss_weight=100,
                 quantize_dropout_cutoff_index=1, target_sample_hz=16000, use_local_attn=True, attn_window_size=128,
                 attn_dim_head=64, attn_heads=8, attn_depth=1, attn_xpos_scale_base=None,
                 attn_dynamic_pos_bias=False, use_gate_loop_layers=False, squeeze_excite=False,
                 complex_stft_discr_logits_abs=True, pad_mode="reflect", stft_discriminator=None,
                 complex_stft_discr_kwargs: dict = dict()):
        super().__init__()
        cfg = dict(locals())
        cfg.pop("self", None)
        cfg.pop("__class__", None)
        self._configs = pickle.dumps(cfg)
        self.target_sample_hz = target_sample_hz
        self.single_channel = input_channels == 1
        self.strides = strides
        layer_channels = (channels, *[m * channels for m in channel_mults])
        pairs = tuple(zip(layer_channels[:-1], layer_channels[1:]))
        # with use_gate_loop_layers a Residual(ChannelTranspose(GateLoop(C))) follows every block, on both sides
        # (soundstream.py:522-525, 618-621), which shifts the later Sequential indices as in the reference
        encoder_blocks = []
        for (ci, co), s in zip(pairs, strides):
            encoder_blocks.append(EncoderBlock(ci, co, s, enc_cycle_dilations, squeeze_excite, pad_mode))
            if use_gate_loop_layers:
                encoder_blocks.append(Residual(ChannelTranspose(GateLoop(co))))
        self.encoder = nn.Sequential(
            CausalConv1d(input_channels, channels, 7, pad_mode=pad_mode),
            *encoder_blocks,
            CausalConv1d(layer_channels[-1], codebook_dim, 3, pad_mode=pad_mode))
        attn_kwargs = dict(dim=codebook_dim, dim_head=attn_dim_head, heads=attn_heads, depth=attn_depth,
                           window_size=attn_window_size, xpos_scale_base=attn_xpos_scale_base,
                           dynamic_pos_bias=attn_dynamic_pos_bias, prenorm=True, causal=True)
        # windowed causal attention bottleneck on both sides of the quantizer (soundstream.py:533-545, 613)
        self.encoder_attn = LocalTransformer(**attn_kwargs) if use_local_attn else None
        self.decoder_attn = LocalTransformer(**attn_kwargs) if use_local_attn else None
        self.num_quantizers = rq_num_quantizers
        self.codebook_dim = codebook_dim
        self.rq_groups = rq_groups
        # quantizer choice and its asserts as soundstream.py:555-609
        assert not (use_lookup_free_quantizer and use_finite_scalar_quantizer)
        self.use_lookup_free_quantizer = use_lookup_free_quantizer
        self.use_finite_scalar_quantizer = use_finite_scalar_quantizer
        rq_common = dict(dim=codebook_dim, num_quantizers=rq_num_quantizers, groups=rq_groups, quantize_dropout=True,
                         quantize_dropout_cutoff_index=quantize_dropout_cutoff_index)
        if use_lookup_free_quantizer:
            assert exists(codebook_size) and not exists(finite_scalar_quantizer_levels), \
                "if use_finite_scalar_quantizer is set to False, `codebook_size` must be set (and not " \
                "`finite_scalar_quantizer_levels`)"
            self.rq = GroupedResidualLFQ(codebook_size=codebook_size, **rq_common, **rq_kwargs)
            self.codebook_size = codebook_size
        elif use_finite_scalar_quantizer:
            assert not exists(codebook_size) and exists(finite_scalar_quantizer_levels), \
                "if use_finite_scalar_quantizer is set to True, `finite_scalar_quantizer_levels` must be set (and not " \
                "`codebook_size`). the effective codebook size is the cumulative product of all the FSQ levels"
            self.rq = GroupedResidualFSQ(levels=finite_scalar_quantizer_levels, **rq_common, **rq_kwargs)
            self.codebook_size = self.rq.codebook_size
        else:
            assert exists(codebook_size) and not exists(finite_scalar_quantizer_levels), \
                "if use_finite_scalar_quantizer is set to False, `codebook_size` must be set (and not " \
                "`finite_scalar_quantizer_levels`)"
            # the training-only kwargs the reference passes (soundstream.py:592-607) are accepted and unused here
            self.rq = GroupedResidualVQ(dim=codebook_dim, num_quantizers=rq_num_quantizers,
                                        codebook_size=codebook_size, groups=rq_groups, decay=rq_ema_decay,
                                        commitment_weight=rq_commitment_weight,
                                        quantize_dropout_multiple_of=rq_quantize_dropout_multiple_of, kmeans_init=True,
                                        threshold_ema_dead_code=2, quantize_dropout=True,
                                        quantize_dropout_cutoff_index=quantize_dropout_cutoff_index,
                                        stochastic_sample_codes=rq_stochastic_sample_codes,
                                        rotation_trick=rq_rotation_trick, **rq_kwargs)
            self.codebook_size = codebook_size
        decoder_blocks = []
        for (ci, co), s in zip(reversed(pairs), reversed(strides)):
            decoder_blocks.append(DecoderBlock(co, ci, s, dec_cycle_dilations, squeeze_excite, pad_mode))
            if use_gate_loop_layers:
                decoder_blocks.append(Residual(ChannelTranspose(GateLoop(ci))))
        self.decoder = nn.Sequential(
            CausalConv1d(codebook_dim, layer_channels[-1], 7, pad_mode=pad_mode),
            *decoder_blocks,
            CausalConv1d(channels, input_channels, 7, pad_mode=pad_mode))
        self.register_buffer("zero", torch.tensor(0.0), persistent=False)

    # ---- bookkeeping -----------------------------------------------------------------------------
    @property
    def device(self):
        return next(self.parameters()).device

    @property
    def configs(self):
        return pickle.loads(self._configs)

    @property
    def seq_len_multiple_of(self):
        return functools.reduce(lambda a, b: a * b, self.strides)

    @property
    def downsample_factor(self):
        return self.seq_len_multiple_of

    def save(self, path):
        torch.save(dict(model=self.state_dict(), config=self._configs, version="2.4.0"), str(Path(path)))

    def load(self, path, strict=False):
        """loads encoder / decoder / rq weights; keys of sub-modules outside this build (discriminators,
        FiLM, mel transforms, local attention) are ignored unless strict=True."""
        pkg = torch.load(str(Path(path)), map_location="cpu", weights_only=False)
        sd = pkg["ema_model"] if "ema_model" in pkg else pkg["model"]
        if "ema_model" in pkg:
            sd = {k[len("ema_model."):]: v for k, v in sd.items() if k.startswith("ema_model.")}
        if not strict:
            mine = self.state_dict()
            sd = {k: v for k, v in sd.items() if k in mine}
        self.load_state_dict(sd, strict=strict)

    @classmethod
    def init_and_load_from(cls, path, strict=False):
        pkg = torch.load(str(Path(path)), map_location="cpu", weights_only=False)
        assert "config" in pkg, "model configs were not found in this saved checkpoint"
        m = cls(**pickle.loads(pkg["config"]))
        m.load(path, strict=strict)
        return m.eval()

    # ---- encoder on the tensor cores (csrc/codec_tc.cu) ------------------------------------------------
    def _tc_plan(self):
        """layer list for the split-bf16 tensor-core encoder, or None when this configuration is outside what those
        kernels are built for (then the fp32 CUDA-core kernels run).  Structure follows soundstream.py:519-531.  Units with
        a SqueezeExcite take alm_codec_ru_se_tc; a gate-loop layer after a block rides with that block's plan entry."""
        if not (ENCODER_ON_TENSOR_CORES and self.single_channel):
            return None
        enc = list(self.encoder)
        first, blocks, last = enc[0], enc[1:-1], enc[-1]
        ok = (isinstance(first, CausalConv1d) and first.conv.kernel_size[0] <= 8 and first.conv.out_channels in (32, 64)
              and first.stride == 1 and first.dilation == 1 and isinstance(last, CausalConv1d) and last.dilation == 1
              and last.conv.in_channels % 16 == 0 and last.conv.out_channels % 64 == 0)
        plan = []
        for blk in blocks if ok else ():
            gl = _gate_loop_of(blk)
            if gl is not None:
                ok = ok and bool(plan) and plan[-1][2] is None and gl.norm.gamma.numel() in GATE_LOOP_TC_CHANNELS
                if ok:
                    plan[-1] = (*plan[-1][:2], gl)
                continue
            *rus, down = list(blk)
            for ru in rus:
                c7, c1 = getattr(ru.fn, "0"), getattr(ru.fn, "2")
                C = c7.conv.in_channels
                ok = ok and (C in (32, 64, 128, 256) and c7.conv.out_channels == C and c7.conv.kernel_size[0] == 7
                             and c1.conv.kernel_size[0] == 1 and 6 * c7.dilation <= 54 and c7.stride == 1
                             and (_se_of(ru) is None or _se_of(ru).net[0].out_channels <= ops.se_inner_pad(C)))
            ok = ok and down.dilation == 1 and down.conv.in_channels % 16 == 0 and down.conv.out_channels % 64 == 0
            plan.append((rus, down, None))
        return (first, plan, last) if ok else None

    @staticmethod
    def _cached(mod, name, params, build):
        key = tuple((p_.data_ptr(), p_._version) for p_ in params)
        hit = mod.__dict__.get(name)
        if hit is None or hit[0] != key:
            with torch.inference_mode(False), torch.no_grad():
                hit = (key, build())
            mod.__dict__[name] = hit
        return hit[1]

    def _ru_tc(self, ru, h, out_phases=1):
        """one residual unit on the tensor cores (C8S in and out); SE units take alm_codec_ru_se_tc"""
        c7, c1 = getattr(ru.fn, "0"), getattr(ru.fn, "2")
        se = _se_of(ru)
        if se is None:
            wu = self._cached(ru, "_tc_units", [c7.conv.weight, c1.conv.weight],
                              lambda: ops.pack_ru_weights(c7.conv.weight, c1.conv.weight))
            return ops.codec_ru_tc(h, wu, c7.conv.bias, c1.conv.bias, dilation=c7.dilation, pad_mode=c7.pad_mode,
                                   out_phases=out_phases)
        w1, w2 = se.net[0], se.net[2]
        wu = self._cached(ru, "_tc_units_se", [c7.conv.weight, c1.conv.weight, w1.weight, w2.weight],
                          lambda: ops.pack_ru_se_weights(c7.conv.weight, c1.conv.weight, w1.weight, w2.weight))
        return ops.codec_ru_se_tc(h, wu, c7.conv.bias, c1.conv.bias, w1.bias, w2.bias, dilation=c7.dilation,
                                  pad_mode=c7.pad_mode, out_phases=out_phases)

    def _encode_tc(self, wave, plan):
        """wave fp32 [B, T] -> encoder output fp32 [B, n, codebook_dim] (channels-last, what the RVQ consumes).
        Activations stay in the C8S split-bf16 layout between layers; every layer is one kernel launch."""
        first, blocks, last = plan
        h = ops.codec_first_conv(wave, first.conv.weight, first.conv.bias, pad_mode=first.pad_mode)
        for rus, down, gl in blocks:
            for i, ru in enumerate(rus):
                h = self._ru_tc(ru, h, out_phases=down.stride if i == len(rus) - 1 else 1)
            if not rus:
                raise NotImplementedError  # (guarded by _tc_plan: every block has residual units)
            wu = self._cached(down, "_tc_units", [down.conv.weight], lambda d=down: ops.pack_conv_weights(d.conv.weight))
            h = ops.codec_conv_tc(h, wu, down.conv.bias, cout=down.conv.out_channels,
                                  kernel_size=down.conv.kernel_size[0], stride=down.stride, pad_mode=down.pad_mode)
            if gl is not None:
                h = gl.block_tc(h)
        wu = self._cached(last, "_tc_units", [last.conv.weight], lambda: ops.pack_conv_weights(last.conv.weight))
        return ops.codec_conv_tc(h, wu, last.conv.bias, cout=last.conv.out_channels,
                                 kernel_size=last.conv.kernel_size[0], stride=1, pad_mode=last.pad_mode, out_fp32=True)

    def _tc_plan_dec(self):
        """layer list for the tensor-core decoder (soundstream.py:615-627) or None"""
        if not (ENCODER_ON_TENSOR_CORES and self.single_channel):
            return None
        dec = list(self.decoder)
        first, blocks, last = dec[0], dec[1:-1], dec[-1]
        ok = (isinstance(first, CausalConv1d) and first.stride == 1 and first.dilation == 1
              and first.conv.in_channels % 16 == 0 and first.conv.out_channels % 64 == 0
              and isinstance(last, CausalConv1d) and last.conv.out_channels == 1 and last.conv.in_channels in (32, 64)
              and last.conv.kernel_size[0] <= 8 and last.stride == 1 and last.dilation == 1)
        plan = []
        for blk in blocks if ok else ():
            gl = _gate_loop_of(blk)
            if gl is not None:
                ok = ok and bool(plan) and plan[-1][2] is None and gl.norm.gamma.numel() in GATE_LOOP_TC_CHANNELS
                if ok:
                    plan[-1] = (*plan[-1][:2], gl)
                continue
            up, *rus = list(blk)
            ok = ok and isinstance(up, CausalConvTranspose1d) and up.conv.in_channels % 16 == 0 \
                and up.conv.out_channels % 16 == 0 and (up.upsample_factor * up.conv.out_channels) % 64 == 0
            for ru in rus:
                c7, c1 = getattr(ru.fn, "0"), getattr(ru.fn, "2")
                C = c7.conv.in_channels
                ok = ok and (C in (32, 64, 128, 256) and c7.conv.out_channels == C and c7.conv.kernel_size[0] == 7
                             and c1.conv.kernel_size[0] == 1 and 6 * c7.dilation <= 54 and c7.stride == 1
                             and (_se_of(ru) is None or _se_of(ru).net[0].out_channels <= ops.se_inner_pad(C)))
            plan.append((up, rus, None))
        return (first, plan, last) if ok else None

    def _decode_tc(self, x, plan):
        """x fp32 [B, n, codebook_dim] channels-last -> wave [B, 1, n * prod(strides)]; C8S between layers"""
        first, blocks, last = plan
        h = ops.codec_pack_c8s(x)
        wu = self._cached(first, "_tc_units", [first.conv.weight], lambda: ops.pack_conv_weights(first.conv.weight))
        h = ops.codec_conv_tc(h, wu, first.conv.bias, cout=first.conv.out_channels,
                              kernel_size=first.conv.kernel_size[0], stride=1, pad_mode=first.pad_mode)
        for up, rus, gl in blocks:
            s_ = up.upsample_factor
            wu = self._cached(up, "_tc_units", [up.conv.weight],
                              lambda up=up, s_=s_: ops.pack_convT_weights(up.conv.weight, s_))
            bias_up = self._cached(up, "_tc_bias", [up.conv.bias],
                                   lambda up=up, s_=s_: up.conv.bias.detach().float().repeat(s_).contiguous())
            h = ops.codec_conv_tc(h, wu, bias_up, cout=s_ * up.conv.out_channels, kernel_size=2, stride=1,
                                  pad_mode="constant", upsample=s_)
            for ru in rus:
                h = self._ru_tc(ru, h)
            if gl is not None:
                h = gl.block_tc(h)
        return ops.codec_last_conv(h, last.conv.weight, last.conv.bias, pad_mode=last.pad_mode)

    def decode_frames(self, x):
        """x [B, n, codebook_dim] channels-last (quantized) -> wave [B, 1, T] (soundstream.py:859-861)"""
        plan = self._tc_plan_dec()
        n = x.shape[1]
        # the first residual units see n x first upsampling factor samples and need more than their reflect halo
        if plan is not None and x.is_cuda and n >= 8 and n * plan[1][0][0].upsample_factor > 54:
            return self._decode_tc(x, plan)
        return self.decoder(x.transpose(1, 2).contiguous())

    def encode_frames(self, x):
        """x [B, 1, T] fp32 -> encoder output [B, n, codebook_dim] channels-last (soundstream.py:827-836)."""
        plan = self._tc_plan()
        T = x.shape[-1]
        frames = T // self.seq_len_multiple_of
        # every residual unit needs more samples than its reflect halo (6 x dilation <= 54); the shortest ones see
        # frames x last stride samples
        if plan is not None and x.is_cuda and T % self.seq_len_multiple_of == 0 and frames >= 4 \
                and frames * self.strides[-1] > 54:
            return self._encode_tc(x[:, 0].to(f32).contiguous(), plan)
        return self.encoder(x.to(f32)).transpose(1, 2).contiguous()

    # ---- hot path ----------------------------------------------------------------------------------
    def process_input(self, x, input_sample_hz=None, curtail_from_left=False):
        lead = x.shape[:-1]
        x = x.reshape(-1, x.shape[-1])  # the reference packs every leading dim ('* n', soundstream.py:785)
        resampling = exists(input_sample_hz) and input_sample_hz != self.target_sample_hz
        total = ops.resample_length(x.shape[-1], input_sample_hz, self.target_sample_hz) if resampling else x.shape[-1]
        start, count = curtail_window(total, self.seq_len_multiple_of, curtail_from_left)
        if resampling:
            x = ops.resample(x, input_sample_hz, self.target_sample_hz, start=start, count=count)
        else:
            x = x[..., start:start + count]
        return x[:, None, :], lead

    def decode_from_codebook_indices(self, quantized_indices):
        assert quantized_indices.dtype in (torch.long, torch.int32)
        if quantized_indices.ndim == 3:
            b, n, gq = quantized_indices.shape
            quantized_indices = quantized_indices.reshape(b, n, self.rq_groups, -1).permute(2, 0, 1, 3)
        return self.decode(self.rq.get_output_from_indices(quantized_indices))

    def decode(self, x, quantize=False):
        if quantize:
            x, *_ = self.rq(x)
        if exists(self.decoder_attn):
            x = self.decoder_attn(x)
        return self.decode_frames(x)

    @torch.no_grad()
    def tokenize(self, audio):
        self.eval()
        return self.forward(audio, return_codes_only=True)

    def forward(self, x, target=None, is_denoising=None, return_encoded=False, return_codes_only=False,
                return_discr_loss=False, return_discr_losses_separately=False, return_loss_breakdown=False,
                return_recons_only=False, input_sample_hz=None, apply_grad_penalty=False, curtail_from_left=False):
        if exists(is_denoising) or exists(target):
            raise NotImplementedError("FiLM denoising / target losses are outside this build")
        x, lead = self.process_input(x, input_sample_hz=input_sample_hz, curtail_from_left=curtail_from_left)
        h = self.encode_frames(x)                                      # b n c
        if exists(self.encoder_attn):
            h = self.encoder_attn(h)
        if self.use_finite_scalar_quantizer:   # FSQ has no aux loss (soundstream.py:839-845)
            quantized, indices = self.rq(h)
            commit_loss = self.zero
        else:
            quantized, indices, commit_loss = self.rq(h)
        if return_codes_only:
            return indices
        if return_encoded:
            g, b, n, q = indices.shape
            return quantized, indices.permute(1, 2, 0, 3).reshape(b, n, g * q), commit_loss
        if exists(self.decoder_attn):
            quantized = self.decoder_attn(quantized)
        recon = self.decode_frames(quantized)
        if return_recons_only:
            return recon.reshape(*lead, *recon.shape[-2:]) if len(lead) != 1 else recon
        raise NotImplementedError("SoundStream training losses (GAN / mel / feature matching) are outside this build")


def AudioLMSoundStream(strides=(2, 4, 5, 8), target_sample_hz=16000, rq_num_quantizers=12, **kwargs):
    return SoundStream(strides=strides, target_sample_hz=target_sample_hz, rq_num_quantizers=rq_num_quantizers, **kwargs)


def MusicLMSoundStream(strides=(3, 4, 5, 8), target_sample_hz=24000, rq_num_quantizers=12, **kwargs):
    return SoundStream(strides=strides, target_sample_hz=target_sample_hz, rq_num_quantizers=rq_num_quantizers, **kwargs)
