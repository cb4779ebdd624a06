"""HubertWithKmeans (hubert_kmeans.py:37-121): semantic tokens from raw audio - HuBERT features at `output_layer`,
then the nearest of the k-means centroids - on the sm_90a kernels, loading fairseq checkpoints without fairseq.

The network is fairseq's `HubertModel.extract_features(mask=False, output_layer=L)`:
  1. the conv feature extractor: "default" mode (base) has a per-channel GroupNorm over time after conv 0,
     "layer_norm" mode (large) a LayerNorm over channels after every conv; each conv is followed by GELU;
  2. LayerNorm, then `post_extract_proj`;
  3. x + GELU(grouped positional conv(x)) (weight norm folded once per weight version);
  4. LayerNorm in post-LN models;
  5. the first L encoder layers, post-LN or pre-LN, with no final LayerNorm;
  6. the nearest centroid of every frame (ops.nearest_centroid).
Precision: every conv and linear runs on the wgmma GEMM in split bf16 (x_hi w_hi + x_lo w_hi + x_hi w_lo, fp32
accumulation); the residual stream, norms and activations are fp32; attention is the one bf16 stage.  There is no CPU
path: CPU inputs raise AlmError.

Envelope (NotImplementedError at construction otherwise): extractor_mode "default" or "layer_norm"; conv widths,
encoder_embed_dim, encoder_ffn_embed_dim and embed_dim / conv_pos_groups multiples of 8; head width
encoder_embed_dim / encoder_attention_heads in {32, 64, 128}; GELU activations.  Both published families (base
768/12/3072 with 12 layers, large 1024/16/4096 with 24) are inside it; xLarge (1280 / 16 = 80) is not.  A clip must
be at least one frame long (400 samples for the published extractor); any batch size and length above that run.
"""
from __future__ import annotations

import argparse
import builtins
import collections
import io
import pickle
import types
from pathlib import Path

import torch
from torch import nn

from . import _lib, ops
from .soundstream import SoundStream

f32 = torch.float32

# ---- checkpoint loading without fairseq -------------------------------------------------------------------------------


class _StandIn:
    """Inert stand-in for a class from fairseq or omegaconf.  Called with one value (how an Enum member unpickles) it
    returns that value; otherwise it is an object that keeps its pickled state as a dict."""

    def __new__(cls, *args):
        if len(args) == 1:
            return args[0]
        return object.__new__(cls)

    def __setstate__(self, state):
        if isinstance(state, tuple) and len(state) == 2:
            state = {**(state[0] or {}), **(state[1] or {})}
        self.__dict__["state"] = state if isinstance(state, dict) else {"value": state}


def _stand_in(module, name):
    return type(name, (_StandIn,), {"__module__": module})


_TORCH_REBUILD = {"_rebuild_tensor", "_rebuild_tensor_v2", "_rebuild_tensor_v3", "_rebuild_parameter",
                  "_rebuild_parameter_with_state"}
_BUILTINS = {"set", "frozenset", "slice", "complex", "int", "float", "bool", "str", "bytes", "bytearray", "list",
             "tuple", "dict", "range"}


def _allowed(module, name):
    import numpy as np

    if module == "torch._utils" and name in _TORCH_REBUILD:
        return getattr(torch._utils, name)
    if module == "torch._tensor" and name == "_rebuild_from_type_v2":
        return torch._tensor._rebuild_from_type_v2
    if module == "torch" and isinstance(getattr(torch, name, None), torch.dtype):
        return getattr(torch, name)
    if (module, name) == ("collections", "OrderedDict"):
        return collections.OrderedDict
    if (module, name) == ("argparse", "Namespace"):
        return argparse.Namespace
    if module == "builtins" and name in _BUILTINS:
        return getattr(builtins, name)
    if module in ("numpy.core.multiarray", "numpy._core.multiarray") and name in ("_reconstruct", "scalar"):
        return getattr(np._core.multiarray if hasattr(np, "_core") else np.core.multiarray, name)
    if module == "numpy" and name in ("ndarray", "dtype"):
        return getattr(np, name)
    if module == "numpy.dtypes" and name.endswith("DType"):
        return getattr(np.dtypes, name)
    return None


class CheckpointUnpickler(pickle.Unpickler):
    """Resolves only torch's tensor / storage rebuild functions and dtypes, collections.OrderedDict,
    argparse.Namespace, numpy arrays and scalars, and plain builtin types.  Every global of fairseq.* or omegaconf.*
    becomes an inert stand-in; anything else raises pickle.UnpicklingError."""

    def find_class(self, module, name):
        if module.split(".")[0] in ("fairseq", "omegaconf"):
            return _stand_in(module, name)
        found = _allowed(module, name)
        if found is None:
            raise pickle.UnpicklingError(f"the HuBERT checkpoint loader does not load the global {module}.{name}")
        return found


_pickle_module = types.ModuleType("hubert_checkpoint_pickle")
_pickle_module.Unpickler = CheckpointUnpickler
_pickle_module.load = lambda f, **kw: CheckpointUnpickler(f, **kw).load()
_pickle_module.__name__ = "hubert_checkpoint_pickle"


def load_checkpoint(path):
    """torch.load of a fairseq checkpoint through CheckpointUnpickler (never weights_only=False)"""
    with open(path, "rb") as fh:
        data = fh.read()
    return torch.load(io.BytesIO(data), map_location="cpu", pickle_module=_pickle_module, weights_only=False)


def _plain(v):
    """stand-ins and OmegaConf node states -> plain Python values"""
    if isinstance(v, _StandIn):
        st = v.__dict__.get("state", {})
        if "_content" in st:
            return _plain(st["_content"])
        if "_val" in st:
            return _plain(st["_val"])
        return {k: _plain(x) for k, x in st.items()}
    if isinstance(v, dict):
        return {k: _plain(x) for k, x in v.items()}
    if isinstance(v, (list, tuple)):
        return type(v)(_plain(x) for x in v)
    return v


ARCH_KEYS = ("extractor_mode", "conv_feature_layers", "conv_bias", "encoder_embed_dim", "encoder_ffn_embed_dim",
             "encoder_attention_heads", "encoder_layers", "layer_norm_first", "conv_pos", "conv_pos_groups")


def read_arch(ckpt):
    """the architecture fields of a fairseq HuBERT checkpoint, from cfg["model"] or, in older checkpoints, args"""
    src = None
    cfg = _plain(ckpt.get("cfg")) if isinstance(ckpt, dict) else None
    if isinstance(cfg, dict) and isinstance(cfg.get("model"), dict):
        src = cfg["model"]
    elif isinstance(ckpt, dict) and ckpt.get("args") is not None:
        args = ckpt["args"]
        src = vars(args) if isinstance(args, argparse.Namespace) else _plain(args)
    if not isinstance(src, dict):
        raise ValueError("cannot read the HuBERT architecture: the checkpoint has neither a cfg['model'] dict nor args")
    missing = [k for k in ARCH_KEYS if k not in src]
    if missing:
        raise ValueError(f"cannot read the HuBERT architecture: the checkpoint's config lacks {', '.join(missing)}")
    arch = {k: _plain(src[k]) for k in ARCH_KEYS}
    arch["extractor_mode"] = str(arch["extractor_mode"])
    arch["activation_fn"] = str(_plain(src.get("activation_fn", "gelu")))
    return arch


def parse_conv_layers(spec):
    """fairseq's `eval(conv_feature_layers)`, restricted to int / list / tuple literals joined by + and *"""
    import ast

    def ev(n):
        if isinstance(n, ast.Expression):
            return ev(n.body)
        if isinstance(n, ast.Constant) and isinstance(n.value, int):
            return n.value
        if isinstance(n, (ast.List, ast.Tuple)):
            vals = [ev(e) for e in n.elts]
            return vals if isinstance(n, ast.List) else tuple(vals)
        if isinstance(n, ast.BinOp) and isinstance(n.op, (ast.Add, ast.Mult)):
            a, b = ev(n.left), ev(n.right)
            return a + b if isinstance(n.op, ast.Add) else a * b
        raise ValueError(f"conv_feature_layers: unsupported expression {spec!r}")

    layers = ev(ast.parse(spec, mode="eval")) if isinstance(spec, str) else spec
    if not isinstance(layers, list) or not all(isinstance(t, (tuple, list)) and len(t) == 3 for t in layers):
        raise ValueError(f"conv_feature_layers must be a list of (dim, kernel, stride), got {spec!r}")
    return [tuple(int(v) for v in t) for t in layers]


def check_envelope(arch):
    """NotImplementedError naming the first field outside what the kernels are built for"""
    if arch["extractor_mode"] not in ("default", "layer_norm"):
        raise NotImplementedError(f"extractor_mode {arch['extractor_mode']!r} (built: 'default', 'layer_norm')")
    if arch["activation_fn"] != "gelu":
        raise NotImplementedError(f"activation_fn {arch['activation_fn']!r} (built: 'gelu')")
    for c, k, s in parse_conv_layers(arch["conv_feature_layers"]):
        if c % 8 or k < 1 or s < 1:
            raise NotImplementedError(f"conv layer ({c}, {k}, {s}): widths must be multiples of 8")
    D, Fi, H, G = (arch[k] for k in ("encoder_embed_dim", "encoder_ffn_embed_dim", "encoder_attention_heads",
                                     "conv_pos_groups"))
    if D % 8 or Fi % 8:
        raise NotImplementedError(f"encoder_embed_dim {D} and encoder_ffn_embed_dim {Fi} must be multiples of 8")
    if D % H or D // H not in ops.ATTN_HEAD_WIDTHS:
        raise NotImplementedError(f"head width encoder_embed_dim / encoder_attention_heads = {D} / {H} "
                                  f"(built: {ops.ATTN_HEAD_WIDTHS})")
    if D % G or (D // G) % 8:
        raise NotImplementedError(f"positional conv group width {D} / {G} must be a multiple of 8")


def fold_pos_conv_weight(st):
    """the positional conv weight with its weight norm (dim=2) folded, w = g v / ||v|| with the norm over dims 0 and 1,
    in fp64, from either key form (weight_g / weight_v or parametrizations.weight.original0 / original1)"""
    p = "encoder.pos_conv.0."
    if p + "weight_g" in st:
        g, v = st[p + "weight_g"], st[p + "weight_v"]
    else:
        g, v = st[p + "parametrizations.weight.original0"], st[p + "parametrizations.weight.original1"]
    g, v = g.double(), v.double()
    return (g * v / v.pow(2).sum(dim=(0, 1), keepdim=True).sqrt()).float()


def receptive_field(layers):
    """samples of wave under one output frame of the conv extractor (400 for the published one)"""
    r = 1
    for _, k, s in reversed(layers):
        r = (r - 1) * s + k
    return r


class _Node(nn.Module):
    """holds the checkpoint's tensors under their fairseq names, so state_dict() keys match the reference's module"""


def _register(root, key, t):
    *path, name = key.split(".")
    mod = root
    for p in path:
        if p not in mod._modules:
            mod.add_module(p, _Node())
        mod = mod._modules[p]
    mod.register_buffer(name, t)


def curtail_to_multiple(t, mult):
    return t[..., :t.shape[-1] // mult * mult]


def resample_curtailed(wave, input_sample_hz, target_sample_hz, mult):
    """the wave resampled from input_sample_hz (None: as is) with only the samples curtail_to_multiple(., mult) keeps
    computed"""
    if input_sample_hz is None:
        return wave
    total = ops.resample_length(wave.shape[-1], input_sample_hz, target_sample_hz)
    return ops.resample(wave, input_sample_hz, target_sample_hz, count=total if mult is None else total // mult * mult)


class HubertWithKmeans(nn.Module):
    """checkpoint and kmeans as published at https://github.com/facebookresearch/fairseq/tree/main/examples/hubert
    (or your own); see the module docstring for what runs where"""

    def __init__(self, checkpoint_path, kmeans_path, target_sample_hz=16000, seq_len_multiple_of=None, output_layer=9):
        super().__init__()
        import joblib

        self.target_sample_hz = target_sample_hz
        self.seq_len_multiple_of = seq_len_multiple_of
        self.output_layer = output_layer
        assert Path(checkpoint_path).exists(), f"path {checkpoint_path} does not exist"
        assert Path(kmeans_path).exists(), f"path {kmeans_path} does not exist"
        ckpt = load_checkpoint(checkpoint_path)
        self.arch = read_arch(ckpt)
        check_envelope(self.arch)
        if not 1 <= output_layer <= self.arch["encoder_layers"]:
            raise ValueError(f"output_layer {output_layer} outside 1..{self.arch['encoder_layers']}")
        self.conv_layers = parse_conv_layers(self.arch["conv_feature_layers"])
        self.model = _Node()
        for k, v in ckpt["model"].items():
            _register(self.model, k, v)
        self.kmeans = joblib.load(kmeans_path)
        self.register_buffer("cluster_centers", torch.from_numpy(self.kmeans.cluster_centers_))

    @property
    def groups(self):
        return 1

    @property
    def codebook_size(self):
        return self.kmeans.n_clusters

    @property
    def downsample_factor(self):
        return 320  # the reference's constant (hubert_kmeans.py:85-88), whatever the extractor's strides

    # ---- weights in the GEMM layouts, rebuilt when a tensor changes -------------------------------------------------
    def _packed(self):
        st = dict(self.model.state_dict(keep_vars=True))
        return SoundStream._cached(self, "_packed_weights", [*st.values(), self.cluster_centers],
                                   lambda: self._pack(st))

    def _pack(self, st):
        a, P = self.arch, {}
        for i, (_, k, _) in enumerate(self.conv_layers):
            w = st[f"feature_extractor.conv_layers.{i}.0.weight"].float()
            P[f"conv{i}"] = w.contiguous() if i == 0 else ops.pack_split_conv_weight(w)
        if "post_extract_proj.weight" in st:
            P["proj"] = ops.pack_split_weight(st["post_extract_proj.weight"].float())
        w = fold_pos_conv_weight(st).to(st["encoder.pos_conv.0.bias"].device)
        D, G, k = w.shape[0], a["conv_pos_groups"], w.shape[2]
        P["pos"] = ops.pack_split_conv_weight(w).view(G, D // G, k * 3 * (D // G))
        for i in range(self.output_layer):
            p = f"encoder.layers.{i}."
            qkv = torch.cat([st[p + f"self_attn.{n}_proj.weight"].float() for n in "qkv"])
            P[p + "qkv"] = ops.pack_split_weight(qkv)
            P[p + "qkv_bias"] = torch.cat([st[p + f"self_attn.{n}_proj.bias"].float() for n in "qkv"]).contiguous()
            for n in ("self_attn.out_proj", "fc1", "fc2"):
                P[p + n] = ops.pack_split_weight(st[p + n + ".weight"].float())
        P["centers"] = ops.rvq_pack_codebooks(self.cluster_centers.float()[None])
        return P

    def _vec(self, name):
        t = getattr_path(self.model, name)
        return t if t.dtype == f32 else t.float()

    # ---- forward -----------------------------------------------------------------------------------------------------
    def extract_features(self, wave):
        """fp32 wave [B, T] on the GPU -> features fp32 [B, n, D] after encoder layer `output_layer`"""
        a, P, v = self.arch, self._packed(), self._vec
        if wave.shape[-1] < receptive_field(self.conv_layers):
            raise ValueError(f"a clip of {wave.shape[-1]} samples is shorter than one frame "
                             f"({receptive_field(self.conv_layers)} samples)")
        wave = wave.to(f32).contiguous()
        B = wave.shape[0]
        ln_mode = a["extractor_mode"] == "layer_norm"
        bias = (lambda i: v(f"feature_extractor.conv_layers.{i}.0.bias")) if a["conv_bias"] else (lambda i: None)
        n_conv = len(self.conv_layers)
        with ops._timed("hubert_conv_extractor", _conv_flops(self.conv_layers, B, wave.shape[-1])):
            for i, (c, k, s) in enumerate(self.conv_layers):
                norm = f"feature_extractor.conv_layers.{i}.2" + (".1" if ln_mode else "")
                if i == 0:
                    y = ops.hubert_conv0(wave, P["conv0"], bias(0), stride=s)
                else:
                    y = ops.hubert_conv_gemm(xs, P[f"conv{i}"], bias(i), kernel_size=k, stride=s)
                last = i == n_conv - 1
                kw = dict(gelu=True, want_out=last, want_split=not last)
                if ln_mode:
                    out, xs = ops.hubert_norm_act(y, ln=True, gamma=v(norm + ".weight"), beta=v(norm + ".bias"), **kw)
                elif i == 0:
                    out, xs = ops.hubert_norm_act(y, stats=ops.hubert_chan_stats(y), gamma=v(norm + ".weight"),
                                                  beta=v(norm + ".bias"), **kw)
                else:
                    out, xs = ops.hubert_norm_act(y, **kw)
            proj = "proj" in P
            x, xs = ops.hubert_norm_act(out, ln=True, gamma=v("layer_norm.weight"), beta=v("layer_norm.bias"),
                                        want_out=not proj, want_split=proj)
            if proj:
                x = ops.split_gemm(xs, P["proj"], v("post_extract_proj.bias"), cls="hubert_proj_gemm")
        T, D = x.shape[1], x.shape[2]
        pre_ln = bool(a["layer_norm_first"])
        L = self.output_layer
        with ops._timed("hubert_pos_conv", 2.0 * B * T * D * (D // a["conv_pos_groups"]) * a["conv_pos"]):
            y = ops.hubert_pos_conv(x, P["pos"], kernel_size=a["conv_pos"])
            nxt = "encoder.layers.0.self_attn_layer_norm" if pre_ln else "encoder.layer_norm"
            xs = ops.hubert_add_ln(x, y, T=T, groups=a["conv_pos_groups"], y_bias=v("encoder.pos_conv.0.bias"),
                                   y_gelu=True, gamma=v(nxt + ".weight"), beta=v(nxt + ".bias"), keep_ln=not pre_ln)
        Fi, H = a["encoder_ffn_embed_dim"], a["encoder_attention_heads"]
        with ops._timed("hubert_layers", L * B * (2.0 * T * D * (4 * D + 2 * Fi) + 4.0 * T * T * D)):
            for i in range(L):
                p = f"encoder.layers.{i}."
                qkv = ops.split_gemm(xs, P[p + "qkv"], P[p + "qkv_bias"], cls="hubert_layer_gemm")
                os_ = ops.hubert_attention(qkv, heads=H)
                y = ops.split_gemm(os_, P[p + "self_attn.out_proj"], v(p + "self_attn.out_proj.bias"),
                                   cls="hubert_layer_gemm")
                nxt = p + ("final_layer_norm" if pre_ln else "self_attn_layer_norm")
                xs = ops.hubert_add_ln(x, y, T=T, gamma=v(nxt + ".weight"), beta=v(nxt + ".bias"), keep_ln=not pre_ln)
                h = ops.split_gemm(xs, P[p + "fc1"], v(p + "fc1.bias"), cls="hubert_layer_gemm")
                _, hs = ops.hubert_norm_act(h, gelu=True)
                y = ops.split_gemm(hs, P[p + "fc2"], v(p + "fc2.bias"), cls="hubert_layer_gemm")
                if pre_ln:
                    nxt = f"encoder.layers.{i + 1}.self_attn_layer_norm" if i + 1 < L else None
                else:
                    nxt = p + "final_layer_norm"
                g_, b_ = (v(nxt + ".weight"), v(nxt + ".bias")) if nxt else (None, None)
                xs = ops.hubert_add_ln(x, y, T=T, gamma=g_, beta=b_, keep_ln=not pre_ln, want_split=i + 1 < L)
        return x

    def assign(self, features):
        """nearest centroid of every frame: features fp32 [B, n, D] -> int64 [B, n]"""
        B, n, D = features.shape
        C = self.cluster_centers.shape[0]
        with ops._timed("hubert_assignment", 2.0 * B * n * C * D):
            return ops.nearest_centroid(features.reshape(B * n, D), self._packed()["centers"]).view(B, n)

    @torch.inference_mode()
    def forward(self, wav_input, flatten=True, input_sample_hz=None):
        if not wav_input.is_cuda:
            raise _lib.AlmError("HubertWithKmeans runs on the GPU only (no CPU fallback); move the module and the "
                                "wave to a CUDA device")
        wav_input = resample_curtailed(wav_input, input_sample_hz, self.target_sample_hz, self.seq_len_multiple_of)
        if self.seq_len_multiple_of is not None:
            wav_input = curtail_to_multiple(wav_input, self.seq_len_multiple_of)
        clusters = self.assign(self.extract_features(wav_input))
        if flatten:
            return clusters
        return clusters.reshape(clusters.shape[0], -1)


def getattr_path(mod, name):
    for p in name.split("."):
        mod = getattr(mod, p)
    return mod


def _conv_flops(layers, B, T):
    """algorithmic FLOPs of the conv feature extractor for B clips of T samples"""
    flops, cin = 0.0, 1
    for c, k, s in layers:
        T = (T - k) // s + 1
        flops += 2.0 * B * T * c * cin * k
        cin = c
    return flops
