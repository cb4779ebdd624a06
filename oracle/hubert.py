"""CPU restatement of fairseq's HuBERT feature path, `HubertModel.extract_features(mask=False, output_layer=L)` as
called by the reference's HubertWithKmeans (hubert_kmeans.py:107-116), and its k-means assignment.

Pure torch on fairseq-layout state dicts (`feature_extractor.conv_layers.{i}.0.weight`, `encoder.layers.{i}.fc1`, ...),
any dtype (tests run it in fp64).  Both published families: the "default" extractor (GroupNorm after conv 0) with
post-LN layers (base), and the "layer_norm" extractor with pre-LN layers (large).  Parity with fairseq itself is
unpinned (fairseq is not installable offline); oracle/make_golden_hubert.py pins it against transformers' HubertModel,
an independent port.
"""
from __future__ import annotations

import argparse
import ast
import enum
import sys
import types

import torch
import torch.nn.functional as F

EPS = 1e-5


def parse_conv_layers(spec: str):
    """fairseq's `eval(conv_feature_layers)` restricted to list / tuple / int literals joined by + and *."""
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
        raise ValueError(f"conv_feature_layers: unsupported expression {ast.dump(n)}")

    layers = ev(ast.parse(spec, mode="eval"))
    if not isinstance(layers, list) or not all(isinstance(t, tuple) and len(t) == 3 for t in layers):
        raise ValueError(f"conv_feature_layers must be a list of (dim, kernel, stride) tuples, got {spec!r}")
    return layers


def fold_weight_norm(g, v):
    """weight_norm(dim=2) of the positional conv: w = g * v / ||v||, the norm over dims 0 and 1 per kernel tap."""
    return g * v / v.pow(2).sum(dim=(0, 1), keepdim=True).sqrt()


def pos_conv_weight(st):
    """the folded positional conv weight from either key form of its weight norm"""
    p = "encoder.pos_conv.0."
    if p + "weight_g" in st:
        return fold_weight_norm(st[p + "weight_g"], st[p + "weight_v"])
    return fold_weight_norm(st[p + "parametrizations.weight.original0"], st[p + "parametrizations.weight.original1"])


def _ln(x, st, name):
    return F.layer_norm(x, x.shape[-1:], st[name + ".weight"], st[name + ".bias"], EPS)


def _lin(x, st, name):
    return F.linear(x, st[name + ".weight"], st.get(name + ".bias"))


def _attn(x, st, p, heads):
    B, T, D = x.shape
    dh = D // heads
    q = _lin(x, st, p + "q_proj") * dh ** -0.5
    k, v = _lin(x, st, p + "k_proj"), _lin(x, st, p + "v_proj")
    q, k, v = (t.view(B, T, heads, dh).transpose(1, 2) for t in (q, k, v))
    o = torch.softmax(q @ k.transpose(-1, -2), dim=-1) @ v
    return _lin(o.transpose(1, 2).reshape(B, T, D), st, p + "out_proj")


def conv_features(st, arch, wave):
    """ConvFeatureExtractionModel: wave [B, T] -> [B, T', C] (channels last)"""
    x = wave[:, None, :]
    for i, (_, k, s) in enumerate(parse_conv_layers(arch["conv_feature_layers"])):
        p = f"feature_extractor.conv_layers.{i}."
        x = F.conv1d(x, st[p + "0.weight"], st.get(p + "0.bias"), stride=s)
        if arch["extractor_mode"] == "layer_norm":
            x = _ln(x.transpose(1, 2), st, p + "2.1").transpose(1, 2)
        elif i == 0:
            x = F.group_norm(x, x.shape[1], st[p + "2.weight"], st[p + "2.bias"], EPS)
        x = F.gelu(x)
    return x.transpose(1, 2)


def extract_features(st, arch, wave, output_layer):
    """[B, T] wave -> [B, T', D] features after encoder layer `output_layer` (1-based), no final LayerNorm"""
    x = _ln(conv_features(st, arch, wave), st, "layer_norm")
    if "post_extract_proj.weight" in st:
        x = _lin(x, st, "post_extract_proj")
    k, groups = arch["conv_pos"], arch["conv_pos_groups"]
    y = F.conv1d(x.transpose(1, 2), pos_conv_weight(st), st["encoder.pos_conv.0.bias"], padding=k // 2, groups=groups)
    x = x + F.gelu(y[:, :, :x.shape[1]].transpose(1, 2))
    pre_ln = arch["layer_norm_first"]
    if not pre_ln:
        x = _ln(x, st, "encoder.layer_norm")
    heads = arch["encoder_attention_heads"]
    for i in range(output_layer):
        p = f"encoder.layers.{i}."
        if pre_ln:
            x = x + _attn(_ln(x, st, p + "self_attn_layer_norm"), st, p + "self_attn.", heads)
            x = x + _lin(F.gelu(_lin(_ln(x, st, p + "final_layer_norm"), st, p + "fc1")), st, p + "fc2")
        else:
            x = _ln(x + _attn(x, st, p + "self_attn.", heads), st, p + "self_attn_layer_norm")
            x = _ln(x + _lin(F.gelu(_lin(x, st, p + "fc1")), st, p + "fc2"), st, p + "final_layer_norm")
    return x


def assign(features, centers):
    """`(-torch.cdist(embed, centers)).argmax(-1)` (hubert_kmeans.py:114-116), lowest index on ties"""
    return torch.cdist(features, centers[None].to(features.dtype).expand(features.shape[0], -1, -1)).argmin(-1)


def margins(features, centers):
    """distance gap between the nearest and the runner-up centroid, per frame"""
    d = torch.cdist(features, centers[None].to(features.dtype).expand(features.shape[0], -1, -1))
    two = d.topk(2, dim=-1, largest=False).values
    return two[..., 1] - two[..., 0]


def random_state(arch, *, seed, final_proj_dim=16, num_classes=8):
    """seeded random weights in the fairseq checkpoint layout, unused tensors included, scaled so activations keep
    unit size through every layer"""
    g = torch.Generator().manual_seed(seed)

    def rn(*shape, scale):
        return torch.randn(*shape, generator=g) * scale

    def ln(name, d):
        st[name + ".weight"] = 1 + rn(d, scale=0.1)
        st[name + ".bias"] = rn(d, scale=0.1)

    def lin(name, n, k):
        st[name + ".weight"] = rn(n, k, scale=k ** -0.5)
        st[name + ".bias"] = rn(n, scale=0.1)

    st = {}
    cin = 1
    for i, (c, k, s) in enumerate(parse_conv_layers(arch["conv_feature_layers"])):
        p = f"feature_extractor.conv_layers.{i}."
        st[p + "0.weight"] = rn(c, cin, k, scale=(cin * k) ** -0.5)
        if arch["conv_bias"]:
            st[p + "0.bias"] = rn(c, scale=0.1)
        if arch["extractor_mode"] == "layer_norm":
            ln(p + "2.1", c)
        elif i == 0:
            ln(p + "2", c)
        cin = c
    D, Fi = arch["encoder_embed_dim"], arch["encoder_ffn_embed_dim"]
    ln("layer_norm", cin)
    if cin != D:
        lin("post_extract_proj", D, cin)
    st["mask_emb"] = rn(D, scale=1.0)
    k, groups = arch["conv_pos"], arch["conv_pos_groups"]
    v = rn(D, D // groups, k, scale=1.0)
    gw = rn(1, 1, k, scale=0.3).abs() + 0.2
    p = "encoder.pos_conv.0."
    st[p + "weight_g"], st[p + "weight_v"] = gw, v
    st[p + "bias"] = rn(D, scale=0.1)
    ln("encoder.layer_norm", D)
    for i in range(arch["encoder_layers"]):
        p = f"encoder.layers.{i}."
        for n_ in ("q_proj", "k_proj", "v_proj", "out_proj"):
            lin(p + "self_attn." + n_, D, D)
        ln(p + "self_attn_layer_norm", D)
        lin(p + "fc1", Fi, D)
        lin(p + "fc2", D, Fi)
        ln(p + "final_layer_norm", D)
    lin("final_proj", final_proj_dim, D)
    st["label_embs_concat"] = rn(num_classes, final_proj_dim, scale=1.0)
    return st


BASE = dict(extractor_mode="default", conv_feature_layers="[(512,10,5)] + [(512,3,2)] * 4 + [(512,2,2)] * 2",
            conv_bias=False, encoder_embed_dim=768, encoder_ffn_embed_dim=3072, encoder_attention_heads=12,
            encoder_layers=12, layer_norm_first=False, conv_pos=128, conv_pos_groups=16)
LARGE = dict(BASE, extractor_mode="layer_norm", conv_bias=True, encoder_embed_dim=1024, encoder_ffn_embed_dim=4096,
             encoder_attention_heads=16, encoder_layers=24, layer_norm_first=True)


# ---- checkpoint and k-means files in the published formats, for tests ------------------------------------------------
FAKE_ENUM_MODULE = "fairseq.dataclass.constants"


def fake_fairseq_enum():
    """an Enum that pickles as a global of fairseq.dataclass.constants, as fairseq's ChoiceEnum members do; installs
    the module and returns (enum class, names of the sys.modules entries it added)"""
    added = [n for n in ("fairseq", "fairseq.dataclass", FAKE_ENUM_MODULE) if n not in sys.modules]
    for n in added:
        sys.modules[n] = types.ModuleType(n)
    mode = enum.Enum("ExtractorMode", {"default": "default", "layer_norm": "layer_norm"}, module=FAKE_ENUM_MODULE)
    sys.modules[FAKE_ENUM_MODULE].ExtractorMode = mode
    return mode, added


def parametrized_weight_norm(st):
    """the same state with the positional conv's weight norm under torch's parametrization key names"""
    p = "encoder.pos_conv.0."
    ren = {p + "weight_g": p + "parametrizations.weight.original0", p + "weight_v": p + "parametrizations.weight.original1"}
    return {ren.get(k, k): v for k, v in st.items()}


def write_checkpoint(path, st, arch, form="cfg"):
    """a fairseq-layout checkpoint: form "cfg" stores cfg = {"model": arch} with extractor_mode as a fairseq enum member
    (the fake module is removed again afterwards), form "args" stores arch as an argparse.Namespace"""
    if form == "args":
        torch.save({"model": st, "args": argparse.Namespace(**arch)}, path)
        return
    mode, added = fake_fairseq_enum()
    try:
        torch.save({"model": st, "cfg": {"model": dict(arch, extractor_mode=mode(arch["extractor_mode"]))}}, path)
    finally:
        for n in added:
            sys.modules.pop(n, None)


def write_kmeans(path, centers):
    """a joblib file holding a fitted-looking sklearn MiniBatchKMeans with these centroids"""
    import joblib
    from sklearn.cluster import MiniBatchKMeans

    km = MiniBatchKMeans(n_clusters=centers.shape[0])
    km.cluster_centers_ = centers.numpy()
    joblib.dump(km, path)
