"""Generate tests/golden/hubert.pt - build container only.

    python -m oracle.make_golden_hubert

1. Pins oracle/hubert.py against transformers' HubertModel (an independent port of fairseq HuBERT) in fp64 on both
   families (a base-like "default"-extractor post-LN model and a large-like "layer_norm"-extractor pre-LN model),
   comparing `hidden_states[L]` with the keys mapped.
2. Runs the REAL reference hubert_kmeans.py (oracle/ref_import.py) with fairseq's
   `checkpoint_utils.load_model_ensemble_and_task` bound to the oracle, on a small seeded base-like model
   (64 conv channels, D = 128, 4 heads, 4 layers, the published positional conv), and records its ids.
3. Writes: the fairseq-layout state dict; its architecture cfg as a plain dict (tests pickle it once with
   `extractor_mode` as a member of a fake `fairseq` enum, oracle.hubert.write_checkpoint, and once as `args`); the
   centroids; waves of several lengths (odd ones and a one-frame clip); the fp64 oracle's features at output_layer;
   the reference's ids.
"""
from __future__ import annotations

import sys
import tempfile
from pathlib import Path
from types import SimpleNamespace

import torch

from . import golden, ref_import
from . import hubert as oh

NAME = "hubert.pt"
SMALL = dict(oh.BASE, conv_feature_layers="[(64,10,5)] + [(64,3,2)] * 4 + [(64,2,2)] * 2",
             encoder_embed_dim=128, encoder_ffn_embed_dim=256, encoder_attention_heads=4, encoder_layers=4)
OUTPUT_LAYER = 3
LENGTHS = (400, 1601, 3203, 8000)
N_CLUSTERS = 50


def to_transformers(st, arch):
    """oracle (fairseq) keys -> transformers HubertModel keys"""
    out = {}
    for k, v in st.items():
        n = k
        if k.startswith("feature_extractor.conv_layers."):
            i, rest = k.split(".")[2], ".".join(k.split(".")[3:])
            rest = {"0.weight": "conv.weight", "0.bias": "conv.bias", "2.weight": "layer_norm.weight",
                    "2.bias": "layer_norm.bias", "2.1.weight": "layer_norm.weight",
                    "2.1.bias": "layer_norm.bias"}[rest]
            n = f"feature_extractor.conv_layers.{i}.{rest}"
        elif k.startswith("layer_norm."):
            n = "feature_projection." + k
        elif k.startswith("post_extract_proj."):
            n = k.replace("post_extract_proj.", "feature_projection.projection.")
        elif k.startswith("encoder.pos_conv.0."):
            n = {"weight_g": "parametrizations.weight.original0", "weight_v": "parametrizations.weight.original1",
                 "bias": "bias"}[k.split(".")[-1]]
            n = "encoder.pos_conv_embed.conv." + n
        elif k.startswith("encoder.layers."):
            n = (k.replace("self_attn.", "attention.").replace("self_attn_layer_norm", "layer_norm")
                 .replace("fc1", "feed_forward.intermediate_dense").replace("fc2", "feed_forward.output_dense"))
        elif k in ("mask_emb",) or k.startswith(("final_proj", "label_embs")):
            continue
        out[n] = v
    return out


def transformers_model(arch):
    from transformers import HubertConfig, HubertModel

    layers = oh.parse_conv_layers(arch["conv_feature_layers"])
    cfg = HubertConfig(
        hidden_size=arch["encoder_embed_dim"], num_hidden_layers=arch["encoder_layers"],
        num_attention_heads=arch["encoder_attention_heads"], intermediate_size=arch["encoder_ffn_embed_dim"],
        hidden_act="gelu", feat_extract_activation="gelu",
        feat_extract_norm="layer" if arch["extractor_mode"] == "layer_norm" else "group",
        conv_dim=[c for c, _, _ in layers], conv_kernel=[k for _, k, _ in layers], conv_stride=[s for _, _, s in layers],
        conv_bias=arch["conv_bias"], num_conv_pos_embeddings=arch["conv_pos"],
        num_conv_pos_embedding_groups=arch["conv_pos_groups"], do_stable_layer_norm=arch["layer_norm_first"],
        feat_proj_layer_norm=True, layer_norm_eps=1e-5, hidden_dropout=0.0, attention_dropout=0.0,
        activation_dropout=0.0, feat_proj_dropout=0.0, layerdrop=0.0, apply_spec_augment=False)
    return HubertModel(cfg).eval()


def pin_against_transformers(arch, seed, layer):
    st = oh.random_state(arch, seed=seed)
    m = transformers_model(arch).double()
    missing, unexpected = m.load_state_dict({k: v.double() for k, v in to_transformers(st, arch).items()},
                                            strict=False)
    assert not unexpected and all("masked_spec_embed" in k for k in missing), (missing, unexpected)
    wave = torch.randn(2, 3203, generator=torch.Generator().manual_seed(seed + 1), dtype=torch.float64)
    with torch.no_grad():
        ref = m(wave, output_hidden_states=True).hidden_states[layer]
    ours = oh.extract_features({k: v.double() for k, v in st.items()}, arch, wave, layer)
    err = ((ours - ref).abs().max() / ref.abs().max()).item()
    print(f"  oracle vs transformers.HubertModel ({arch['extractor_mode']}, layer {layer}): max rel err {err:.2e}")
    assert err < 1e-10, err


class _OracleHubert(torch.nn.Module):
    def __init__(self, st, arch):
        super().__init__()
        self.st, self.arch = st, arch

    def forward(self, wav, features_only=True, mask=False, output_layer=None):
        assert features_only and not mask
        return {"x": oh.extract_features(self.st, self.arch, wav.float(), output_layer)}


def load_model_ensemble_and_task(inputs):
    (ckpt,) = inputs.values()
    return [_OracleHubert(ckpt["model"], ckpt["cfg"]["model"])], ckpt["cfg"], None


def main():
    print("oracle vs transformers:")
    pin_against_transformers(dict(SMALL, encoder_layers=3), seed=11, layer=3)
    pin_against_transformers(dict(oh.LARGE, conv_feature_layers=SMALL["conv_feature_layers"], encoder_embed_dim=128,
                                  encoder_ffn_embed_dim=256, encoder_attention_heads=4, encoder_layers=3),
                             seed=12, layer=2)

    st = oh.random_state(SMALL, seed=21)
    gen = torch.Generator().manual_seed(22)
    waves = [torch.randn(2 if n > 400 else 1, n, generator=gen) for n in LENGTHS]
    feats64 = [oh.extract_features({k: v.double() for k, v in st.items()}, SMALL, w.double(), OUTPUT_LAYER)
               for w in waves]
    # centroids: frames of the clips themselves, perturbed, so the assignment has realistic margins
    pool = torch.cat([f.reshape(-1, f.shape[-1]) for f in feats64]).float()
    centers = (pool[torch.randperm(pool.shape[0], generator=gen)[:N_CLUSTERS]]
               + 0.3 * torch.randn(N_CLUSTERS, pool.shape[1], generator=gen)).contiguous()

    ref = ref_import.load()
    sys.modules["fairseq"].checkpoint_utils = SimpleNamespace(load_model_ensemble_and_task=load_model_ensemble_and_task)
    import audiolm_pytorch.hubert_kmeans as hk  # noqa: E402  (the reference module, through ref_import's package)

    del ref
    with tempfile.TemporaryDirectory() as d:
        ck, km = Path(d) / "hubert.pt", Path(d) / "km.bin"
        torch.save({"model": st, "cfg": {"model": dict(SMALL)}}, ck)
        oh.write_kmeans(km, centers)
        ref_model = hk.HubertWithKmeans(str(ck), str(km), output_layer=OUTPUT_LAYER)
        ids = [ref_model(w) for w in waves]
    for w, f, i in zip(waves, feats64, ids):
        assert torch.equal(i, oh.assign(f, centers)), "reference ids differ from the fp64 oracle's"
        m = oh.margins(f, centers)
        print(f"  wave {tuple(w.shape)}: {i.shape[1]} frames, smallest centroid gap {m.min():.2e}")
    print("  [ok] reference ids equal the fp64 oracle's")

    with tempfile.TemporaryDirectory() as d:
        oh.write_checkpoint(Path(d) / "enum.pt", {}, SMALL)
        assert b"fairseq.dataclass.constants" in (Path(d) / "enum.pt").read_bytes(), "the enum must pickle as a global"
    out = dict(arch=SMALL, output_layer=OUTPUT_LAYER, state=st, centers=centers, waves=waves,
               features=[f.float() for f in feats64], ids=ids)
    golden.save(out, NAME)
    size = sum(p.stat().st_size for p in golden.GOLDEN.glob(NAME + "*"))
    print(f"wrote {NAME}: {size / 1e6:.2f} MB")


if __name__ == "__main__":
    sys.exit(main())
