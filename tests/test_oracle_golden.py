"""CPU: the oracle restatements reproduce the committed goldens (generated from the real reference by
oracle/make_golden.py).  This is what pins the oracle; GPU tests then compare the CUDA path to it."""
import pytest
import torch

from oracle import codec as oc
from oracle import golden
from oracle import transformer as ot


def load(name):
    return golden.load(name)


def close(a, b, tol=2e-4):
    return (a.float() - b.float()).abs().max().item() <= tol * max(1.0, b.float().abs().max().item())


def test_attend():
    g = load("attend.pt")
    q, k, v, mask, bias, out = g["q"], g["k"], g["v"], g["mask"], g["bias"], g["out"]
    assert close(ot.attend(q, k, v, mask=mask), out["math_masked"])
    assert close(ot.attend(q, k, v, mask=mask), out["flash_masked"])
    assert close(ot.attend(q, k, v, mask=mask, attn_bias=bias), out["math_bias"])
    assert close(ot.attend(q, k, v), out["math_causal"])
    assert close(ot.attend(q[:, :, -5:], k, v, mask=mask), out["math_cached"])


def test_semantic():
    g = load("semantic.pt")
    hk = dict(heads=g["kwargs"]["heads"], depth=g["kwargs"]["depth"])
    st, ids = g["state"], g["ids"]
    assert close(ot.semantic_forward(st, ids, **hk)[0], g["logits"])
    assert close(ot.semantic_forward(st, ids, self_attn_mask=g["mask"], **hk)[0], g["logits_masked"])
    _, c12 = ot.semantic_forward(st, ids[:, :12], **hk)
    assert close(c12, g["cache12"])
    inc, _ = ot.semantic_forward(st, ids, kv_cache=c12, **hk)
    assert close(inc, g["logits_inc"])
    assert close(inc, g["logits"][:, 13:], 1e-3)  # KV-cache decode == full forward


def test_semantic_single_residual_stream():
    g = load("semantic_plain.pt")
    hk = dict(heads=2, depth=2, num_streams=1)
    assert close(ot.semantic_forward(g["state"], g["ids"], **hk)[0], g["logits"])
    assert close(ot.semantic_forward(g["state"], g["ids"], self_attn_mask=g["mask"], **hk)[0], g["logits_masked"])


def test_semantic_grads():
    g = load("semantic.pt")
    st = {k: v.clone().requires_grad_(v.is_floating_point()) for k, v in g["state"].items()}
    ids = g["ids"]
    labels = torch.cat((ids, torch.full((2, 1), 50)), dim=1)
    logits, _ = ot.semantic_forward(st, labels[:, :-1], heads=2, depth=2)
    loss = ot.cross_entropy(logits, labels)
    assert close(loss, g["loss"], 1e-5)
    loss.backward()
    for k, gr in g["grads"].items():
        # grad_shrink (audiolm_pytorch.py:93-94) scales what flows into the embeddings by 0.1
        scale = 0.1 if k in ("start_token", "semantic_embedding.weight") else 1.0
        assert close(st[k].grad * scale, gr, 1e-3), k


def test_coarse():
    g = load("coarse.pt")
    kw = g["kwargs"]
    hk = dict(heads=kw["heads"], depth=kw["depth"], codebook_size=kw["codebook_size"],
              num_coarse_quantizers=kw["num_coarse_quantizers"])
    st, sem, coarse = g["state"], g["sem"], g["coarse"]
    (sl, cl), _ = ot.coarse_forward(st, sem, coarse, **hk)
    assert close(sl, g["sem_logits"]) and close(cl, g["coarse_logits"])
    (slm, clm), _ = ot.coarse_forward(st, sem, coarse, self_attn_mask=g["mask"], **hk)
    assert close(slm, g["sem_logits_masked"]) and close(clm, g["coarse_logits_masked"])
    (_, _), (kv_a, emb_a) = ot.coarse_forward(st, sem, coarse[:, :9], return_only_coarse_logits=True, **hk)
    assert close(kv_a, g["kv_a"]) and close(emb_a, g["emb_a"])
    (_, cb), _ = ot.coarse_forward(st, sem, coarse[:, :10], kv_cache=kv_a, embed_cache=emb_a,
                                   return_only_coarse_logits=True, **hk)
    assert close(cb, g["coarse_logits_b"])


def test_fine():
    g = load("fine.pt")
    kw = g["kwargs"]
    hk = dict(heads=kw["heads"], depth=kw["depth"], codebook_size=kw["codebook_size"],
              num_coarse_quantizers=kw["num_coarse_quantizers"], num_fine_quantizers=kw["num_fine_quantizers"])
    (cl, fl), _ = ot.fine_forward(g["state"], g["coarse"], g["fine"], **hk)
    assert close(cl, g["coarse_logits"]) and close(fl, g["fine_logits"])


def test_sampling():
    g = load("sampling.pt")
    filt = ot.top_k_filter(g["logits"])
    assert torch.equal(filt, g["filtered"])
    assert int((filt > float("-inf")).sum(-1)[0]) == max(int(0.1 * 65), 1)
    assert torch.equal(ot.gumbel_argmax(filt, g["uniform"]), g["ids"])


def test_soundstream():
    g = load("soundstream.pt")
    st, wave = g["state"], g["wave"]
    assert close(oc.encoder(ot.sub(st, "encoder"), wave[:, None]), g["enc"])
    quant, idx = oc.soundstream_tokenize(st, wave)
    assert torch.equal(idx, g["idx"])
    assert torch.equal(idx[None], g["codes"])  # tokenize returns raw (g, b, n, q)
    assert close(quant, g["quant"])
    assert close(oc.soundstream_decode_indices(st, idx), g["recon"][:, None] if g["recon"].dim() == 2 else g["recon"])


@pytest.mark.parametrize("name", ["k7", "k7d3", "k7d9", "k1", "s2", "s4", "s5", "s8", "k3"])
@pytest.mark.parametrize("mode", ["reflect", "constant"])
def test_causal_convs(name, mode):
    c = load("soundstream.pt")["convs"][f"{name}/{mode}"]
    y = oc.causal_conv1d(c["x"], c["w"], c["b"], c["stride"], c["dilation"], c["mode"])
    assert close(y, c["y"], 1e-5)
    # causality past the reflect halo: output t only depends on inputs <= t*stride
    x2 = c["x"].clone()
    x2[..., 60:] += 1.0
    y2 = oc.causal_conv1d(x2, c["w"], c["b"], c["stride"], c["dilation"], c["mode"])
    t_safe = 59 // c["stride"]
    assert torch.equal(y[..., :t_safe], y2[..., :t_safe])


@pytest.mark.parametrize("s", [2, 4, 5, 8])
def test_causal_conv_transpose(s):
    c = load("soundstream.pt")["convs"][f"convT{s}"]
    y = oc.causal_conv_transpose1d(c["x"], c["w"], c["b"], s)
    assert y.shape[-1] == c["x"].shape[-1] * s
    assert close(y, c["y"], 1e-5)


def test_relative_position_bias_models():
    """flash_attn=False models (SURVEY §8 a7): RelativePositionBias / cross_attn_bias / pos_bias_mlp."""
    import torch.nn.functional as F

    g = load("relpos.pt")

    def ce(lg, lb):
        return F.cross_entropy(lg.transpose(1, 2), lb)

    s = g["semantic"]
    hk = dict(heads=2, depth=2)
    lg, _ = ot.semantic_forward(s["state"], s["ids"], **hk)
    assert close(lg, s["logits"])
    assert close(ot.semantic_forward(s["state"], s["ids"], self_attn_mask=s["mask"], **hk)[0], s["logits_masked"])
    _, c12 = ot.semantic_forward(s["state"], s["ids"][:, :12], **hk)
    assert close(ot.semantic_forward(s["state"], s["ids"][:, :13], kv_cache=c12, **hk)[0], s["logits_inc"])
    assert close(ce(lg, s["labels"]), s["loss"], 1e-5)

    c = g["coarse"]
    hk = dict(heads=2, depth=2, codebook_size=64, num_coarse_quantizers=3)
    (sl, cl), _ = ot.coarse_forward(c["state"], c["sem"], c["coarse"], **hk)
    assert close(sl, c["sem_logits"]) and close(cl, c["coarse_logits"])
    _, (kv_a, emb_a) = ot.coarse_forward(c["state"], c["sem"], c["coarse"][:, :9], return_only_coarse_logits=True, **hk)
    (_, cl_b), _ = ot.coarse_forward(c["state"], c["sem"], c["coarse"][:, :10], kv_cache=kv_a, embed_cache=emb_a,
                                     return_only_coarse_logits=True, **hk)
    assert close(cl_b, c["coarse_logits_b"])

    f = g["fine"]
    hk = dict(heads=2, depth=2, codebook_size=64, num_coarse_quantizers=3, num_fine_quantizers=5)
    (cl, fl), _ = ot.fine_forward(f["state"], f["coarse"], f["fine"], **hk)
    assert close(cl, f["coarse_logits"]) and close(fl, f["fine_logits"])
    _, (kv_a, emb_a) = ot.fine_forward(f["state"], f["coarse"], f["fine"][:, :7], return_only_fine_logits=True, **hk)
    (_, fl_b), _ = ot.fine_forward(f["state"], f["coarse"], f["fine"][:, :8], kv_cache=kv_a, embed_cache=emb_a,
                                   return_only_fine_logits=True, **hk)
    assert close(fl_b, f["fine_logits_b"])
    assert close(ce(cl, f["c_labels"]) + ce(fl, f["f_labels"]), f["loss"], 1e-5)


def test_relative_position_bias_grads():
    """oracle autograd reproduces the reference's gradients of the bias parameters."""
    import torch.nn.functional as F

    g = load("relpos.pt")["coarse"]
    st = {k: v.clone().requires_grad_(v.is_floating_point()) for k, v in g["state"].items()}
    (sl, cl), _ = ot.coarse_forward(st, g["sem"], g["coarse"], heads=2, depth=2, codebook_size=64,
                                    num_coarse_quantizers=3)
    loss = F.cross_entropy(sl.transpose(1, 2), g["sem_labels"]) + F.cross_entropy(cl.transpose(1, 2), g["coarse_labels"])
    loss.backward()
    for k in ("cross_attn_bias", "transformer.rel_pos_bias.net.0.0.weight", "transformer.rel_pos_bias.net.2.0.weight",
              "transformer.rel_pos_bias.net.3.bias"):
        assert close(st[k].grad, g["grads"][k], 1e-3), k
