"""Generate tests/golden/dim_head.pt from the REAL reference (oracle/ref_import.py) - build container only.

    python -m oracle.make_golden_dim_head

For dim_head in {32, 128} and the small Semantic, Coarse and Fine transformers: with flash_attn=True the reference
state_dict, seeded inputs, logits, the wrapper's training loss and every parameter gradient; with flash_attn=False
(relative-position, cross and 2-D biases) the extra bias parameters and the logits.  Plus one `Transformer` forward
with kv_cache against the full forward (the semantic flash_attn=False model's stack).  The other fixtures (oracle/make_golden.py) are not touched.

To keep the file in one piece (under golden.PART_BYTES) the models are tiny (dim 32; depth 2 and 2 heads for the semantic
model, whose second layer exercises the value residual, depth 1 and 1 head for the other two) and every parameter is rounded to a
bf16-representable value BEFORE the reference runs, so that weights and gradients are stored as bf16: the weights
without loss, the gradients with 2^-9 relative rounding, far inside the tests' gradient tolerance."""
from __future__ import annotations

import random
import sys
import warnings

import torch

from . import golden, ref_import
from .make_golden import bf16_noise, perturb

NAME = "dim_head.pt"
WIDTHS = (32, 128)


def _round_bf16(m):
    with torch.no_grad():
        for p in m.parameters():
            p.copy_(p.to(torch.bfloat16).float())
    return m


def _bias_perturb(m, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in m.named_parameters():
            if name in ("cross_attn_bias", "null_pos_bias"):
                p.copy_(torch.randn(p.shape, generator=g) * 0.5)
            elif "rel_pos_bias" in name or "pos_bias_mlp" in name:
                p.add_(torch.randn(p.shape, generator=g) * 0.05)


UNUSED = ("proj_text_embed.weight",)   # [dim, 768] of the text conditioning, which these models do not run


def _pack(d):
    """a dict of tensors as one flat bf16 tensor plus names and shapes (a zip entry per tensor would cost more than
    the tiny tensors themselves); `unpack` in the tests is the inverse.  Integer buffers are kept as they are.  The
    values of UNUSED entries are left out (name and shape stay): they unpack as zeros."""
    fl = {k: v.detach() for k, v in d.items() if v.is_floating_point()}
    vals = [v.reshape(-1) for k, v in fl.items() if k not in UNUSED]
    return dict(names=list(fl), shapes=[tuple(v.shape) for v in fl.values()], unused=[k for k in fl if k in UNUSED],
                flat=torch.cat(vals).to(torch.bfloat16) if vals else torch.empty(0),
                other={k: v.detach().clone() for k, v in d.items() if not v.is_floating_point()})


def _grads(m):
    return {k: p.grad.detach().clone() for k, p in m.named_parameters() if p.grad is not None}


def _math_twin(cls, kw, m, seed):
    """the flash_attn=False model over the same weights: returns (module, its extra (bias) parameters)"""
    mm = cls(**{**kw, "flash_attn": False}).eval()
    missing = mm.load_state_dict(m.state_dict(), strict=False).missing_keys
    _bias_perturb(mm, seed)
    _round_bf16(mm)
    return mm, {k: v for k, v in mm.state_dict().items() if k in missing}


def _semantic(ref, D, seed):
    torch.manual_seed(seed)
    kw = dict(num_semantic_tokens=20, dim=32, depth=2, heads=2, dim_head=D, flash_attn=True)
    m = ref.lm.SemanticTransformer(**kw).eval()
    perturb(m, seed + 1)
    _round_bf16(m)
    ids = torch.randint(0, 20, (2, 17))
    with torch.no_grad():
        logits = m(ids=ids)
    mm, extra = _math_twin(ref.lm.SemanticTransformer, kw, m, seed + 2)
    with torch.no_grad():
        logits_math = mm(ids=ids)
    w = ref.lm.SemanticTransformerWrapper(transformer=m, unique_consecutive=False, mask_prob=0.0).train()
    loss = w(semantic_token_ids=ids, return_loss=True)
    loss.backward()
    gr = _grads(m)
    noise = bf16_noise(m, lambda: w(semantic_token_ids=ids, return_loss=True), gr)
    return dict(kwargs=kw, state=_pack(m.state_dict()), math_extra=_pack(extra), ids=ids, logits=logits,
                logits_math=logits_math, loss=loss.detach(), grads=_pack(gr), bf16_noise=noise,
                transformer=_kv_cache(mm, D, seed + 3))


def _coarse(ref, D, seed):
    torch.manual_seed(seed)
    kw = dict(num_semantic_tokens=20, codebook_size=16, num_coarse_quantizers=3, dim=32, depth=1, heads=1, dim_head=D,
              flash_attn=True)
    m = ref.lm.CoarseTransformer(**kw).eval()
    perturb(m, seed + 1)
    _round_bf16(m)
    sem = torch.randint(0, 20, (2, 7))
    coarse = torch.randint(0, 16, (2, 13))     # 4 frames * 3 + 1: the remainder head path
    with torch.no_grad():
        sl, cl = m(semantic_token_ids=sem, coarse_token_ids=coarse)
    mm, extra = _math_twin(ref.lm.CoarseTransformer, kw, m, seed + 2)
    with torch.no_grad():
        slm, clm = mm(semantic_token_ids=sem, coarse_token_ids=coarse)
    ss = ref.ss.SoundStream(codebook_size=16, rq_num_quantizers=8, channels=4, use_local_attn=False, codebook_dim=32)
    w = ref.lm.CoarseTransformerWrapper(transformer=m, codec=ss, unique_consecutive=False, mask_prob=0.0).train()
    frames = coarse[:, :12]
    loss = w(semantic_token_ids=sem, coarse_token_ids=frames, return_loss=True)
    loss.backward()
    gr = _grads(m)
    noise = bf16_noise(m, lambda: w(semantic_token_ids=sem, coarse_token_ids=frames, return_loss=True), gr)
    return dict(kwargs=kw, state=_pack(m.state_dict()), math_extra=_pack(extra), sem=sem, coarse=coarse, sem_logits=sl,
                coarse_logits=cl, sem_logits_math=slm, coarse_logits_math=clm, loss=loss.detach(), grads=_pack(gr),
                bf16_noise=noise)


def _fine(ref, D, seed):
    torch.manual_seed(seed)
    kw = dict(num_coarse_quantizers=2, num_fine_quantizers=3, codebook_size=16, dim=32, depth=1, heads=1, dim_head=D,
              flash_attn=True)
    m = ref.lm.FineTransformer(**kw).eval()
    perturb(m, seed + 1)
    _round_bf16(m)
    coarse = torch.randint(0, 16, (2, 4, 2))
    fine = torch.randint(0, 16, (2, 4, 3))
    c2, f2 = coarse.reshape(2, -1), fine.reshape(2, -1)[:, :-1]
    with torch.no_grad():
        cl, fl = m(coarse_token_ids=c2, fine_token_ids=f2)
    mm, extra = _math_twin(ref.lm.FineTransformer, kw, m, seed + 2)
    with torch.no_grad():
        clm, flm = mm(coarse_token_ids=c2, fine_token_ids=f2)
    ss = ref.ss.SoundStream(codebook_size=16, rq_num_quantizers=5, channels=4, use_local_attn=False, codebook_dim=32)
    w = ref.lm.FineTransformerWrapper(transformer=m, codec=ss, mask_prob=0.0).train()
    loss = w(coarse_token_ids=coarse, fine_token_ids=fine, return_loss=True)
    loss.backward()
    gr = _grads(m)
    noise = bf16_noise(m, lambda: w(coarse_token_ids=coarse, fine_token_ids=fine, return_loss=True), gr)
    return dict(kwargs=kw, state=_pack(m.state_dict()), math_extra=_pack(extra), coarse=coarse, fine=fine,
                coarse_logits=cl, fine_logits=fl, coarse_logits_math=clm, fine_logits_math=flm, loss=loss.detach(),
                grads=_pack(gr), bf16_noise=noise)


def _kv_cache(mm, D, seed):
    """the bare Transformer of the semantic model's flash_attn=False twin (the reference's flash path aligns a cached
    query top-left, see golden_semantic in make_golden.py; no state of its own is stored): 9 positions, then all 14
    with the cache, against the full forward"""
    torch.manual_seed(seed)
    t = mm.transformer
    x = torch.randn(2, 14, 32).to(torch.bfloat16).float()
    with torch.no_grad():
        full = t(x)
        _, cache = t(x[:, :9], return_kv_cache=True)
        inc, cache2 = t(x, kv_cache=cache, return_kv_cache=True)
    assert cache.shape == (2, 2, 2, 9, D) and cache2.shape == (2, 2, 2, 14, D)   # [depth, k | v, b, n, dim_head]
    assert torch.allclose(inc, full[:, 9:], atol=1e-4), "reference: cached forward != full forward"
    return dict(x=x, out=full, out_inc=inc, cache9=cache)


def main():
    ref = ref_import.load()
    out = {}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for D in WIDTHS:
            random.seed(20240607 + D)   # hyper-connections picks its initial stream with `random.randrange`
            out[D] = dict(semantic=_semantic(ref, D, 100 + D), coarse=_coarse(ref, D, 200 + D),
                          fine=_fine(ref, D, 300 + D))
    golden.save(out, NAME)
    size = sum(p.stat().st_size for p in golden.GOLDEN.glob(NAME + "*"))
    print(f"wrote {NAME}: {size / 1e6:.2f} MB")
    assert (golden.GOLDEN / NAME).exists(), "the fixture must stay in one piece"


if __name__ == "__main__":
    sys.exit(main())
