#!/usr/bin/env python
"""Generate tests/golden/streams.pt: models with 2, 3 and 8 hyper-connection residual streams, from the REAL reference
(oracle/ref_import.py, on top of the oracle's hyper-connections restatement) — build container only.

    python tools/make_golden_streams.py

Per model it stores the constructor kwargs, the reference's state_dict, seeded inputs, logits with and without a key
mask, the wrapper loss, the parameter gradients and the reference's own bf16-autocast noise (of the gradients and, for
the Semantic models, of the logits), and it checks that
the functional oracle (oracle/transformer.py) reproduces the logits and the loss.  The other fixtures are untouched.
"""
import random
import sys
import warnings
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from oracle import golden, ref_import  # noqa: E402
from oracle import transformer as ot  # noqa: E402
from oracle.make_golden import bf16_noise, check, clone_state, perturb, rms_rel  # noqa: E402


def semantic(ref, S, seed):
    torch.manual_seed(seed)
    kw = dict(num_semantic_tokens=50, dim=64, depth=2, heads=2, flash_attn=True, num_residual_streams=S)
    m = ref.lm.SemanticTransformer(**kw).eval()
    perturb(m, seed)
    ids = torch.randint(0, 50, (2, 19))
    mask = ot.fcm_mask((2, 19), 0.15, torch.Generator().manual_seed(seed))
    with torch.no_grad():
        logits = m(ids=ids)
        logits_masked = m(ids=ids, self_attn_mask=mask)
    with torch.no_grad(), torch.autocast("cpu", dtype=torch.bfloat16):  # the reference's own bf16-autocast logits
        logits_bf16_noise = (rms_rel(m(ids=ids), logits), rms_rel(m(ids=ids, self_attn_mask=mask), logits_masked))
    st = clone_state(m)
    print(f"semantic ({S} residual streams): logits bf16 noise {logits_bf16_noise}")
    hk = dict(heads=2, depth=2, num_streams=S)
    check("logits", ot.semantic_forward(st, ids, **hk)[0], logits)
    check("logits masked", ot.semantic_forward(st, ids, self_attn_mask=mask, **hk)[0], logits_masked)
    w = ref.lm.SemanticTransformerWrapper(transformer=m, unique_consecutive=False, mask_prob=0.0).train()
    loss = w(semantic_token_ids=ids, return_loss=True)
    loss.backward()
    grads = {k: p.grad.detach().clone() for k, p in m.named_parameters() if p.grad is not None}
    noise = bf16_noise(m, lambda: w(semantic_token_ids=ids, return_loss=True), grads)
    labels = torch.cat((ids, torch.full((2, 1), 50)), dim=1)
    check("wrapper loss", ot.cross_entropy(ot.semantic_forward(st, labels[:, :-1], **hk)[0], labels), loss.detach())
    return dict(kind="semantic", kwargs=kw, state=st, ids=ids, mask=mask, logits=logits, logits_masked=logits_masked,
                loss=loss.detach(), grads=grads, bf16_noise=noise, logits_bf16_noise=logits_bf16_noise)


def coarse(ref, S, seed):
    """flash_attn=False: the relative-position bias (and the cross-segment bias) together with hyper-connections"""
    torch.manual_seed(seed)
    kw = dict(num_semantic_tokens=50, codebook_size=64, num_coarse_quantizers=3, dim=64, depth=2, heads=2,
              flash_attn=False, num_residual_streams=S)
    m = ref.lm.CoarseTransformer(**kw).eval()
    perturb(m, seed)
    sem = torch.randint(0, 50, (2, 10))
    co = torch.randint(0, 64, (2, 22))
    mask = ot.fcm_mask((2, 1 + 10 + 1 + 22), 0.15, torch.Generator().manual_seed(seed))
    with torch.no_grad():
        sl, cl = m(semantic_token_ids=sem, coarse_token_ids=co)
        slm, clm = m(semantic_token_ids=sem, coarse_token_ids=co, self_attn_mask=mask)
    st = clone_state(m)
    print(f"coarse ({S} residual streams, relative-position bias):")
    hk = dict(heads=2, depth=2, codebook_size=64, num_coarse_quantizers=3, num_streams=S)
    (osl, ocl), _ = ot.coarse_forward(st, sem, co, **hk)
    check("semantic logits", osl, sl)
    check("coarse logits", ocl, cl)
    (oslm, oclm), _ = ot.coarse_forward(st, sem, co, self_attn_mask=mask, **hk)
    check("coarse logits masked", oclm, clm)
    ss = ref.ss.SoundStream(codebook_size=64, rq_num_quantizers=8, channels=4, use_local_attn=False, codebook_dim=32)
    w = ref.lm.CoarseTransformerWrapper(transformer=m, codec=ss, unique_consecutive=False, mask_prob=0.0).train()
    frames = co[:, :21]
    loss = w(semantic_token_ids=sem, coarse_token_ids=frames, return_loss=True)
    loss.backward()
    grads = {k: p.grad.detach().clone() for k, p in m.named_parameters() if p.grad is not None}
    noise = bf16_noise(m, lambda: w(semantic_token_ids=sem, coarse_token_ids=frames, return_loss=True), grads)
    return dict(kind="coarse", kwargs=kw, state=st, sem=sem, coarse=co, frames=frames, mask=mask, sem_logits=sl,
                coarse_logits=cl, sem_logits_masked=slm, coarse_logits_masked=clm, loss=loss.detach(), grads=grads,
                bf16_noise=noise)


def main():
    ref = ref_import.load()
    out = {}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for name, fn, S, seed in (("semantic_s2", semantic, 2, 61), ("semantic_s3", semantic, 3, 62),
                                  ("semantic_s8", semantic, 8, 63), ("coarse_s2", coarse, 2, 64)):
            # hyper-connections picks its initial stream with `random.randrange`: seed per model
            random.seed(20240607 + seed)
            out[name] = fn(ref, S, seed)
    golden.save(out, "streams.pt")
    print("wrote streams.pt")


if __name__ == "__main__":
    sys.exit(main())
