"""References for the residual VQ's `rq_kwargs` options (TEST INFRASTRUCTURE — never imported by the product).

PARITY UNPINNED: vector-quantize-pytorch (>= 1.19.3) is absent offline.  `ResidualVQ` / `GroupedResidualVQ` below
extend the eval-path restatement of oracle/third_party.py (same codebook keys, same Euclidean rule, which they reuse)
with the two `rq_kwargs` options that change what eval computes, `use_cosine_sim` and `codebook_dim`, and ignore the
training-only ones.  `register` puts them under the reference's soundstream.py (oracle/make_golden_rvq_options.py):

  r = project_in(x) (Linear(Dg, dc) with bias, identity when dc == Dg); acc = 0
  per stage q: Euclidean  idx = argmin_c |r - e_c|                       (oracle/nearest_code.py)
               cosine     idx = argmax_c F.normalize(r) . e_c, lowest index on ties, e_c the stored row as is
               r = r - e_idx; acc = acc + e_idx
  quantized = project_out(acc); get_output_from_indices = project_out(sum_q e_{q, idx_q}), id -1 contributes 0

Cosine band.  The kernels rank the candidates by r.e_c in fp32 (the ranking of r^.e_c: r^ is r over a positive
scalar).  Any fp32 evaluation of that D-term dot product is within gamma_D sum_d |r_d e_cd| <= gamma_D |r| |e_c| of the
exact value, so the chosen code a and the fp64 argmax b satisfy  t_b - t_a <= gamma_D |r| (|e_a| + |e_b|),  t = r.e in
fp64; where every other code is further than that below the maximum, the id must be the fp64 argmax.  A zero residual
scores 0 everywhere, and F.normalize + argmax pick code 0.

Also: the seeded codec weights of tests/golden/rvq_options.pt (`seeded_state`, regenerated instead of stored: the
tensor-core codec's 9 M parameters would not fit a fixture) and the functional SoundStream with this quantizer.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F
from torch import nn

from . import codec as oc
from . import third_party as tp
from .nearest_code import gamma, replay
from .transformer import sub


# ---- the restated quantizer -------------------------------------------------------------------------------------------
def cosine_nearest(x, embed):
    """x [n, d], embed [c, d] fp32 -> index of the most similar code; ties -> lowest index.

    idx = argmax(F.normalize(x) @ embed^T)   (CosineSimCodebook.forward in eval; the stored rows are not re-normalised)
    """
    return (F.normalize(x.float(), dim=-1) @ embed.float().t()).argmax(dim=-1)


class ResidualVQ(nn.Module):
    """ResidualVQ(dim, codebook_dim=dc, use_cosine_sim): project_in = Linear(dim, dc) and project_out = Linear(dc, dim),
    both with bias and both Identity (no keys) when dc == dim; layers.{q}._codebook.embed [1, C, dc] (the keys of
    oracle/third_party.py).  r = project_in(x); per stage idx = nearest (Euclidean) or most similar (cosine) code,
    r -= e_idx, acc += e_idx; quantized = project_out(acc)."""

    def __init__(self, *, dim, num_quantizers, codebook_size, codebook_dim=None, use_cosine_sim=False, **_):
        super().__init__()
        dc = dim if codebook_dim is None else codebook_dim
        self.project_in = nn.Linear(dim, dc) if dc != dim else nn.Identity()
        self.project_out = nn.Linear(dc, dim) if dc != dim else nn.Identity()
        self.nearest = cosine_nearest if use_cosine_sim else tp.euclid_nearest
        self.layers = nn.ModuleList([tp._VQLayer(dc, codebook_size) for _ in range(num_quantizers)])

    @property
    def codebooks(self):
        return torch.stack([l._codebook.embed[0] for l in self.layers])  # q c d

    def forward(self, x):
        assert not self.training, "oracle RVQ restates the eval path only"
        b, n, d = x.shape
        residual = self.project_in(x.float().reshape(b * n, d))
        out = torch.zeros_like(residual)
        idxs = []
        for cb in self.codebooks:
            idx = self.nearest(residual, cb)
            quant = cb[idx]
            residual = residual - quant
            out = out + quant
            idxs.append(idx)
        indices = torch.stack(idxs, dim=-1).reshape(b, n, -1)
        return self.project_out(out).reshape(b, n, d), indices, torch.zeros(1, len(idxs), device=x.device)

    def get_output_from_indices(self, indices):
        cbs = self.codebooks
        out = 0
        for q in range(indices.shape[-1]):
            idx = indices[..., q]
            out = out + cbs[q][idx.clamp(min=0)].masked_fill((idx < 0)[..., None], 0.0)
        return self.project_out(out)


class GroupedResidualVQ(tp.GroupedResidualVQ):
    """oracle/third_party.py's grouping (channels split into `groups`) over the ResidualVQ above"""

    def __init__(self, *, dim, groups=1, **kwargs):
        nn.Module.__init__(self)
        assert dim % groups == 0
        self.groups = groups
        self.kwargs = dict(dim=dim, groups=groups, **kwargs)
        self.rvqs = nn.ModuleList([ResidualVQ(dim=dim // groups, **kwargs) for _ in range(groups)])


def register(ref):
    """run the reference's soundstream.py on this quantizer instead of oracle/ref_import.py's"""
    ref.ss.GroupedResidualVQ = GroupedResidualVQ


# ---- cosine search against fp64 --------------------------------------------------------------------------------------
def cosine_search_fp64(x, cb):
    """the rule in fp64 on the fp64 residual: -> (quantized fp64, ids int64 [N, Q])"""
    r = x.double()
    quant = torch.zeros_like(r)
    ids = []
    for s in range(cb.shape[0]):
        e = cb[s].double()
        i = (r @ e.T).argmax(1)
        ids.append(i)
        r = r - e[i]
        quant = quant + e[i]
    return quant, torch.stack(ids, 1)


def check_cosine_fp64(x, cb, ids, *, quant=None, label=""):
    """replays the stages with the kernel's ids (fp32 residual, as the kernels update it) and asserts at every stage:
    the chosen code lies within the cosine band of the fp64 maximum, the fp64 argmax is chosen wherever it is isolated
    by the band, code 0 on zero residuals; `quant` (when given) equals the fp32 replay bit for bit.
    -> share of (row, stage) pairs whose maximum is not isolated by the band"""
    D = x.shape[1]
    q, residuals = replay(x, cb, ids)
    if quant is not None:
        assert torch.equal(quant.contiguous().view(torch.int32), q.view(torch.int32)), f"{label}: quantized != replay"
    g = gamma(D)
    near_pairs = 0
    for s, r in enumerate(residuals):
        r64, e64 = r.double(), cb[s].double()
        t = r64 @ e64.T
        rn, en = r64.norm(dim=1, keepdim=True), e64.norm(dim=1)[None]
        err = g * rn * en + 1e-13 * rn * en                    # fp32 dot error of each code, plus fp64's own
        best = t.argmax(1, keepdim=True)
        tb = t.gather(1, best)
        i = ids[:, s:s + 1]
        band = err.gather(1, i) + err.gather(1, best)
        gap = tb - t.gather(1, i)
        bad = gap > band
        assert not bad.any(), (f"{label} stage {s}: {int(bad.sum())} rows chose a code outside the fp32 band, worst "
                               f"gap / band {(gap / band.clamp_min(1e-300)).max().item():.3g}")
        near = ((tb - t) <= err + err.gather(1, best)).sum(1) > 1
        assert torch.equal(i[~near], best[~near]), f"{label} stage {s}: isolated maximum not chosen"
        zero = rn[:, 0] == 0
        assert not i[zero].any(), f"{label} stage {s}: a zero residual must take code 0"
        near_pairs += int(near.sum())
    return near_pairs / (x.shape[0] * cb.shape[0])


def linear_fp64(x, w, b):
    return x.double() @ w.double().T + b.double()


# ---- seeded codec weights and the functional SoundStream ----------------------------------------------------------
def seeded_state(keys, seed):
    """{key: tensor} for [(key, shape)]: weights U(-1, 1) / sqrt(fan in) (the conv default's scale), biases
    U(-0.1, 0.1), drawn in list order from one CPU generator"""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for k, shape in keys:
        u = torch.rand(shape, generator=g) * 2 - 1
        out[k] = u / math.sqrt(math.prod(shape[1:])) if len(shape) > 1 else 0.1 * u
    return out


def build_rq(kwargs, rq_state):
    """the residual VQ of SoundStream(**kwargs) with the state `rq.*` (prefix stripped) loaded strictly"""
    rq = GroupedResidualVQ(dim=kwargs.get("codebook_dim", 512), num_quantizers=kwargs.get("rq_num_quantizers", 8),
                           codebook_size=kwargs["codebook_size"], groups=kwargs.get("rq_groups", 1),
                           **kwargs.get("rq_kwargs", {}))
    rq.load_state_dict(rq_state, strict=True)
    return rq.eval()


def soundstream_tokenize(kwargs, st, wave):
    """wave [b, T] -> (encoder output [b, n, D], quantized [b, n, D], indices [g, b, n, q])"""
    x = oc.encoder(sub(st, "encoder"), wave[:, None, :]).transpose(1, 2)
    with torch.no_grad():
        out = build_rq(kwargs, sub(st, "rq"))(x)
    return x, out[0], out[1]


def soundstream_decode_indices(kwargs, st, indices):
    """decode_from_codebook_indices: indices [g, b, n, q'] -> wave [b, 1, T]"""
    with torch.no_grad():
        x = build_rq(kwargs, sub(st, "rq")).get_output_from_indices(indices)
    return oc.decoder(sub(st, "decoder"), x.transpose(1, 2))

