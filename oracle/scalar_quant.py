"""Oracle restatement of vector-quantize-pytorch's GroupedResidualFSQ / GroupedResidualLFQ (TEST INFRASTRUCTURE — never
imported by the product), eval path only.

PARITY UNPINNED: like the residual VQ in oracle/third_party.py, the package is declared in /root/reference/setup.py but
its source is absent and not installable offline.  These classes restate the published algorithms (FSQ, arXiv
2309.15505; LFQ, arXiv 2310.05737) with the constructor kwargs the reference passes (soundstream.py:561-587) and the
upstream state_dict keys (`rvqs.{g}.project_in.*`, `rvqs.{g}.project_out.*`; levels, basis, scales and masks are
non-persistent buffers).  They follow the formulas below; some upstream revisions of ResidualFSQ also bound the input
before the first stage, which this restatement does not do.

  r = project_in(x) (Linear(Dg, dc) with bias, identity when Dg == dc), acc = 0
  for q < Q: c = stage_q(r); r = r - c; acc = acc + c
  quantized = project_out(acc)
  FSQ stage: c = FSQ(r / scale_q) * scale_q, scale_q = (L - 1) ** -q;
             FSQ(z) = round(tanh(z + shift) * half_l - offset) / (L // 2), half_l = (L - 1) * (1 + 1e-3) / 2,
             offset = 0.5 for even L else 0, shift = atanh(offset / half_l); index = sum_j (z'_j + L_j // 2) basis_j.
  LFQ stage: c = where(r > 0, 2 ** -q, -2 ** -q); index = sum_j [r_j > 0] 2 ** (dc - 1 - j).

oracle/make_golden_quantizers.py puts these classes under the reference's soundstream.py.  `residual_sq_fp64` restates
the same arithmetic in fp64 with the margins the GPU tests use to decide which rows must match bit for bit.
"""
from __future__ import annotations

import math

import torch
from torch import nn

from . import codec as oc
from .transformer import sub


def fsq_buffers(levels, num_quantizers):
    """(levels int32, basis int32, half_l, offset, shift, scales [Q, dc]) in fp32 as the upstream modules build them"""
    lv = torch.tensor(levels, dtype=torch.int32)
    basis = torch.cumprod(torch.tensor([1] + list(levels[:-1])), dim=0, dtype=torch.int32)
    half_l = (lv - 1) * (1 + 1e-3) / 2
    offset = torch.where(lv % 2 == 0, 0.5, 0.0)
    shift = (offset / half_l).atanh()
    levels_tensor = torch.Tensor(levels)
    scales = torch.stack([(levels_tensor - 1) ** -q for q in range(num_quantizers)])
    return lv, basis, half_l, offset, shift, scales


class _Projected(nn.Module):
    def __init__(self, dim, codebook_dim):
        super().__init__()
        proj = dim != codebook_dim
        self.project_in = nn.Linear(dim, codebook_dim) if proj else nn.Identity()
        self.project_out = nn.Linear(codebook_dim, dim) if proj else nn.Identity()

    def _pad(self, indices):
        """indices [..., q'] -> [..., Q] with -1 for the missing stages, and the mask of dropped entries"""
        q = indices.shape[-1]
        if q < self.num_quantizers:
            indices = torch.nn.functional.pad(indices, (0, self.num_quantizers - q), value=-1)
        return indices, indices < 0

    def get_output_from_indices(self, indices):
        indices, dropped = self._pad(indices)
        acc = 0.0
        for q in range(self.num_quantizers):
            code = self.codes_of(indices[..., q].clamp(min=0), q).masked_fill(dropped[..., q, None], 0.0)
            acc = acc + code
        return self.project_out(acc)


class ResidualFSQ(_Projected):
    def __init__(self, *, dim, levels, num_quantizers, **_):
        super().__init__(dim, len(levels))
        self.num_quantizers = num_quantizers
        self.codebook_size = math.prod(levels)
        lv, basis, half_l, offset, shift, scales = fsq_buffers(levels, num_quantizers)
        for name, t in dict(_levels=lv, _basis=basis, half_l=half_l, offset=offset, shift=shift, scales=scales).items():
            self.register_buffer(name, t, persistent=False)

    def forward(self, x):
        assert not self.training, "oracle FSQ restates the eval path only"
        r = self.project_in(x).float()
        hw = self._levels // 2
        acc, idxs = 0.0, []
        for scale in self.scales:
            zq = ((r / scale + self.shift).tanh() * self.half_l - self.offset).round()   # half to even
            c = (zq / hw) * scale
            r = r - c
            acc = acc + c
            idxs.append(((zq.long() + hw) * self._basis).sum(dim=-1).to(torch.int32))   # integer, exact below 2^31
        return self.project_out(acc), torch.stack(idxs, dim=-1)

    def codes_of(self, idx, q):
        hw = self._levels // 2
        zq = (idx[..., None] // self._basis) % self._levels - hw
        return (zq / hw) * self.scales[q]


class ResidualLFQ(_Projected):
    def __init__(self, *, dim, num_quantizers, codebook_size, **_):
        dc = int(math.log2(codebook_size))
        assert 2 ** dc == codebook_size
        super().__init__(dim, dc)
        self.num_quantizers = num_quantizers
        self.codebook_size = codebook_size
        self.scales = [2.0 ** -q for q in range(num_quantizers)]
        self.register_buffer("mask", 2 ** torch.arange(dc - 1, -1, -1), persistent=False)

    def forward(self, x):
        assert not self.training, "oracle LFQ restates the eval path only"
        r = self.project_in(x).float()
        acc, idxs = 0.0, []
        for scale in self.scales:
            c = torch.where(r > 0, torch.ones_like(r) * scale, -torch.ones_like(r) * scale)
            idxs.append(((r > 0).long() * self.mask).sum(dim=-1))
            r = r - c
            acc = acc + c
        return self.project_out(acc), torch.stack(idxs, dim=-1), torch.zeros(self.num_quantizers)

    def codes_of(self, idx, q):
        bits = ((idx[..., None] & self.mask) != 0).float()
        return bits * self.scales[q] * 2 - self.scales[q]


class _Grouped(nn.Module):
    residual_cls = None

    def __init__(self, *, dim, groups=1, **kwargs):
        super().__init__()
        assert dim % groups == 0
        self.groups = groups
        self.kwargs = dict(dim=dim, groups=groups, **kwargs)
        self.rvqs = nn.ModuleList([self.residual_cls(dim=dim // groups, **kwargs) for _ in range(groups)])
        self.codebook_size = self.rvqs[0].codebook_size

    def _outs(self, x):
        return [rvq(c) for rvq, c in zip(self.rvqs, x.chunk(self.groups, dim=-1))]

    def get_output_from_indices(self, indices):  # g b n q'
        return torch.cat([rvq.get_output_from_indices(i) for rvq, i in zip(self.rvqs, indices)], dim=-1)


class GroupedResidualFSQ(_Grouped):
    residual_cls = ResidualFSQ

    def forward(self, x):
        outs = self._outs(x)
        return torch.cat([o[0] for o in outs], dim=-1), torch.stack([o[1] for o in outs])


class GroupedResidualLFQ(_Grouped):
    residual_cls = ResidualLFQ

    def forward(self, x):
        outs = self._outs(x)
        return (torch.cat([o[0] for o in outs], dim=-1), torch.stack([o[1] for o in outs]),
                torch.stack([o[2] for o in outs]))


def register(ref):
    """run the reference's soundstream.py on these restatements instead of oracle/ref_import.py's placeholders"""
    ref.ss.GroupedResidualFSQ = GroupedResidualFSQ
    ref.ss.GroupedResidualLFQ = GroupedResidualLFQ


def build_rq(kwargs, rq_state):
    """the grouped quantizer of SoundStream(**kwargs) with the state `rq.*` (prefix stripped) loaded strictly"""
    common = dict(dim=kwargs.get("codebook_dim", 512), num_quantizers=kwargs.get("rq_num_quantizers", 8),
                  groups=kwargs.get("rq_groups", 1))
    if kwargs.get("use_finite_scalar_quantizer"):
        rq = GroupedResidualFSQ(levels=kwargs["finite_scalar_quantizer_levels"], **common)
    else:
        rq = GroupedResidualLFQ(codebook_size=kwargs["codebook_size"], **common)
    rq.load_state_dict(rq_state, strict=True)
    return rq.eval()


def soundstream_tokenize(kwargs, st, wave):
    """SoundStream.forward(..., return_encoded=True) without local attention on the functional codec oracle:
    wave [b, T] -> (encoder output [b, n, D], quantized [b, n, D], indices [g, b, n, q])"""
    x = oc.encoder(sub(st, "encoder"), wave[:, None, :]).transpose(1, 2)
    with torch.no_grad():
        out = build_rq(kwargs, sub(st, "rq"))(x)
    return x, out[0], out[1]


def soundstream_decode_indices(kwargs, st, indices):
    """decode_from_codebook_indices: indices [g, b, n, q'] -> wave [b, 1, T]"""
    with torch.no_grad():
        x = build_rq(kwargs, sub(st, "rq")).get_output_from_indices(indices)
    return oc.decoder(sub(st, "decoder"), x.transpose(1, 2))


def residual_sq_fp64(x, *, mode, groups, levels=None, codebook_dim=None, num_quantizers, weights=None,
                     fp32_projection_error=0.0):
    """the quantizer arithmetic in fp64, for testing the fp32 kernels.

    x [N, groups * Dg]; weights = (w_in [g, dc, Dg], b_in [g, dc], w_out [g, Dg, dc], b_out [g, Dg]) or None (identity).
    The stage constants are the fp32 ones (fsq_buffers) widened, so the rounding boundaries are the kernel's.
    Returns (quantized fp64 [N, D], indices int64 [g, N, Q], margin [g, N, Q]): margin[..., q] is, over stages 0..q and
    all dimensions, the smallest distance of a decision (FSQ pre-round value from its nearest .5 boundary; LFQ stage
    input from 0) to its boundary, divided by a bound on how far an fp32 evaluation can move that value.  Where
    margin[..., q] > 1, any fp32 evaluation whose project_in error is below `fp32_projection_error` (absolute) must
    produce the same indices for stages 0..q."""
    x = x.double()
    N, D = x.shape
    Dg = D // groups
    Q = num_quantizers
    if mode == "fsq":
        lv, basis, half_l, offset, shift, scales = (t.double() for t in fsq_buffers(levels, Q))
        hw = torch.div(lv, 2, rounding_mode="floor")
        dc = len(levels)
    else:
        dc = codebook_dim
        basis = (2 ** torch.arange(dc - 1, -1, -1)).double()
        scales = torch.tensor([2.0 ** -q for q in range(Q)], dtype=torch.float64)[:, None].expand(Q, dc)
    eps = 2.0 ** -23
    quant, idx, margin = [], [], []
    for g in range(groups):
        xg = x[:, g * Dg:(g + 1) * Dg]
        if weights is None:
            r = xg.clone()
            err = torch.zeros_like(r)
        else:
            w_in, b_in = weights[0][g].double(), weights[1][g].double()
            r = xg @ w_in.t() + b_in
            err = torch.full_like(r, fp32_projection_error)
        acc = torch.zeros_like(r)
        rmax = r.abs().amax(dim=-1, keepdim=True)
        m = torch.full((N,), float("inf"), dtype=torch.float64)
        ids, ms = [], []
        for q in range(Q):
            s = scales[q]
            # fp32 error of r at this stage: the projection's, plus one rounding per earlier stage (|r| <= rmax)
            dr = err + 2 * eps * rmax * (q + 1)
            if mode == "fsq":
                z = r / s
                v = torch.tanh(z + shift) * half_l - offset
                dv = half_l * (dr / s + 2 * eps * (z.abs() + shift.abs())) + 2 * eps * (v.abs() + half_l)
                m = torch.minimum(m, ((v - v.floor() - 0.5).abs() / dv).amin(dim=-1))
                zq = torch.round(v)
                c = zq / hw * s
                ids.append(((zq + hw) * basis).sum(-1).round().long())
            else:
                m = torch.minimum(m, (r.abs() / (dr + 1e-300)).amin(dim=-1))
                c = torch.where(r > 0, s, -s).expand_as(r)
                ids.append(((r > 0).double() * basis).sum(-1).long())
            ms.append(m)
            r = r - c
            acc = acc + c
        quant.append(acc if weights is None else acc @ weights[2][g].double().t() + weights[3][g].double())
        idx.append(torch.stack(ids, dim=-1))
        margin.append(torch.stack(ms, dim=-1))
    return torch.cat(quant, dim=-1), torch.stack(idx), torch.stack(margin)


def decode_fp64(indices, *, mode, levels=None, codebook_dim=None, num_quantizers, weights=None):
    """get_output_from_indices in fp64: indices [g, N, q'] (-1 dropped, missing stages dropped) -> [N, g * Dg]"""
    Q = num_quantizers
    if mode == "fsq":
        lv, basis, _, _, _, scales = fsq_buffers(levels, Q)
        lv, basis, scales = lv.long(), basis.long(), scales.double()
        hw = lv // 2
    else:
        dc = codebook_dim
        basis = 2 ** torch.arange(dc - 1, -1, -1)
        scales = torch.tensor([2.0 ** -q for q in range(Q)], dtype=torch.float64)[:, None].expand(Q, dc)
    outs = []
    for g in range(indices.shape[0]):
        ids = indices[g].long()
        acc = torch.zeros(ids.shape[0], basis.numel(), dtype=torch.float64)
        for q in range(ids.shape[-1]):
            i = ids[:, q, None].clamp(min=0)
            if mode == "fsq":
                code = ((i // basis) % lv - hw).double() / hw * scales[q]
            else:
                code = torch.where((i // basis) % 2 == 1, scales[q], -scales[q])
            acc = acc + code.masked_fill(ids[:, q, None] < 0, 0.0)
        if weights is not None:
            acc = acc @ weights[2][g].double().t() + weights[3][g].double()
        outs.append(acc)
    return torch.cat(outs, dim=-1)
