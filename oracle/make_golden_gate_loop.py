"""Generate tests/golden/gate_loop.pt from the REAL reference (oracle/ref_import.py) - build container only.

    python -m oracle.make_golden_gate_loop

`SoundStream(use_gate_loop_layers=True)` (soundstream.py:29, 314-330, 524-525, 620-621) on a small seeded model (channels
4, no local attention), with the reference's `GateLoop` bound to the restatement oracle.codec_gate_loop.SimpleGateLoopLayer
(gateloop-transformer is not available offline; its parity is unpinned).  Records the reference's encoder / decoder / rq
key list with shapes for this model and, names and shapes only, for the C1 layout (channels 32); the state_dict; a
wave, the encoder output, quantized frames, code indices and both reconstructions.  The gate-loop weights are moved
off their init so the gates spread over (0, 1) and some channels pass sigmoid(a) > 0.95.  The run asserts that
oracle/codec_gate_loop.py reproduces the reference to fp32 round-off and the code indices exactly.
"""
from __future__ import annotations

import math
import random
import sys
import warnings

import torch

from . import codec_gate_loop as ogl
from . import golden, ref_import
from . import third_party as tp
from .make_golden import check, clone_state
from .transformer import sub

NAME = "gate_loop.pt"
PARTS = ("encoder", "decoder", "rq")


def _keys(ss):
    return [(k, tuple(v.shape)) for k, v in ss.state_dict().items() if k.split(".")[0] in PARTS]


def gate_values(ss, wave):
    """sigmoid(a) of every gate-loop layer on the way through encode and decode"""
    seen = []

    def hook(mod, args):
        x = args[0]
        xn = torch.nn.functional.normalize(x, dim=-1) * math.sqrt(x.shape[-1]) * mod.norm.gamma
        seen.append(torch.sigmoid(xn @ mod.to_qkva[0].weight[2 * x.shape[-1]:].t()).flatten())

    hs = [m.register_forward_pre_hook(hook) for m in ss.modules() if isinstance(m, ogl.SimpleGateLoopLayer)]
    with torch.no_grad():
        ss(wave, return_recons_only=True)
    for h in hs:
        h.remove()
    return torch.cat(seen)


def gate_loop_model(ref):
    torch.manual_seed(91)
    kw = dict(codebook_size=64, rq_num_quantizers=4, channels=4, use_local_attn=False, codebook_dim=32,
              target_sample_hz=24000, use_gate_loop_layers=True)
    ss = ref.ss.SoundStream(**kw).eval()
    tp.seed_codebooks(ss.rq, seed=7, std=0.5)
    g = torch.Generator().manual_seed(92)
    with torch.no_grad():
        for n_, p_ in ss.named_parameters():
            if n_.endswith("fn.fn.norm.gamma"):
                p_.copy_(1 + 0.3 * torch.randn(p_.shape, generator=g))
            elif n_.endswith("fn.fn.to_qkva.0.weight"):
                C = p_.shape[1]
                p_.copy_(torch.randn(p_.shape, generator=g) / math.sqrt(C))
                p_[2 * C:] *= 2.0   # a = W_a x^ ~ N(0, 4 gamma^2): gates over (0, 1), a few percent above 0.95
    wave = torch.randn(2, 3200)
    with torch.no_grad():
        enc = ss.encoder(wave[:, None, :])
        quant, idx, _ = ss(wave, return_encoded=True)
        recon = ss(wave, return_recons_only=True)
        recon_idx = ss.decode_from_codebook_indices(idx)
    st = {k: v for k, v in clone_state(ss).items() if k.split(".")[0] in PARTS}
    keys = _keys(ss)
    assert ("encoder.2.fn.fn.norm.gamma", (8,)) in keys and ("encoder.2.fn.fn.to_qkva.0.weight", (24, 8)) in keys
    print("gate loops (channels 4):")
    check("encoder", ogl.encoder(sub(st, "encoder"), wave[:, None, :]), enc)
    oq, oi = ogl.soundstream_tokenize(st, wave)
    assert torch.equal(oi, idx), "rvq indices differ"
    print("  [ok] rvq indices bit-exact")
    check("quantized", oq, quant)
    check("decode from indices", ogl.soundstream_decode_indices(st, idx), recon_idx)
    check("round trip (README.md:100-113)", recon_idx, recon, tol=1e-5)
    gates = gate_values(ss, wave)
    frac = (gates > 0.95).float().mean().item()
    assert frac > 0.005 and (gates < 0.05).any(), "perturbation left the gates near their init"
    print(f"  gates: {100 * frac:.1f} % above 0.95, range [{gates.min():.3f}, {gates.max():.3f}]")
    return dict(kwargs=kw, state=st, keys=keys, wave=wave, enc=enc, quant=quant, idx=idx, recon=recon,
                recon_idx=recon_idx)


def c1_keys(ref):
    ss = ref.ss.SoundStream(codebook_size=1024, use_gate_loop_layers=True, use_local_attn=False)
    return _keys(ss)


def main():
    ref = ref_import.load()
    ref.ss.GateLoop = ogl.SimpleGateLoopLayer   # the name soundstream.py:29 binds; looked up at construction
    random.seed(20240607)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        out = dict(small=gate_loop_model(ref), c1=dict(kwargs=dict(codebook_size=1024, use_gate_loop_layers=True,
                                                                   use_local_attn=False), keys=c1_keys(ref)))
    golden.save(out, NAME)
    size = sum(p.stat().st_size for p in golden.GOLDEN.glob(NAME + "*"))
    print(f"wrote {NAME}: {size / 1e6:.2f} MB")


if __name__ == "__main__":
    sys.exit(main())
