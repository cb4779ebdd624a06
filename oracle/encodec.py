"""The 24 kHz EnCodec (encodec 0.1.1's `EncodecModel.encodec_model_24khz()` with normalize=False) in fp64, restated from
its description: SEANet encoder and decoder with causal weight-normalised convs and reflect padding, a 2-layer LSTM
block with a skip, and a residual VQ of 32 codebooks of 1024 x 128.  The state dict uses encodec's own key names.

`random_state(seed)` builds a full-size seeded state (about 15 M parameters) on the CPU generator; the codebooks are
drawn from the random encoder's outputs on noise, so nearest-code margins are not degenerate.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

f64 = torch.float64

RATIOS = (2, 4, 5, 8)            # encoder strides; the decoder runs them reversed
CHANNELS = (32, 64, 128, 256)    # resnet-block widths, encoder order
H = 512                          # LSTM width = last encoder width
DIM = 128                        # codebook dim
N_CODEBOOKS, CODEBOOK_SIZE = 32, 1024
HOP = math.prod(RATIOS)          # 320 samples per frame
BANDWIDTHS = {1.5: 2, 3.0: 4, 6.0: 8, 12.0: 16, 24.0: 32}
ENC_RES, ENC_DOWN, ENC_LSTM, ENC_LAST = (1, 4, 7, 10), (3, 6, 9, 12), 13, 15
DEC_FIRST, DEC_LSTM, DEC_UP, DEC_RES, DEC_LAST = 0, 1, (3, 6, 9, 12), (4, 7, 10, 13), 15


def n_frames(T):
    return -(-T // HOP)


def conv_specs():
    """(key prefix, kind, Cin, Cout, K) of every weight-normalised conv; kind 'conv' or 'convtr'."""
    out = [("encoder.model.0.conv.conv", "conv", 1, 32, 7)]
    for i, (c, s) in enumerate(zip(CHANNELS, RATIOS)):
        r = f"encoder.model.{ENC_RES[i]}"
        out += [(f"{r}.block.1.conv.conv", "conv", c, c // 2, 3), (f"{r}.block.3.conv.conv", "conv", c // 2, c, 1),
                (f"{r}.shortcut.conv.conv", "conv", c, c, 1),
                (f"encoder.model.{ENC_DOWN[i]}.conv.conv", "conv", c, 2 * c, 2 * s)]
    out.append((f"encoder.model.{ENC_LAST}.conv.conv", "conv", H, DIM, 7))
    out.append((f"decoder.model.{DEC_FIRST}.conv.conv", "conv", DIM, H, 7))
    for i, (c, s) in enumerate(zip(reversed(CHANNELS), reversed(RATIOS))):
        r = f"decoder.model.{DEC_RES[i]}"
        out += [(f"decoder.model.{DEC_UP[i]}.convtr.convtr", "convtr", 2 * c, c, 2 * s),
                (f"{r}.block.1.conv.conv", "conv", c, c // 2, 3), (f"{r}.block.3.conv.conv", "conv", c // 2, c, 1),
                (f"{r}.shortcut.conv.conv", "conv", c, c, 1)]
    out.append((f"decoder.model.{DEC_LAST}.conv.conv", "conv", 32, 1, 7))
    return out


def state_shapes():
    """every key of the encodec checkpoint -> shape"""
    sh = {}
    for p, kind, ci, co, k in conv_specs():
        if kind == "conv":
            sh[f"{p}.weight_g"], sh[f"{p}.weight_v"] = (co, 1, 1), (co, ci, k)
        else:  # ConvTranspose1d weight [Cin, Cout, K]; weight norm over dim 0 = the input channel
            sh[f"{p}.weight_g"], sh[f"{p}.weight_v"] = (ci, 1, 1), (ci, co, k)
        sh[f"{p}.bias"] = (co,)
    for side, idx in (("encoder", ENC_LSTM), ("decoder", DEC_LSTM)):
        for l in range(2):
            for n, s in (("weight_ih", (4 * H, H)), ("weight_hh", (4 * H, H)), ("bias_ih", (4 * H,)),
                         ("bias_hh", (4 * H,))):
                sh[f"{side}.model.{idx}.lstm.{n}_l{l}"] = s
    for q in range(N_CODEBOOKS):
        p = f"quantizer.vq.layers.{q}._codebook"
        sh[f"{p}.inited"], sh[f"{p}.cluster_size"] = (1,), (CODEBOOK_SIZE,)
        sh[f"{p}.embed"], sh[f"{p}.embed_avg"] = (CODEBOOK_SIZE, DIM), (CODEBOOK_SIZE, DIM)
    return sh


def fold_weight_norm(g, v):
    """torch.nn.utils.weight_norm(dim=0): w = g * v / ||v||, the norm over every dim but 0, in fp64"""
    v = v.to(f64)
    return g.to(f64) * v / v.flatten(1).norm(dim=1).view(-1, *([1] * (v.dim() - 1)))


def pad1d(x, pl, pr):
    """reflect padding as EnCodec does it: a row no longer than the larger pad is zero-extended first"""
    L = x.shape[-1]
    extra = max(pl, pr) - L + 1 if L <= max(pl, pr) else 0
    if extra:
        x = F.pad(x, (0, extra))
    y = F.pad(x, (pl, pr), mode="reflect")
    return y[..., : y.shape[-1] - extra]


def conv(st, p, x, stride=1):
    w = fold_weight_norm(st[f"{p}.weight_g"], st[f"{p}.weight_v"])
    k, L = w.shape[-1], x.shape[-1]
    x = pad1d(x, k - stride, -L % stride)
    return F.conv1d(x, w, st[f"{p}.bias"].to(f64), stride=stride)


def convtr(st, p, x, stride):
    w = fold_weight_norm(st[f"{p}.weight_g"], st[f"{p}.weight_v"])
    y = F.conv_transpose1d(x, w, st[f"{p}.bias"].to(f64), stride=stride)
    return y[..., : y.shape[-1] - stride]  # causal: the whole k - s trim on the right


def resblock(st, p, x):
    h = conv(st, f"{p}.block.1.conv.conv", F.elu(x))
    h = conv(st, f"{p}.block.3.conv.conv", F.elu(h))
    return conv(st, f"{p}.shortcut.conv.conv", x) + h


def lstm_block(st, p, x):
    """y = LSTM2(LSTM1(x)) + x, x [B, H, T]; gates i, f, g, o; zero initial state"""
    seq = x.permute(2, 0, 1)
    for l in range(2):
        wi, wh = st[f"{p}.lstm.weight_ih_l{l}"].to(f64), st[f"{p}.lstm.weight_hh_l{l}"].to(f64)
        b = st[f"{p}.lstm.bias_ih_l{l}"].to(f64) + st[f"{p}.lstm.bias_hh_l{l}"].to(f64)
        xp = seq @ wi.T + b
        h = torch.zeros(seq.shape[1], H, dtype=f64, device=x.device)
        c = torch.zeros_like(h)
        outs = []
        for t in range(seq.shape[0]):
            i, f, g, o = (xp[t] + h @ wh.T).chunk(4, dim=-1)
            c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(g)
            h = torch.sigmoid(o) * torch.tanh(c)
            outs.append(h)
        seq = torch.stack(outs)
    return seq.permute(1, 2, 0) + x


def encoder(st, wave):
    """wave [B, 1, T] -> [B, 128, ceil(T / 320)]"""
    x = conv(st, "encoder.model.0.conv.conv", wave.to(f64))
    for i, s in enumerate(RATIOS):
        x = resblock(st, f"encoder.model.{ENC_RES[i]}", x)
        x = conv(st, f"encoder.model.{ENC_DOWN[i]}.conv.conv", F.elu(x), stride=s)
    x = lstm_block(st, f"encoder.model.{ENC_LSTM}", x)
    return conv(st, f"encoder.model.{ENC_LAST}.conv.conv", F.elu(x))


def decoder(st, emb):
    """emb [B, 128, n] -> wave [B, 1, 320 n]"""
    x = conv(st, f"decoder.model.{DEC_FIRST}.conv.conv", emb.to(f64))
    x = lstm_block(st, f"decoder.model.{DEC_LSTM}", x)
    for i, s in enumerate(reversed(RATIOS)):
        x = convtr(st, f"decoder.model.{DEC_UP[i]}.convtr.convtr", F.elu(x), s)
        x = resblock(st, f"decoder.model.{DEC_RES[i]}", x)
    return conv(st, f"decoder.model.{DEC_LAST}.conv.conv", F.elu(x))


def codebooks(st, n_q=N_CODEBOOKS):
    return torch.stack([st[f"quantizer.vq.layers.{q}._codebook.embed"].to(f64) for q in range(n_q)])


def rvq_encode(emb, cbs):
    """emb [N, 128], cbs [Q, 1024, 128] -> (codes [N, Q], quantized [N, 128], margin [N, Q]): per stage the nearest
    code by -(|r|^2 - 2 r.e + |e|^2), lowest index on ties; margin = runner-up distance minus the best one."""
    r = emb.to(f64).clone()
    codes, margins = [], []
    for cb in cbs:
        d = (r * r).sum(-1, keepdim=True) - 2 * r @ cb.T + (cb * cb).sum(-1)
        two = d.topk(2, dim=-1, largest=False)
        idx = d.argmin(-1)
        codes.append(idx)
        margins.append(two.values[:, 1] - two.values[:, 0])
        r = r - cb[idx]
    return torch.stack(codes, -1), emb.to(f64) - r, torch.stack(margins, -1)


def rvq_decode(codes, cbs):
    """codes [N, Q] -> sum of the selected codes [N, 128]"""
    return sum(cbs[q][codes[:, q]] for q in range(codes.shape[1]))


def random_state(seed, noise_clips=4, noise_samples=48000):
    gen = torch.Generator().manual_seed(seed)
    st = {}
    for p, kind, ci, co, k in conv_specs():
        n = co if kind == "conv" else ci
        v = torch.randn(*state_shapes()[f"{p}.weight_v"], generator=gen)
        st[f"{p}.weight_v"] = v
        st[f"{p}.weight_g"] = (0.8 + 0.4 * torch.rand(n, 1, 1, generator=gen))
        st[f"{p}.bias"] = 0.1 * torch.randn(co, generator=gen)
    a = 1.0 / math.sqrt(H)
    for side, idx in (("encoder", ENC_LSTM), ("decoder", DEC_LSTM)):
        for l in range(2):
            for n in ("weight_ih", "weight_hh"):
                st[f"{side}.model.{idx}.lstm.{n}_l{l}"] = (2 * torch.rand(4 * H, H, generator=gen) - 1) * a
            for n in ("bias_ih", "bias_hh"):
                st[f"{side}.model.{idx}.lstm.{n}_l{l}"] = (2 * torch.rand(4 * H, generator=gen) - 1) * a
    wave = torch.randn(noise_clips, 1, noise_samples, generator=gen, dtype=f64) * 0.3
    r = encoder(st, wave).permute(0, 2, 1).reshape(-1, DIM)
    for q in range(N_CODEBOOKS):
        pick = torch.randint(0, r.shape[0], (CODEBOOK_SIZE,), generator=gen)
        cb = r[pick] + 0.05 * r.std() * torch.randn(CODEBOOK_SIZE, DIM, generator=gen, dtype=f64)
        idx, _, _ = rvq_encode(r, cb[None])
        r = r - cb[idx[:, 0]]
        p = f"quantizer.vq.layers.{q}._codebook"
        st[f"{p}.embed"] = cb.float()
        st[f"{p}.embed_avg"] = cb.float().clone()
        st[f"{p}.cluster_size"] = torch.ones(CODEBOOK_SIZE)
        st[f"{p}.inited"] = torch.ones(1)
    return {k: v.float().contiguous() for k, v in st.items()}


def checksum(st):
    """[n_keys, 2] fp64: (sum, sum of |.|) of every tensor in key order; catches generator drift"""
    return torch.tensor([[st[k].double().sum().item(), st[k].double().abs().sum().item()] for k in sorted(st)],
                        dtype=f64)
