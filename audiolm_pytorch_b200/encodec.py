"""EncodecWrapper: the pretrained 24 kHz EnCodec as the codec of the Coarse / Fine wrappers and AudioLM, on sm_90a
kernels and without the encodec package (audiolm_pytorch/encodec.py).

The network is encodec 0.1.1's `EncodecModel.encodec_model_24khz()` with `normalize = False`: a causal SEANet encoder
(strides 2, 4, 5, 8; 320 samples per frame), a 2-layer LSTM block of width 512 with a skip on each side, a residual VQ
of 32 codebooks of 1024 x 128 of which the bandwidth selects the first n_q, and the mirrored decoder.  The weights come
from encodec's published checkpoint file, read as a plain state dict; the package never downloads it.

Every ELU of the network sits between a resnet block or an LSTM block and the conv after it, so the block kernels
apply it in their epilogue (`elu_out`) and the convs run on the SoundStream conv kernels unchanged.  A clip of whole
frames (T a multiple of 320, at least 8 frames) runs on the tensor cores in split bf16 with C8S activations; every
other length runs on the fp32 CUDA-core kernels.
"""
from __future__ import annotations

import math
from pathlib import Path

import torch
from torch import nn

from . import ops
from ._lib import AlmError
from .soundstream import ResidualVQ, SoundStream

f32, f64 = torch.float32, torch.float64

CHECKPOINT_NAME = "encodec_24khz-d7cc33bc.th"
CHECKPOINT_URL = "https://dl.fbaipublicfiles.com/encodec/v0/" + CHECKPOINT_NAME
BANDWIDTH_QUANTIZERS = {1.5: 2, 3.0: 4, 6.0: 8, 12.0: 16, 24.0: 32}
RATIOS = (2, 4, 5, 8)           # encoder strides; the decoder runs them reversed
CHANNELS = (32, 64, 128, 256)   # resnet-block widths in encoder order
LSTM_H, DIM, N_CODEBOOKS, CODEBOOK_SIZE = 512, 128, 32, 1024
TC_MIN_FRAMES = 8  # the frame-level k7 convs reflect 6 samples
ENC_RES, ENC_DOWN, ENC_LSTM, ENC_LAST = (1, 4, 7, 10), (3, 6, 9, 12), 13, 15
DEC_FIRST, DEC_LSTM, DEC_UP, DEC_RES, DEC_LAST = 0, 1, (3, 6, 9, 12), (4, 7, 10, 13), 15


def _conv_shapes(prefix, cin, cout, k, transposed=False):
    # weight_norm(dim=0): g has one entry per output channel of a Conv1d, per INPUT channel of a ConvTranspose1d
    if transposed:
        return {f"{prefix}.weight_g": (cin, 1, 1), f"{prefix}.weight_v": (cin, cout, k), f"{prefix}.bias": (cout,)}
    return {f"{prefix}.weight_g": (cout, 1, 1), f"{prefix}.weight_v": (cout, cin, k), f"{prefix}.bias": (cout,)}


def _resblock_shapes(prefix, c):
    return {**_conv_shapes(f"{prefix}.block.1.conv.conv", c, c // 2, 3),
            **_conv_shapes(f"{prefix}.block.3.conv.conv", c // 2, c, 1),
            **_conv_shapes(f"{prefix}.shortcut.conv.conv", c, c, 1)}


def _lstm_shapes(prefix):
    return {f"{prefix}.lstm.{n}_l{l}": s for l in range(2)
            for n, s in (("weight_ih", (4 * LSTM_H, LSTM_H)), ("weight_hh", (4 * LSTM_H, LSTM_H)),
                         ("bias_ih", (4 * LSTM_H,)), ("bias_hh", (4 * LSTM_H,)))}


def checkpoint_shapes():
    """key -> shape of every tensor in encodec's 24 kHz checkpoint (encodec 0.1.1 module tree)."""
    sh = _conv_shapes("encoder.model.0.conv.conv", 1, 32, 7)
    for i, (c, s) in enumerate(zip(CHANNELS, RATIOS)):
        sh |= _resblock_shapes(f"encoder.model.{ENC_RES[i]}", c)
        sh |= _conv_shapes(f"encoder.model.{ENC_DOWN[i]}.conv.conv", c, 2 * c, 2 * s)
    sh |= _lstm_shapes(f"encoder.model.{ENC_LSTM}")
    sh |= _conv_shapes(f"encoder.model.{ENC_LAST}.conv.conv", LSTM_H, DIM, 7)
    sh |= _conv_shapes(f"decoder.model.{DEC_FIRST}.conv.conv", DIM, LSTM_H, 7)
    sh |= _lstm_shapes(f"decoder.model.{DEC_LSTM}")
    for i, (c, s) in enumerate(zip(reversed(CHANNELS), reversed(RATIOS))):
        sh |= _conv_shapes(f"decoder.model.{DEC_UP[i]}.convtr.convtr", 2 * c, c, 2 * s, transposed=True)
        sh |= _resblock_shapes(f"decoder.model.{DEC_RES[i]}", c)
    sh |= _conv_shapes(f"decoder.model.{DEC_LAST}.conv.conv", 32, 1, 7)
    for q in range(N_CODEBOOKS):
        p = f"quantizer.vq.layers.{q}._codebook"
        sh |= {f"{p}.inited": (1,), f"{p}.cluster_size": (CODEBOOK_SIZE,), f"{p}.embed": (CODEBOOK_SIZE, DIM),
               f"{p}.embed_avg": (CODEBOOK_SIZE, DIM)}
    return sh


def default_checkpoint_path() -> Path:
    return Path(torch.hub.get_dir()) / "checkpoints" / CHECKPOINT_NAME


def load_checkpoint(path) -> dict:
    """encodec's checkpoint (a plain state dict) -> {key: fp32 tensor}; refuses missing, unexpected or mis-shaped keys"""
    sd = torch.load(path, map_location="cpu", weights_only=True)
    if not isinstance(sd, dict):
        raise ValueError(f"{path}: expected a state dict, got {type(sd).__name__}")
    shapes = checkpoint_shapes()
    missing = [k for k in shapes if k not in sd]
    unexpected = [k for k in sd if k not in shapes]
    if missing:
        raise KeyError(f"{path}: missing key {missing[0]!r} ({len(missing)} missing)")
    if unexpected:
        raise KeyError(f"{path}: unexpected key {unexpected[0]!r} ({len(unexpected)} unexpected)")
    for k, s in shapes.items():
        if tuple(sd[k].shape) != s:
            raise ValueError(f"{path}: {k!r} has shape {tuple(sd[k].shape)}, expected {s}")
    return {k: sd[k].to(f32) for k in shapes}


class _Tree(nn.Module):
    """holds checkpoint tensors under their dotted keys: weights as frozen parameters, codebook state as buffers"""

    def add(self, key, t):
        mod = self
        *path, name = key.split(".")
        for p in path:
            if p not in mod._modules:
                mod.add_module(p, _Tree())
            mod = mod._modules[p]
        if ".quantizer." in f".{key}":
            mod.register_buffer(name, t.clone())
        else:
            mod.register_parameter(name, nn.Parameter(t.clone(), requires_grad=False))


def _fold(g, v):
    """weight norm w = g v / ||v|| (norm over every dim but 0) in fp64 -> fp32"""
    v = v.detach().to(f64)
    return (g.detach().to(f64) * v / v.flatten(1).norm(dim=1).view(-1, *([1] * (v.dim() - 1)))).to(f32).contiguous()


class EncodecWrapper(nn.Module):
    """audiolm_pytorch/encodec.py's EncodecWrapper (24 kHz, normalize=False) on libalm_b200.

    checkpoint_path: encodec's `encodec_24khz-d7cc33bc.th`; None reads it from torch hub's checkpoint directory.
    `num_quantizers` is ignored, as in the reference: the bandwidth selects n_q (1.5/3/6/12/24 kbps -> 2/4/8/16/32)."""

    def __init__(self, target_sample_hz=24000, strides=(2, 4, 5, 8), num_quantizers=8, bandwidth=6.0, *,
                 checkpoint_path=None):
        super().__init__()
        if float(bandwidth) not in BANDWIDTH_QUANTIZERS:
            raise ValueError(f"bandwidth {bandwidth} kbps: the 24 kHz EnCodec supports {sorted(BANDWIDTH_QUANTIZERS)}")
        self.target_sample_hz = target_sample_hz
        assert self.target_sample_hz == 24000, "haven't done anything with non-24kHz yet"
        if checkpoint_path is None:
            checkpoint_path = default_checkpoint_path()
            if not checkpoint_path.exists():
                raise FileNotFoundError(f"EnCodec checkpoint not found at {checkpoint_path}; download it from "
                                        f"{CHECKPOINT_URL} to that path, or pass checkpoint_path=")
        sd = load_checkpoint(checkpoint_path)
        self.bandwidth = float(bandwidth)
        self.num_quantizers = BANDWIDTH_QUANTIZERS[self.bandwidth]
        self.codebook_dim = DIM
        self.rq_groups = 1
        self.strides = strides
        self.model = _Tree()
        for k, t in sd.items():
            self.model.add(k, t)
        self.rq = ResidualVQ(dim=DIM, codebook_size=CODEBOOK_SIZE, num_quantizers=self.num_quantizers)
        with torch.no_grad():
            for q, layer in enumerate(self.rq.layers):
                layer._codebook.embed.copy_(sd[f"quantizer.vq.layers.{q}._codebook.embed"][None])
                layer._codebook.initted.fill_(True)
        self.eval()

    @property
    def seq_len_multiple_of(self):
        return math.prod(self.strides)

    @property
    def downsample_factor(self):
        return self.seq_len_multiple_of

    # ---- weights ----------------------------------------------------------------------------------------
    def _weights(self):
        """folded fp32 weights of every layer, rebuilt when any parameter changes"""
        params = [p for _, p in sorted(self.model.named_parameters())]
        return SoundStream._cached(self, "_folded", params, self._build_weights)

    def _build_weights(self):
        p = dict(self.model.named_parameters())

        def conv(prefix):
            w = _fold(p[f"{prefix}.weight_g"], p[f"{prefix}.weight_v"])
            return w, p[f"{prefix}.bias"].detach().float().contiguous(), w.permute(1, 2, 0).contiguous()

        def convtr(prefix):
            return _fold(p[f"{prefix}.weight_g"], p[f"{prefix}.weight_v"]), p[f"{prefix}.bias"].detach().float()

        def resblock(prefix):
            w3, b3, _ = conv(f"{prefix}.block.1.conv.conv")
            w1, b1, _ = conv(f"{prefix}.block.3.conv.conv")
            ws, bs, _ = conv(f"{prefix}.shortcut.conv.conv")
            b_out = (b1.double() + bs.double()).float()
            return w3, b3, w1[..., 0].contiguous(), ws[..., 0].contiguous(), b_out

        def lstm(prefix):
            get = lambda n: [p[f"{prefix}.lstm.{n}_l{l}"].detach() for l in range(2)]  # noqa: E731
            return ops.encodec_lstm_pack(get("weight_ih"), get("weight_hh"), get("bias_ih"), get("bias_hh"))

        def resblock_tc(rb):
            w3, b3, w1, ws, b_out = rb
            b3p = torch.zeros_like(b_out)
            b3p[: b3.numel()] = b3
            return ops.pack_encodec_resblock(w3, w1, ws), b3p, b_out

        enc_blocks = [(resblock(f"encoder.model.{r}"), conv(f"encoder.model.{d}.conv.conv"), s)
                      for r, d, s in zip(ENC_RES, ENC_DOWN, RATIOS)]
        dec_blocks = [(convtr(f"decoder.model.{u}.convtr.convtr"), resblock(f"decoder.model.{r}"), s)
                      for u, r, s in zip(DEC_UP, DEC_RES, reversed(RATIOS))]
        enc_last, dec_first = conv(f"encoder.model.{ENC_LAST}.conv.conv"), conv(f"decoder.model.{DEC_FIRST}.conv.conv")
        # the tensor-core plan (T a multiple of 320): split-bf16 units of the same weights
        tc = dict(
            enc_blocks=[(resblock_tc(rb), ops.pack_conv_weights(down[0])) for rb, down, _ in enc_blocks],
            enc_last=ops.pack_conv_weights(enc_last[0]),
            dec_first=ops.pack_conv_weights(dec_first[0]),
            dec_blocks=[(ops.pack_convT_weights(wt, s), bt.repeat(s).contiguous(), resblock_tc(rb))
                        for (wt, bt), rb, s in dec_blocks],
        )
        return dict(
            tc=tc,
            enc_first=conv("encoder.model.0.conv.conv"),
            enc_blocks=enc_blocks,
            enc_lstm=lstm(f"encoder.model.{ENC_LSTM}"),
            enc_last=enc_last,
            dec_first=dec_first,
            dec_lstm=lstm(f"decoder.model.{DEC_LSTM}"),
            dec_blocks=dec_blocks,
            dec_last=conv(f"decoder.model.{DEC_LAST}.conv.conv"),
        )

    # ---- network ----------------------------------------------------------------------------------------
    @staticmethod
    def _conv(x, w, stride=1):
        weight, bias, packed = w
        return ops.encodec_conv(x, weight, bias, stride=stride, weight_packed=packed)

    @staticmethod
    def tc_plan(n_frames, T=None):
        """whether a clip of n_frames frames (and T samples) runs on the tensor-core plan: T a multiple of 320, and
        enough frames that every reflect halo (6 samples of the frame-level k7 convs) lies inside the input"""
        return n_frames >= TC_MIN_FRAMES and (T is None or T == n_frames * math.prod(RATIOS))

    def encode_frames(self, wave):
        """wave fp32 [B, T] on the GPU -> encoder output [B, ceil(T / 320), 128] channels-last"""
        T = wave.shape[-1]
        if self.tc_plan(T // math.prod(RATIOS), T):
            return self._encode_tc(wave)
        W = self._weights()
        x = self._conv(wave[:, None, :], W["enc_first"])
        for rb, down, s in W["enc_blocks"]:
            x = ops.encodec_resblock(x, *rb, elu_out=True)
            x = self._conv(x, down, stride=s)
        x = ops.encodec_lstm(x, W["enc_lstm"], elu_out=True)
        return self._conv(x, W["enc_last"]).transpose(1, 2).contiguous()

    def _encode_tc(self, wave):
        """the tensor-core plan: C8S split-bf16 activations between layers, one launch per layer"""
        W = self._weights()
        tc = W["tc"]
        w0, b0, _ = W["enc_first"]
        h = ops.codec_first_conv(wave, w0, b0)
        for ((units, b3p, b_out), down_units), (_, down, s) in zip(tc["enc_blocks"], W["enc_blocks"]):
            h = ops.encodec_resblock_tc(h, units, b3p, b_out, elu_out=True, out_phases=s)
            h = ops.codec_conv_tc(h, down_units, down[1], cout=down[0].shape[0], kernel_size=2 * s, stride=s)
        h = ops.encodec_lstm(h, W["enc_lstm"], elu_out=True)
        return ops.codec_conv_tc(h, tc["enc_last"], W["enc_last"][1], cout=DIM, kernel_size=7, stride=1, out_fp32=True)

    def _decode_tc(self, emb):
        W = self._weights()
        tc = W["tc"]
        h = ops.codec_pack_c8s(emb)
        h = ops.codec_conv_tc(h, tc["dec_first"], W["dec_first"][1], cout=LSTM_H, kernel_size=7, stride=1)
        h = ops.encodec_lstm(h, W["dec_lstm"], elu_out=True)
        for (up_units, b_up, (units, b3p, b_out)), ((wt, _), _, s) in zip(tc["dec_blocks"], W["dec_blocks"]):
            h = ops.codec_conv_tc(h, up_units, b_up, cout=s * wt.shape[1], kernel_size=2, stride=1,
                                  pad_mode="constant", upsample=s)
            h = ops.encodec_resblock_tc(h, units, b3p, b_out, elu_out=True)
        w_last, b_last, _ = W["dec_last"]
        return ops.codec_last_conv(h, w_last, b_last)

    def decode(self, emb):
        """emb [b, n, 128] -> wave [b, 1, 320 n]; every row is decoded on its own"""
        if not emb.is_cuda:
            raise AlmError("EncodecWrapper.decode: the input is on the CPU; the hot path has no CPU implementation")
        if self.tc_plan(emb.shape[1]):
            return self._decode_tc(emb.to(f32).contiguous())
        W = self._weights()
        x = self._conv(emb.to(f32).transpose(1, 2).contiguous(), W["dec_first"])
        x = ops.encodec_lstm(x, W["dec_lstm"], elu_out=True)
        for (wt, bt), rb, s in W["dec_blocks"]:
            x = ops.causal_conv_transpose1d(x, wt, bt, stride=s)
            x = ops.encodec_resblock(x, *rb, elu_out=True)
        return self._conv(x, W["dec_last"])

    # ---- reference surface --------------------------------------------------------------------------------
    def forward(self, x, input_sample_hz=None, return_encoded=False, **kwargs):
        assert not self.training, "Encodec is pretrained and should never be called outside eval mode."
        lead = x.shape[:-1]
        x = x.reshape(-1, x.shape[-1])  # the reference packs every leading dim ('* n')
        if not x.is_cuda:
            raise AlmError("EncodecWrapper: the input is on the CPU; the hot path has no CPU implementation")
        if input_sample_hz is not None and input_sample_hz != self.target_sample_hz:
            x = ops.resample(x, input_sample_hz, self.target_sample_hz)
        with torch.no_grad():
            h = self.encode_frames(x.to(f32).contiguous())
            _, codes, _ = self.rq(h)
        emb = None
        if return_encoded:
            emb = self.get_emb_from_indices(codes).reshape(*lead, *codes.shape[-2:-1], DIM)
        return emb, codes.reshape(*lead, *codes.shape[-2:]), None

    def get_emb_from_indices(self, indices):
        """codes [b, n, q] -> sum of the selected codes [b, n, 128]"""
        return self.rq.get_output_from_indices(indices)

    def decode_from_codebook_indices(self, quantized_indices):
        """codes [b, n, q] -> wave [b, 1, 320 n].  The reference runs the batch through encodec's overlap-add as if it
        were a list of frames, which blends the rows of a batch; this decodes every row on its own (its B = 1 result)."""
        assert quantized_indices.dtype in (torch.long, torch.int32)
        return self.decode(self.get_emb_from_indices(quantized_indices.long()))
