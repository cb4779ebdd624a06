"""EncodecWrapper on the GPU (csrc/encodec.cu + the SoundStream conv kernels + the tensor-core RVQ).

* the resnet-block kernels (fp32 and tensor-core, the latter also writing phase planes) and the LSTM kernel (fp32 and
  C8S in / out, its barrier error flag read back) against fp64, C in {32, ..., 256}, B in {1, 3, 16}, one frame to 30 s, with and
  without elu_out, each element held to a bound of the error model below;
* the whole encoder and decoder against the fp64 oracle (oracle/encodec.py) at 1 s and 10 s (the tensor-core plan) and
  at T in {1, 319, 321, 240017} (the fp32 plan), asserting which plan runs; codes equal to the fp64 codes on every stage that, with every earlier stage of its frame, clears its
  distance margin;
* the golden (the reference's own encodec.py on the seeded oracle model) end to end, bitwise determinism, a clip alone
  vs inside a batch of 8, the per-row decode, and the Coarse / Fine wrappers and AudioLM driven by EncodecWrapper.

Error model (fp32 arithmetic, unit roundoff u = 2^-24):
  a K-term fp32 dot product: K u sum |x| |w|                                           (ACC)
  ELU (expm1f) adds ACT_U u |y|, ACT_U = 4; an error e on an ELU input leaves at most |e| on its output (slope <= 1)
  LSTM: the bound is propagated through the recurrence next to the fp64 reference (_lstm_ref_bound): a gate
  pre-activation carries 1025 u sum |w| |v| (ACC) plus sum |w| e_v for the bounds e_v of its inputs h and x; sigmoid
  has slope <= 1/4 and tanh <= 1, each adds ACT_U u of its output; then e_c = s(f) e_c' + |c'| e_f / 4 + |g| e_i / 4
  + s(i) e_g + ACT_U u |c| and e_h = s(o) (e_c + ACT_U u) + |tanh c| e_o / 4 + ACT_U u |h|.
  Tensor cores (split bf16, as tests/test_codec_envelope_gpu.py): SPLIT = 2^-15 relative per product, a C8S value
  (hi + lo) within C8S = 2^-16 of the fp32 it holds, __expf-based ELU within ELU_TC = 2^-20 absolute.
  Whole codec: every layer's relative error is ~1e-6 (fp32) or ~1e-5 (split bf16); the model bound is
  MODEL_REL * max |y|.
"""
import torch
import torch.nn.functional as F
import pytest

from oracle import encodec as oe
from oracle import golden

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24
ACT_U = 4
MODEL_REL = 2e-4
SPLIT = 2.0 ** -15
C8S = 2.0 ** -16
ELU_TC = 2.0 ** -20
F64 = torch.float64


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


@pytest.fixture(scope="module")
def state():
    return oe.random_state(5, noise_clips=1, noise_samples=24000)


@pytest.fixture(scope="module")
def ckpt(tmp_path_factory, state):
    p = tmp_path_factory.mktemp("encodec") / "encodec_24khz.th"
    torch.save(state, p)
    return p


def _wrapper(ckpt, bandwidth=6.0):
    from audiolm_pytorch_b200 import EncodecWrapper

    return EncodecWrapper(bandwidth=bandwidth, checkpoint_path=ckpt).to(DEV)


# ---- kernels --------------------------------------------------------------------------------------------------
def _resblock_ref(x, w3, b3, w1, ws, bo, elu_out):
    """(y, bound) in fp64"""
    ex = F.elu(x)
    a3 = oe.pad1d(ex, 2, 0)
    pre = F.conv1d(a3, w3, b3)
    pre_abs = F.conv1d(a3.abs(), w3.abs(), b3.abs())
    h = F.elu(pre)
    err_h = (3 * x.shape[1] + 1) * U * pre_abs + ACT_U * U * h.abs()
    y = F.conv1d(h, w1[..., None]) + F.conv1d(x, ws[..., None]) + bo[:, None]
    acc = F.conv1d(h.abs(), w1.abs()[..., None]) + F.conv1d(x.abs(), ws.abs()[..., None]) + bo.abs()[:, None]
    bound = (w1.shape[1] + ws.shape[1] + 1) * U * acc + F.conv1d(err_h, w1.abs()[..., None])
    if elu_out:
        y = F.elu(y)
        bound = bound + ACT_U * U * y.abs()
    return y, bound


@pytest.mark.parametrize("C", [32, 64, 128, 256])
@pytest.mark.parametrize("B,T", [(1, 1), (3, 2), (16, 321), (3, 24000), (1, 720000)])
@pytest.mark.parametrize("elu_out", [False, True])
def test_resblock_kernel(C, B, T, elu_out):
    from audiolm_pytorch_b200 import ops

    g = _gen(C + T)
    x = torch.randn(B, C, T, device=DEV, generator=g)
    w3 = torch.randn(C // 2, C, 3, device=DEV, generator=g) / (3 * C) ** 0.5
    b3 = 0.1 * torch.randn(C // 2, device=DEV, generator=g)
    w1 = torch.randn(C, C // 2, device=DEV, generator=g) / (C // 2) ** 0.5
    ws = torch.randn(C, C, device=DEV, generator=g) / C ** 0.5
    bo = 0.1 * torch.randn(C, device=DEV, generator=g)
    y = ops.encodec_resblock(x, w3, b3, w1, ws, bo, elu_out=elu_out)
    ref, bound = _resblock_ref(*(t.double() for t in (x, w3, b3, w1, ws, bo)), elu_out)
    ratio = ((y.double() - ref).abs() / bound).max().item()
    assert ratio <= 1.0, f"err/bound {ratio:.3f}"


@pytest.mark.parametrize("C", [32, 64, 128, 256])
@pytest.mark.parametrize("B,T", [(1, 3), (3, 64), (16, 321), (3, 24000), (1, 720000)])
@pytest.mark.parametrize("elu_out,phases", [(False, 1), (True, 1), (True, 8)])
def test_resblock_tc_kernel(C, B, T, elu_out, phases):
    from audiolm_pytorch_b200 import ops

    T = -(-T // phases) * phases
    g = _gen(C + T + 1)
    x = ops.c8s_unpack(ops.c8s_pack(torch.randn(B, C, T, device=DEV, generator=g)))
    w3 = torch.randn(C // 2, C, 3, device=DEV, generator=g) / (3 * C) ** 0.5
    b3 = 0.1 * torch.randn(C // 2, device=DEV, generator=g)
    w1 = torch.randn(C, C // 2, device=DEV, generator=g) / (C // 2) ** 0.5
    ws = torch.randn(C, C, device=DEV, generator=g) / C ** 0.5
    bo = 0.1 * torch.randn(C, device=DEV, generator=g)
    b3p = torch.cat((b3, torch.zeros(C - C // 2, device=DEV)))
    y = ops.encodec_resblock_tc(ops.c8s_pack(x), ops.pack_encodec_resblock(w3, w1, ws).to(DEV), b3p, bo,
                                elu_out=elu_out, out_phases=phases)
    y = ops.c8s_unpack(y.reshape(B, C // 4, phases, T // phases, 8)).double()
    xd, w3d, b3d, w1d, wsd, bod = (t.double() for t in (x, w3, b3, w1, ws, bo))
    ex = F.elu(xd)
    a3 = oe.pad1d(ex, 2, 0)
    pre = F.conv1d(a3, w3d, b3d)
    acc3 = F.conv1d(a3.abs(), w3d.abs(), b3d.abs())
    h = F.elu(pre)
    e_h = (SPLIT + C8S + 3 * C * U) * acc3 + ELU_TC + C8S * h.abs()
    ref = F.conv1d(h, w1d[..., None]) + F.conv1d(xd, wsd[..., None]) + bod[:, None]
    acc = F.conv1d(h.abs(), w1d.abs()[..., None]) + F.conv1d(xd.abs(), wsd.abs()[..., None]) + bod.abs()[:, None]
    bound = (SPLIT + (C + C // 2 + 1) * U) * acc + F.conv1d(e_h, w1d.abs()[..., None])
    if elu_out:
        ref = F.elu(ref)
        bound = bound + ELU_TC
    bound = bound + C8S * ref.abs()
    ratio = ((y - ref).abs() / bound).max().item()
    assert ratio <= 1.0, f"err/bound {ratio:.3f}"


def _lstm_ref_bound(x, st):
    """(y, bound) of LSTM2(LSTM1(x)) + x in fp64, the bound propagated as in the module docstring"""
    seq, eseq = x.permute(2, 0, 1), torch.zeros_like(x.permute(2, 0, 1))
    for l in range(2):
        wi, wh = st[f"l.lstm.weight_ih_l{l}"].double(), st[f"l.lstm.weight_hh_l{l}"].double()
        b = st[f"l.lstm.bias_ih_l{l}"].double() + st[f"l.lstm.bias_hh_l{l}"].double()
        h = torch.zeros(seq.shape[1], 512, dtype=F64, device=x.device)
        c, eh, ec = torch.zeros_like(h), torch.zeros_like(h), torch.zeros_like(h)
        outs, eouts = [], []
        for t in range(seq.shape[0]):
            pre = seq[t] @ wi.T + h @ wh.T + b
            acc = seq[t].abs() @ wi.abs().T + h.abs() @ wh.abs().T + b.abs()
            ep = 1025 * U * acc + eseq[t] @ wi.abs().T + eh @ wh.abs().T
            i, f, g, o = pre.chunk(4, -1)
            ei, ef, eg, eo = ep.chunk(4, -1)
            si, sf, tg, so = torch.sigmoid(i), torch.sigmoid(f), torch.tanh(g), torch.sigmoid(o)
            ei, ef, eo = ei / 4 + ACT_U * U * si, ef / 4 + ACT_U * U * sf, eo / 4 + ACT_U * U * so
            eg = eg + ACT_U * U * tg.abs()
            c_new = sf * c + si * tg
            ec = sf * ec + c.abs() * ef + tg.abs() * ei + si * eg + ACT_U * U * c_new.abs()
            c = c_new
            tc = torch.tanh(c)
            h = so * tc
            eh = so * (ec + ACT_U * U * tc.abs()) + tc.abs() * eo + ACT_U * U * h.abs()
            outs.append(h)
            eouts.append(eh)
        seq, eseq = torch.stack(outs), torch.stack(eouts)
    return seq.permute(1, 2, 0) + x, eseq.permute(1, 2, 0) + ACT_U * U * (seq.permute(1, 2, 0) + x).abs()


def _lstm_state(seed):
    g = torch.Generator().manual_seed(seed)
    a = 1 / 512 ** 0.5
    return {f"l.lstm.{n}_l{l}": ((2 * torch.rand(*s, generator=g) - 1) * a)
            for l in range(2) for n, s in (("weight_ih", (2048, 512)), ("weight_hh", (2048, 512)),
                                           ("bias_ih", (2048,)), ("bias_hh", (2048,)))}


@pytest.mark.parametrize("B,T", [(1, 1), (3, 2), (16, 75), (1, 2250), (3, 750)])
@pytest.mark.parametrize("elu_out", [False, True])
def test_lstm_kernel(B, T, elu_out):
    from audiolm_pytorch_b200 import ops

    st = _lstm_state(B * 1000 + T)
    packed = ops.encodec_lstm_pack(*([st[f"l.lstm.{n}_l{l}"].to(DEV) for l in range(2)]
                                     for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")))
    x = torch.randn(B, 512, T, device=DEV, generator=_gen(T))
    y = ops.encodec_lstm(x, packed, elu_out=elu_out, check=True)
    ref, bound = _lstm_ref_bound(x.double(), {k: v.to(DEV) for k, v in st.items()})
    if elu_out:
        ref = F.elu(ref)
        bound = bound + ACT_U * U * ref.abs()
    ratio = ((y.double() - ref).abs() / bound).max().item()
    assert ratio <= 1.0, f"err/bound {ratio:.3f}"
    # the same kernel on the tensor-core codec layout: input and output as C8S
    yc = ops.c8s_unpack(ops.encodec_lstm(ops.c8s_pack(x), packed, elu_out=elu_out, check=True))
    xr = ops.c8s_unpack(ops.c8s_pack(x)).double()
    ref, bound = _lstm_ref_bound(xr, {k: v.to(DEV) for k, v in st.items()})
    if elu_out:
        ref = F.elu(ref)
        bound = bound + ACT_U * U * ref.abs()
    ratio = ((yc.double() - ref).abs() / (bound + C8S * ref.abs())).max().item()
    assert ratio <= 1.0, f"C8S err/bound {ratio:.3f}"


def test_lstm_batch_invariance_and_determinism():
    from audiolm_pytorch_b200 import ops

    st = _lstm_state(3)
    packed = ops.encodec_lstm_pack(*([st[f"l.lstm.{n}_l{l}"].to(DEV) for l in range(2)]
                                     for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")))
    x = torch.randn(11, 512, 40, device=DEV, generator=_gen(1))
    y = ops.encodec_lstm(x, packed, elu_out=True)
    assert torch.equal(y, ops.encodec_lstm(x, packed, elu_out=True))
    assert torch.equal(y[9:10], ops.encodec_lstm(x[9:10], packed, elu_out=True))


# ---- whole codec ------------------------------------------------------------------------------------------------
def _model_err(y, ref):
    return ((y.double() - ref).abs().max() / ref.abs().max()).item()


@pytest.mark.parametrize("T", [1, 319, 321, 24000, 240000, 240017])
def test_encoder_decoder_against_fp64(ckpt, state, T):
    w = _wrapper(ckpt)
    st = {k: v.to(DEV) for k, v in state.items()}
    wave = 0.3 * torch.randn(2, T, device=DEV, generator=_gen(T))
    # T a multiple of 320 with >= 8 frames takes the tensor-core plan, every other length the fp32 kernels
    assert w.tc_plan(T // 320, T) == (T % 320 == 0 and T >= 8 * 320)
    with torch.no_grad():
        emb = w.encode_frames(wave)
        ref = oe.encoder(st, wave[:, None].double())
        assert emb.shape == (2, oe.n_frames(T), 128)
        e_err = _model_err(emb.transpose(1, 2), ref)
        assert e_err < MODEL_REL, e_err
        dec = w.decode(ref.transpose(1, 2).float())
        dref = oe.decoder(st, ref)
        assert dec.shape == (2, 1, 320 * oe.n_frames(T))
        d_err = _model_err(dec, dref)
        assert d_err < MODEL_REL, d_err
        # codes: every stage of a frame must clear its margin (squared distances) by the emb error's effect on it
        _, codes, _ = w(wave)
        rc, _, margin = oe.rvq_encode(ref.transpose(1, 2).reshape(-1, 128), oe.codebooks(st, 8))
        de = (emb.reshape(-1, 128).double() - ref.transpose(1, 2).reshape(-1, 128)).norm(dim=-1, keepdim=True)
        scale = ref.transpose(1, 2).reshape(-1, 128).norm(dim=-1, keepdim=True) + oe.codebooks(st, 8).norm(dim=-1).max()
        # a stage is compared when it and every earlier stage of its frame clear the bound (later residuals differ
        # once a code differs)
        safe = (margin > 8 * de * scale + 1e-9).long().cumprod(-1).bool()
        assert safe[:, 0].float().mean() > 0.5 or safe.shape[0] < 75
        assert torch.equal(codes.reshape(-1, 8)[safe], rc[safe])


@pytest.fixture(scope="module")
def golden_fx(tmp_path_factory):
    g = golden.load("encodec.pt")
    st = oe.random_state(g["seed"])
    assert torch.allclose(oe.checksum(st), g["checksum"], rtol=1e-12, atol=0), "the seeded generator drifted"
    p = tmp_path_factory.mktemp("encodec_golden") / "encodec_24khz.th"
    torch.save(st, p)
    return g, st, p


@pytest.mark.parametrize("bw", [1.5, 6.0])
def test_golden_end_to_end(golden_fx, bw):
    g, st, p = golden_fx
    w = _wrapper(p, bw)
    assert w.num_quantizers == g["n_q"][bw]
    for wave, codes_ref, emb_ref in zip(g["waves"], g["codes"][bw], g["emb"][bw]):
        emb, codes, none = w(wave.to(DEV), return_encoded=True)
        assert none is None and codes.shape == codes_ref.shape and codes.dtype == torch.int64
        e64 = oe.encoder(st, wave[:, None].double()).transpose(1, 2).reshape(-1, 128)
        rc, _, margin = oe.rvq_encode(e64, oe.codebooks(st, w.num_quantizers))
        assert torch.equal(rc, codes_ref.reshape(rc.shape))
        safe = (margin > 1e-3).long().cumprod(-1).bool()
        assert safe[:, 0].float().mean() > 0.9
        assert torch.equal(codes.reshape(rc.shape).cpu()[safe], rc[safe])
        assert torch.allclose(emb.cpu(), w.get_emb_from_indices(codes).cpu()) and emb.shape == emb_ref.shape
        same = (codes.cpu() == codes_ref).all(-1)
        assert torch.allclose(emb.cpu()[same], emb_ref[same], atol=1e-5)
    if bw == 6.0:
        codes = g["codes"][bw][0].to(DEV)
        one = w.decode_from_codebook_indices(codes[:1])
        assert one.shape == g["decoded_b1"].shape
        assert _model_err(one.cpu(), g["decoded_b1"].double()) < MODEL_REL
        # the reference blends a batch into one [1, 1, T + B - 1] wave; every row here is its own B = 1 decode
        both = w.decode_from_codebook_indices(codes)
        assert g["decoded_batch_ref"].shape == (1, 1, one.shape[-1] + 1) and both.shape == (2, 1, one.shape[-1])
        assert torch.equal(both[:1], one)


def test_determinism_and_batch_invariance(ckpt):
    w = _wrapper(ckpt)
    wave = 0.3 * torch.randn(8, 24000, device=DEV, generator=_gen(2))
    with torch.no_grad():
        e8 = w.encode_frames(wave)
        assert torch.equal(e8, w.encode_frames(wave))
        assert torch.equal(e8[5:6], w.encode_frames(wave[5:6]))
        _, c8, _ = w(wave)
        _, c1, _ = w(wave[5:6])
        assert torch.equal(c8[5:6], c1)
        d8 = w.decode_from_codebook_indices(c8)
        assert torch.equal(d8, w.decode_from_codebook_indices(c8))
        assert torch.equal(d8[5:6], w.decode_from_codebook_indices(c1))


def test_leading_dims_and_cpu_input(ckpt):
    from audiolm_pytorch_b200._lib import AlmError

    w = _wrapper(ckpt)
    wave = 0.3 * torch.randn(2, 3, 3200, device=DEV, generator=_gen(3))
    emb, codes, _ = w(wave, return_encoded=True)
    assert codes.shape == (2, 3, 10, 8) and emb.shape == (2, 3, 10, 128)
    with pytest.raises(AlmError):
        w(wave.cpu())


SMALL_KW = dict(dim=64, depth=2, heads=2, flash_attn=True)


def test_coarse_and_fine_wrappers(ckpt):
    from audiolm_pytorch_b200 import (CoarseTransformer, CoarseTransformerWrapper, FineTransformer,
                                      FineTransformerWrapper)

    codec = _wrapper(ckpt)
    torch.manual_seed(1)
    coarse = CoarseTransformer(num_semantic_tokens=50, codebook_size=1024, num_coarse_quantizers=3, **SMALL_KW).to(DEV)
    cw = CoarseTransformerWrapper(transformer=coarse, codec=codec, mask_prob=0.0).eval()
    wave = 0.3 * torch.randn(2, 6400, device=DEV, generator=_gen(4))
    sem = torch.randint(0, 50, (2, 20), device=DEV, generator=_gen(5))
    with torch.no_grad():
        assert torch.isfinite(cw(semantic_token_ids=sem, raw_wave_for_codec=wave, return_loss=True))
    fine = FineTransformer(num_coarse_quantizers=3, num_fine_quantizers=5, codebook_size=1024, **SMALL_KW).to(DEV)
    fw = FineTransformerWrapper(transformer=fine, codec=codec).eval()
    with torch.no_grad():
        assert torch.isfinite(fw(raw_wave=wave, return_loss=True))


def test_audiolm_generate(ckpt, monkeypatch):
    from audiolm_pytorch_b200 import AudioLM, CoarseTransformer, FineTransformer, SemanticTransformer

    codec = _wrapper(ckpt, bandwidth=1.5)
    torch.manual_seed(5)
    sem = SemanticTransformer(num_semantic_tokens=50, **SMALL_KW).to(DEV)
    coarse = CoarseTransformer(num_semantic_tokens=50, codebook_size=1024, num_coarse_quantizers=1, **SMALL_KW).to(DEV)
    fine = FineTransformer(num_coarse_quantizers=1, num_fine_quantizers=1, codebook_size=1024, **SMALL_KW).to(DEV)
    lm = AudioLM(wav2vec=None, codec=codec, semantic_transformer=sem, coarse_transformer=coarse, fine_transformer=fine)
    real = lm.coarse.generate
    monkeypatch.setattr(lm.coarse, "generate", lambda **k: real(**{**k, "max_time_steps": 8}))
    wav = lm(batch_size=1, max_length=6)
    wavs = [wav] if torch.is_tensor(wav) and wav.dim() == 1 else list(wav)
    assert len(wavs) == 1
    for w_ in wavs:
        assert w_ is not None and w_.numel() % 320 == 0 and w_.numel() > 0 and torch.isfinite(w_).all()
