"""EncodecWrapper on the host: checkpoint loading without the encodec package, key and shape refusals, bandwidth ->
number of quantizers, state-dict keys, frame and padding arithmetic, and the fp64 oracle against transformers."""
import sys

import pytest
import torch

from oracle import encodec as oe


@pytest.fixture(scope="module")
def state():
    return oe.random_state(3, noise_clips=1, noise_samples=9600)


@pytest.fixture()
def ckpt(tmp_path, state):
    p = tmp_path / "encodec_24khz.th"
    torch.save(state, p)
    return p


def test_loads_without_encodec_package(ckpt, state, monkeypatch):
    monkeypatch.setitem(sys.modules, "encodec", None)  # `import encodec` raises
    from audiolm_pytorch_b200 import EncodecWrapper

    w = EncodecWrapper(checkpoint_path=ckpt)
    assert not w.training and w.num_quantizers == 8 and w.codebook_dim == 128 and w.rq_groups == 1
    assert w.seq_len_multiple_of == w.downsample_factor == 320 and w.target_sample_hz == 24000
    keys = set(w.state_dict())
    rq = {f"rq.layers.{q}._codebook.{n}" for q in range(8) for n in ("initted", "cluster_size", "embed_avg", "embed")}
    assert keys == {f"model.{k}" for k in state} | rq
    for q in range(8):
        assert torch.equal(w.rq.layers[q]._codebook.embed[0], state[f"quantizer.vq.layers.{q}._codebook.embed"])
        assert bool(w.rq.layers[q]._codebook.initted.item())
    assert torch.equal(w.state_dict()["model.encoder.model.13.lstm.weight_hh_l1"],
                       state["encoder.model.13.lstm.weight_hh_l1"])


def test_checkpoint_shapes_match_oracle():
    from audiolm_pytorch_b200.encodec import checkpoint_shapes

    assert checkpoint_shapes() == oe.state_shapes()


@pytest.mark.parametrize("bw,n_q", [(1.5, 2), (3, 4), (6, 8), (12.0, 16), (24, 32)])
def test_bandwidth_selects_quantizers(ckpt, bw, n_q):
    from audiolm_pytorch_b200 import EncodecWrapper

    w = EncodecWrapper(bandwidth=bw, num_quantizers=3, checkpoint_path=ckpt)
    assert w.num_quantizers == n_q and len(w.rq.layers) == n_q


def test_bad_bandwidth(ckpt):
    from audiolm_pytorch_b200 import EncodecWrapper

    with pytest.raises(ValueError, match="bandwidth"):
        EncodecWrapper(bandwidth=5.0, checkpoint_path=ckpt)


@pytest.mark.parametrize("edit", ["missing", "unexpected", "shape"])
def test_key_refusals(tmp_path, state, edit):
    from audiolm_pytorch_b200 import EncodecWrapper

    sd = dict(state)
    key = "decoder.model.6.convtr.convtr.weight_g"
    if edit == "missing":
        del sd[key]
    elif edit == "unexpected":
        key = "decoder.model.16.conv.conv.bias"
        sd[key] = torch.zeros(1)
    else:
        sd[key] = torch.zeros(128, 1, 1)  # a ConvTranspose1d's g runs over its 256 input channels
    p = tmp_path / "bad.th"
    torch.save(sd, p)
    with pytest.raises((KeyError, ValueError), match=key.replace(".", r"\.")):
        EncodecWrapper(checkpoint_path=p)


def test_missing_default_checkpoint(tmp_path, monkeypatch):
    from audiolm_pytorch_b200 import EncodecWrapper

    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(tmp_path))
    with pytest.raises(FileNotFoundError, match="encodec_24khz-d7cc33bc.th"):
        EncodecWrapper()


def test_cpu_input_raises(ckpt):
    from audiolm_pytorch_b200 import EncodecWrapper
    from audiolm_pytorch_b200._lib import AlmError

    with pytest.raises(AlmError):
        EncodecWrapper(checkpoint_path=ckpt)(torch.randn(1, 640))


@pytest.mark.parametrize("L,pl,pr", [(1, 6, 0), (3, 6, 0), (6, 6, 0), (7, 6, 0), (1, 2, 1), (5, 8, 3), (9, 8, 7)])
def test_pad_arithmetic(L, pl, pr):
    """the rule alm_encodec_pad1d implements (position q reads x[j], j reflected in the zero-extended row) equals
    EnCodec's pad-then-trim"""
    x = torch.arange(1, L + 1, dtype=torch.float64)[None]
    ref = oe.pad1d(x, pl, pr)
    mx = max(pl, pr)
    L0 = mx + 1 if L <= mx else L
    out = []
    for q in range(-pl, L + pr):
        j = -q if q < 0 else (q if q < L0 else 2 * (L0 - 1) - q)
        out.append(float(x[0, j]) if j < L else 0.0)
    assert torch.equal(ref[0], torch.tensor(out, dtype=torch.float64))


@pytest.mark.parametrize("T", [1, 319, 320, 321, 641])
def test_frame_count(state, T):
    e = oe.encoder(state, torch.zeros(1, 1, T, dtype=torch.float64))
    assert e.shape[-1] == oe.n_frames(T) == -(-T // 320)
    assert oe.decoder(state, e).shape[-1] == 320 * e.shape[-1]


@pytest.mark.parametrize("T", [1, 321])
def test_oracle_against_transformers(state, T):
    pytest.importorskip("transformers")
    from oracle.make_golden_encodec import to_transformers
    from transformers import EncodecConfig, EncodecModel

    m = EncodecModel(EncodecConfig()).double().eval()
    m.load_state_dict(to_transformers(state), strict=True)
    x = torch.randn(2, 1, T, generator=torch.Generator().manual_seed(T), dtype=torch.float64)
    with torch.no_grad():
        e_hf, e = m.encoder(x), oe.encoder(state, x)
        codes_hf = m.encode(x, bandwidth=6.0).audio_codes
        d_hf, d = m.decoder(e_hf), oe.decoder(state, e)
    assert torch.allclose(e, e_hf, rtol=0, atol=1e-12 * e.abs().max().item())
    assert torch.allclose(d, d_hf, rtol=0, atol=1e-12 * d.abs().max().item())
    codes, _, _ = oe.rvq_encode(e.permute(0, 2, 1).reshape(-1, 128), oe.codebooks(state, 8))
    assert torch.equal(codes_hf.reshape(2, 8, -1).permute(0, 2, 1).reshape(-1, 8), codes)


def test_golden_checksum():
    from oracle import golden

    g = golden.load("encodec.pt")
    assert torch.allclose(oe.checksum(oe.random_state(g["seed"])), g["checksum"], rtol=1e-12, atol=0)
