"""Head widths 32 / 64 / 128 without a GPU: constructors, parameter shapes and state-dict keys against the reference's
fixture (tests/golden/dim_head.pt), the C entry points that carry the width, and the unchanged dim_head-64 defaults."""
import inspect
import re
import sys
from pathlib import Path

import pytest
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
from test_dim_head_gpu import MODELS, WIDTHS, fixture, unpack  # noqa: E402

ROOT = Path(__file__).resolve().parent.parent
NEW_SYMBOLS = ["alm_mqa_attn_fwd_dh", "alm_mqa_attn_bwd_dh", "alm_attn_delta_dh", "alm_kv_append_dh",
               "alm_mqa_attn_decode_dh", "alm_decode_stack_plan_dh"]


def _cls(model):
    from audiolm_pytorch_b200 import audiolm
    return getattr(audiolm, model.capitalize() + "Transformer")


@pytest.mark.parametrize("D", [32, 64, 128])
def test_constructors_accept_the_three_widths(D):
    from audiolm_pytorch_b200.transformer import Attention, Transformer

    a = Attention(dim=64, heads=4, dim_head=D)
    assert a.dim_head == D and a.to_q.weight.shape == (4 * D, 64) and a.to_kv.weight.shape == (2 * D, 64)
    assert a.to_out[0].weight.shape == (64, 4 * D)
    assert Transformer(dim=64, depth=1, heads=4, dim_head=D).dim_head == D
    assert Transformer(dim=64, depth=1, heads=4).dim_head == 64


@pytest.mark.parametrize("D", [48, 256])
def test_other_widths_raise_with_the_supported_ones_named(D):
    from audiolm_pytorch_b200.audiolm import SemanticTransformer
    from audiolm_pytorch_b200.transformer import Attention

    for make in (lambda: Attention(dim=64, heads=2, dim_head=D),
                 lambda: SemanticTransformer(dim=64, depth=1, heads=2, dim_head=D, num_semantic_tokens=10)):
        with pytest.raises(NotImplementedError, match=r"dim_head in \(32, 64, 128\)"):
            make()


def test_full_width_semantic_model_constructs():
    from audiolm_pytorch_b200.audiolm import SemanticTransformer

    m = SemanticTransformer(dim=1024, depth=6, heads=8, dim_head=128, num_semantic_tokens=500, flash_attn=True)
    assert m.transformer.layers[0][0].branch.to_q.weight.shape == (1024, 1024)


@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("D", WIDTHS)
def test_state_dict_keys_and_shapes_equal_the_reference(D, model):
    g = fixture(D, model)
    for extra, kw in ((False, g["kwargs"]), (True, {**g["kwargs"], "flash_attn": False})):
        want = unpack(g["state"])
        if extra:
            want.update(unpack(g["math_extra"]))
        have = _cls(model)(**kw).state_dict()
        assert set(have) == set(want)
        assert {k: tuple(v.shape) for k, v in have.items()} == {k: tuple(v.shape) for k, v in want.items()}
        kv = [k for k in have if k.endswith("to_kv.weight")]
        assert kv and all(have[k].shape[0] == 2 * D for k in kv)


@pytest.mark.parametrize("D", WIDTHS)
def test_fixture_self_checks(D):
    """the reference's cached forward equals its full forward, and the fixture is finite and complete"""
    g = fixture(D, "semantic")
    f = g["transformer"]
    assert f["cache9"].shape == (2, 2, 2, 9, D)
    assert torch.allclose(f["out_inc"], f["out"][:, 9:], atol=1e-4)
    for model in MODELS:
        g = fixture(D, model)
        assert g["kwargs"]["dim_head"] == D and torch.isfinite(g["loss"])
        grads, state = unpack(g["grads"]), unpack(g["state"])
        assert set(grads) <= set(state) and all(torch.isfinite(v).all() for v in grads.values())
        assert all(grads[k].shape == state[k].shape for k in grads)


def test_new_entry_points_are_declared_and_exported():
    from audiolm_pytorch_b200 import _lib

    header = (ROOT / "include" / "alm_b200.h").read_text()
    lib = _lib.load()
    for name in NEW_SYMBOLS:
        assert re.search(rf"\b{name}\(", header), name
        assert getattr(lib, name) is not None
    assert lib.alm_decode_stack_plan_dh(1, 512, 8, 1365, 6, 128, None) == -4   # ALM_ERR_UNSUPPORTED, before any device call


def test_ops_signatures_keep_their_defaults():
    from audiolm_pytorch_b200 import ops

    def defaults(fn):
        return {k: p.default for k, p in inspect.signature(fn).parameters.items()}

    assert defaults(ops.mqa_attn_fwd) == dict(q=inspect._empty, k=inspect._empty, v=inspect._empty,
                                              heads=inspect._empty, key_mask=None, causal=True, scale=None,
                                              return_lse=True, bias=None, dropout=None)
    assert defaults(ops.mqa_attn_bwd)["scale"] is None and "dim_head" not in defaults(ops.mqa_attn_bwd)
    assert list(defaults(ops.kv_append)) == ["kv_new", "k_cache", "v_cache", "cache_len"]
    assert defaults(ops.mqa_attn_decode)["scale"] is None and defaults(ops.mqa_attn_decode)["splits"] is None
    assert defaults(ops.decode_stack_plan)["dim_head"] == 64
    assert ops.ATTN_HEAD_WIDTHS == (32, 64, 128)
