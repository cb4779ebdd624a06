"""H100: hyper-connections with 2 to 8 residual streams — the four ops against fp32 autograd (and the in-kernel
parameter gradients against fp64), the 4-stream ring backward at C3-sized token counts, the models against the
reference goldens of tests/golden/streams.pt, KV-cache decoding on the engine, and the training plumbing."""
import sys
from pathlib import Path

import pytest
import torch
import torch.nn.functional as F

from oracle import golden

sys.path.insert(0, str(Path(__file__).resolve().parent))
from test_models_gpu import check_grads, rms_rel  # noqa: E402
from test_ops_gpu import DEV, bf16, hc_ref, make_hc, rel_err  # noqa: E402

pytestmark = pytest.mark.gpu

C3_TAIL = 8 * 2048 + 37  # wraps the backward's ring many times; not a multiple of the grid


def _inputs(M, S, d, expand, seed):
    torch.manual_seed(seed)
    if expand:
        x = torch.randn(M, d, device=DEV)
        return dict(x_expand=x), dict(x=x)
    R_in = torch.randn(M, S, d, device=DEV).to(bf16)
    Y = torch.randn(M, d, device=DEV).to(bf16)
    bp = 1 + 0.2 * torch.randn(M, S, device=DEV)
    return dict(R_in=R_in, Y=Y, beta_prev=bp), dict(R_in=R_in, Y=Y, bp=bp)


def _reference(hc, ln_gamma, raw, expand, S, d, M, dtype, w):
    """forward outputs and autograd of hc_ref in `dtype`: (outputs, data-input grads, hc grads, ln_gamma grad)"""
    hc_leaf = {k: v.to(dtype).clone().requires_grad_(True) for k, v in hc.items()}
    lng_leaf = ln_gamma.to(dtype).clone().requires_grad_(True)
    if expand:
        x_leaf = raw["x"].to(dtype).clone().requires_grad_(True)
        R = x_leaf[:, None, :].expand(M, S, d)
        data = (x_leaf,)
    else:
        data = tuple(raw[k].to(dtype).clone().requires_grad_(True) for k in ("R_in", "Y", "bp"))
        R = data[0] + data[2][..., None] * data[1][:, None, :]
    outs = hc_ref(hc_leaf, lng_leaf, R, d)
    r_out, r_bin, r_xn, r_beta = outs
    w1, w2, w3, w4 = w
    loss = (r_out * w1.to(dtype)).sum() + (r_xn * w2.to(dtype)).sum() + (r_beta * w4.to(dtype)).sum()
    if w3 is not None:
        loss = loss + (r_bin * w3.to(dtype)).sum()
    loss.backward()
    return ([o.detach() for o in outs], [t.grad for t in data], {k: v.grad for k, v in hc_leaf.items()},
            lng_leaf.grad)


@pytest.mark.parametrize("S", [2, 3, 4, 5, 6, 7, 8])
@pytest.mark.parametrize("d", [64, 1000, 1024, 2048])
@pytest.mark.parametrize("expand", [False, True])
def test_hc_pre_fwd_bwd_streams(S, d, expand):
    from audiolm_pytorch_b200 import ops

    M = C3_TAIL if d <= 1024 else 777
    hc, ln_gamma = make_hc(d, S=S, seed=S * 100 + d)
    kin, raw = _inputs(M, S, d, expand, S + d)
    R_out, bin_, xn, beta, aux = ops.hc_pre_fwd(hc, ln_gamma, **kin, M=M, d=d, streams=S)
    assert R_out.shape == (M, S, d) and beta.shape == (M, S) and aux.shape == (M, ops.hc_aux_floats(S))
    w = (torch.randn(M, S, d, device=DEV).to(bf16), torch.randn(M, d, device=DEV).to(bf16),
         torch.randn(M, d, device=DEV).to(bf16), torch.randn(M, S, device=DEV))
    for with_dbin in (True, False):
        ww = w if with_dbin else (*w[:2], None, w[3])
        outs, ref_data, ref_hc, ref_ln = _reference(hc, ln_gamma, raw, expand, S, d, M, torch.float32, ww)
        if with_dbin:  # the bounds of test_ops_gpu.py::test_hc_pre_fwd_bwd
            for got, ref, tol in zip((R_out, bin_, xn, beta), outs, (1e-2, 1e-2, 1.5e-2, 1e-3)):
                assert rel_err(got, ref) < tol
        grads = {k: torch.zeros_like(v) for k, v in hc.items()}
        g_ln = torch.zeros_like(ln_gamma)
        if expand:
            dx = ops.hc_pre_bwd(hc, ln_gamma, grads, g_ln, aux, w[0], w[1], w[3], dbin_extra=ww[2],
                                x_expand=kin["x_expand"], dx_scale=0.1, M=M, d=d, streams=S)
            assert rel_err(dx, 0.1 * ref_data[0]) < 2e-2
        else:
            dR_in, dY, dbp = ops.hc_pre_bwd(hc, ln_gamma, grads, g_ln, aux, w[0], w[1], w[3], dbin_extra=ww[2], **kin,
                                            M=M, d=d, streams=S)
            assert rel_err(dR_in, ref_data[0]) < 2e-2
            assert rel_err(dY, ref_data[1]) < 2e-2
            assert rel_err(dbp, ref_data[2]) < 2e-2
        torch.cuda.synchronize()
        for k in hc:
            assert rel_err(grads[k], ref_hc[k]) < 3e-2, (k, with_dbin)
        assert rel_err(g_ln, ref_ln) < 3e-2


@pytest.mark.parametrize("S", [2, 4, 5, 8])
@pytest.mark.parametrize("d", [64, 1000, 1024])
@pytest.mark.parametrize("dc,expand", [(1024.0, False), (1024.0, True), (8192.0, True)])
def test_hc_pre_fwd_dc_offset(S, d, dc, expand):
    """branch inputs with a DC offset on the second-generation forward (d <= 1024: S <= 4 at one and two chunks per
    thread, S >= 5 at 128 threads per token): R_in = dc with the variation carried by Y, or x_expand = dc + noise.
    xn and the LayerNorm statistics in aux against an fp64 hc_ref; a variance taken as E[x^2] - mean^2 in fp32 is
    rounding noise on these rows.  (With R_in = 8192 the fp32 residual R_in + beta Y itself carries 2^-11 per element,
    more than the bound allows once the stream weights nearly cancel.)"""
    from audiolm_pytorch_b200 import ops

    M = 777
    hc, ln_gamma = make_hc(d, S=S, seed=S + d)
    kin, raw = _inputs(M, S, d, expand, S * d)
    if expand:
        kin["x_expand"] = raw["x"] = raw["x"] + dc
    else:
        kin["R_in"] = raw["R_in"] = torch.full_like(raw["R_in"], dc)
    _, _, xn, _, aux = ops.hc_pre_fwd(hc, ln_gamma, **kin, M=M, d=d, streams=S)
    hc64 = {k: v.double() for k, v in hc.items()}
    R = (raw["x"].double()[:, None, :].expand(M, S, d) if expand
         else raw["R_in"].double() + raw["bp"].double()[..., None] * raw["Y"].double()[:, None, :])
    _, bin_ref, xn_ref, _ = hc_ref(hc64, ln_gamma.double(), R, d)
    rstd_ref = (bin_ref.var(-1, unbiased=False) + 1e-5).rsqrt()
    # the rows are ill-conditioned (less than dc where the branch's stream weights nearly cancel)
    assert (bin_ref.mean(-1).abs() / bin_ref.std(-1, unbiased=False)).min() > dc / 64
    assert rel_err(xn, xn_ref) < 1.5e-2
    assert ((aux[:, -1].double() - rstd_ref).abs() / rstd_ref).max().item() < 1e-2


@pytest.mark.parametrize("S", [2, 3, 5, 8])
@pytest.mark.parametrize("d,expand", [(1024, False), (1000, True), (2048, False)])
def test_hc_param_grads_vs_fp64_streams(S, d, expand):
    """the in-kernel fp32 parameter-gradient sums against an fp64 restatement of the whole op (printed with -s)"""
    from audiolm_pytorch_b200 import ops

    M = C3_TAIL if d <= 1024 else 777
    hc, ln_gamma = make_hc(d, S=S, seed=7 + S)
    kin, raw = _inputs(M, S, d, expand, 11 + S)
    aux = ops.hc_pre_fwd(hc, ln_gamma, **kin, M=M, d=d, streams=S)[4]
    w = (torch.randn(M, S, d, device=DEV).to(bf16), torch.randn(M, d, device=DEV).to(bf16),
         torch.randn(M, d, device=DEV).to(bf16), torch.randn(M, S, device=DEV))
    _, _, ref_hc, ref_ln = _reference(hc, ln_gamma, raw, expand, S, d, M, torch.float64, w)
    grads = {k: torch.zeros_like(v) for k, v in hc.items()}
    g_ln = torch.zeros_like(ln_gamma)
    ops.hc_pre_bwd(hc, ln_gamma, grads, g_ln, aux, w[0], w[1], w[3], dbin_extra=w[2], **kin,
                   **({"dx_scale": 1.0} if expand else {}), M=M, d=d, streams=S)
    torch.cuda.synchronize()
    errs = {k: rel_err(grads[k], ref_hc[k]) for k in hc}
    errs["ln_gamma"] = rel_err(g_ln, ref_ln)
    print(f"\nS={S} d={d} expand={expand} parameter-gradient error vs fp64:",
          " ".join(f"{k}={v:.2e}" for k, v in errs.items()))
    for k, v in errs.items():
        assert v < 1e-2, k


# ---------------------------------------------------------------------------------------------------------------------
# the 4-stream backward on the shared-memory ring (d <= 1024) and the forward without `bin`: token counts that wrap the
# ring many times, odd d, no dbin_extra, expand mode
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,d,expand,with_dbin", [(C3_TAIL, 1024, False, True), (C3_TAIL, 1024, False, False),
                                                  (3001, 1000, False, True), (517, 64, False, False),
                                                  (C3_TAIL, 1024, True, True), (777, 1000, True, False)])
def test_hc_pre_bwd_ring(M, d, expand, with_dbin):
    from audiolm_pytorch_b200 import ops

    S = 4
    hc, ln_gamma = make_hc(d, seed=d + 1)
    kin, raw = _inputs(M, S, d, expand, M + d)
    R_out, bin_, xn, beta, aux = ops.hc_pre_fwd(hc, ln_gamma, **kin, M=M, d=d)
    w1 = torch.randn(M, S, d, device=DEV).to(bf16)
    w2 = torch.randn(M, d, device=DEV).to(bf16)
    w3 = torch.randn(M, d, device=DEV).to(bf16) if with_dbin else None
    w4 = torch.randn(M, S, device=DEV)
    _, ref_data, ref_hc, ref_ln = _reference(hc, ln_gamma, raw, expand, S, d, M, torch.float32, (w1, w2, w3, w4))
    grads = {k: torch.zeros_like(v) for k, v in hc.items()}
    g_ln = torch.zeros_like(ln_gamma)
    if expand:
        dx = ops.hc_pre_bwd(hc, ln_gamma, grads, g_ln, aux, w1, w2, w4, dbin_extra=w3, x_expand=kin["x_expand"],
                            dx_scale=0.1, M=M, d=d)
        assert rel_err(dx, 0.1 * ref_data[0]) < 2e-2
    else:
        dR_in, dY, dbp = ops.hc_pre_bwd(hc, ln_gamma, grads, g_ln, aux, w1, w2, w4, dbin_extra=w3, **kin, M=M, d=d)
        assert rel_err(dR_in, ref_data[0]) < 2e-2
        assert rel_err(dY, ref_data[1]) < 2e-2
        assert rel_err(dbp, ref_data[2]) < 2e-2
    torch.cuda.synchronize()
    for k in hc:
        assert rel_err(grads[k], ref_hc[k]) < 3e-2, k
    assert rel_err(g_ln, ref_ln) < 3e-2


@pytest.mark.parametrize("M,d,expand", [(C3_TAIL, 1024, False), (3001, 1000, True)])
def test_hc_param_grads_vs_fp64(M, d, expand):
    """The per-channel parameter gradients are summed in fp32 inside the kernel; their error against an fp64
    restatement of the whole op is printed (pytest -s) and bounded."""
    from audiolm_pytorch_b200 import ops

    S = 4
    hc, ln_gamma = make_hc(d, seed=7)
    kin, raw = _inputs(M, S, d, expand, 11)
    _, _, _, _, aux = ops.hc_pre_fwd(hc, ln_gamma, **kin, M=M, d=d)
    w = (torch.randn(M, S, d, device=DEV).to(bf16), torch.randn(M, d, device=DEV).to(bf16),
         torch.randn(M, d, device=DEV).to(bf16), torch.randn(M, S, device=DEV))
    _, _, ref_hc, ref_ln = _reference(hc, ln_gamma, raw, expand, S, d, M, torch.float64, w)
    grads = {k: torch.zeros_like(v) for k, v in hc.items()}
    g_ln = torch.zeros_like(ln_gamma)
    ops.hc_pre_bwd(hc, ln_gamma, grads, g_ln, aux, w[0], w[1], w[3], dbin_extra=w[2], **kin,
                   **({"dx_scale": 1.0} if expand else {}), M=M, d=d)
    torch.cuda.synchronize()
    errs = {k: rel_err(grads[k], ref_hc[k]) for k in hc}
    errs["ln_gamma"] = rel_err(g_ln, ref_ln)
    print("\nparameter-gradient error vs fp64 (max abs / max |ref|):",
          " ".join(f"{k}={v:.2e}" for k, v in errs.items()))
    for k, v in errs.items():
        assert v < 1e-2, k


@pytest.mark.parametrize("M,d,expand", [(C3_TAIL, 1024, False), (300, 1000, False), (200, 1024, True)])
def test_hc_pre_fwd_without_bin(M, d, expand):
    from audiolm_pytorch_b200 import ops

    hc, ln_gamma = make_hc(d, seed=3)
    kin, _ = _inputs(M, 4, d, expand, 5)
    full = ops.hc_pre_fwd(hc, ln_gamma, **kin, M=M, d=d)
    lean = ops.hc_pre_fwd(hc, ln_gamma, **kin, M=M, d=d, want_bin=False)
    assert full[1] is not None and lean[1] is None
    for i in (0, 2, 3, 4):
        assert torch.equal(full[i], lean[i]), i


@pytest.mark.parametrize("S", [2, 3, 5, 8])
@pytest.mark.parametrize("d", [64, 1000, 1024, 2048])
def test_hc_post_fwd_bwd_streams(S, d):
    from audiolm_pytorch_b200 import ops

    M = C3_TAIL if d <= 1024 else 777
    torch.manual_seed(M + S)
    R_in = torch.randn(M, S, d, device=DEV).to(bf16)
    Y = torch.randn(M, d, device=DEV).to(bf16)
    bp = 1 + 0.2 * torch.randn(M, S, device=DEV)
    lng = 1 + 0.1 * torch.randn(d, device=DEV)
    Ri, Yl, bpl, gl = (t.float().clone().requires_grad_(True) for t in (R_in, Y, bp, lng))
    ref = F.layer_norm((Ri + bpl[..., None] * Yl[:, None, :]).sum(1), (d,)) * gl
    out, stats = ops.hc_post_fwd(R_in, Y, bp, lng, M=M, d=d, streams=S)
    assert rel_err(out, ref) < 1.5e-2
    w = torch.randn(M, d, device=DEV).to(bf16)
    (ref * w.float()).sum().backward()
    g_ln = torch.zeros_like(lng)
    dR, dY, dbp = ops.hc_post_bwd(R_in, Y, bp, lng, stats, w, g_ln, M=M, d=d, streams=S)
    assert dR.shape == (M, S, d) and dbp.shape == (M, S)
    assert rel_err(dR, Ri.grad) < 2e-2
    assert rel_err(dY, Yl.grad) < 2e-2
    assert rel_err(dbp, bpl.grad) < 2e-2
    assert rel_err(g_ln, gl.grad) < 2e-2


# ---------------------------------------------------------------------------------------------------------------------
# models vs the reference goldens
# ---------------------------------------------------------------------------------------------------------------------
def _model(key):
    from audiolm_pytorch_b200 import audiolm

    g = golden.load("streams.pt")[key]
    cls = audiolm.SemanticTransformer if g["kind"] == "semantic" else audiolm.CoarseTransformer
    m = cls(**g["kwargs"])
    m.load_state_dict(g["state"], strict=True)
    return m.to(DEV), g


@pytest.mark.parametrize("key", ["semantic_s2", "semantic_s3", "semantic_s8"])
def test_semantic_streams_vs_golden(key):
    from audiolm_pytorch_b200.audiolm import SemanticTransformerWrapper

    m, g = _model(key)
    m.eval()
    ids = g["ids"].to(DEV)
    with torch.no_grad():
        logits = m(ids=ids)
        masked = m(ids=ids, self_attn_mask=g["mask"].to(DEV))
        _, cache = m(ids=ids[:, :12], return_kv_cache=True)
        inc, _ = m(ids=ids, kv_cache=cache, return_kv_cache=True)
    # 1e-2 RMS, or twice the deviation of the reference's own bf16-autocast logits where that is larger (8 streams
    # summed through a bf16 residual), as check_grads bounds the gradients
    tol, tol_m = (max(1e-2, 2.0 * n) for n in g["logits_bf16_noise"])
    err, err_m = rms_rel(logits, g["logits"]), rms_rel(masked, g["logits_masked"])
    print(f"\n{key} logits rms err {err:.4f} (tol {tol:.4f}), masked {err_m:.4f} (tol {tol_m:.4f})")
    assert err < tol and err_m < tol_m
    assert rms_rel(inc, logits[:, 13:]) < 1.5e-2
    w = SemanticTransformerWrapper(transformer=m, unique_consecutive=False, mask_prob=0.0).train()
    loss = w(semantic_token_ids=ids, return_loss=True)
    assert abs(loss.item() - g["loss"].item()) < 2e-2 * abs(g["loss"].item())
    loss.backward()
    check_grads(dict(m.named_parameters()), g["grads"], g["bf16_noise"])


def test_coarse_streams_bias_vs_golden():
    """2 streams with flash_attn=False: the relative-position and cross-segment biases next to hyper-connections"""
    from audiolm_pytorch_b200.audiolm import CoarseTransformerWrapper

    m, g = _model("coarse_s2")
    m.eval()
    sem, co = g["sem"].to(DEV), g["coarse"].to(DEV)
    with torch.no_grad():
        sl, cl = m(semantic_token_ids=sem, coarse_token_ids=co)
        _, clm = m(semantic_token_ids=sem, coarse_token_ids=co, self_attn_mask=g["mask"].to(DEV))
    assert rms_rel(sl, g["sem_logits"]) < 1e-2 and rms_rel(cl, g["coarse_logits"]) < 1e-2
    assert rms_rel(clm, g["coarse_logits_masked"]) < 1e-2

    class _Codec:  # the wrapper constructor only reads rq_groups
        rq_groups = 1

    w = CoarseTransformerWrapper(transformer=m, codec=_Codec(), unique_consecutive=False, mask_prob=0.0).train()
    loss = w(semantic_token_ids=sem, coarse_token_ids=g["frames"].to(DEV), return_loss=True)
    assert abs(loss.item() - g["loss"].item()) < 2e-2 * abs(g["loss"].item())
    loss.backward()
    check_grads(dict(m.named_parameters()), g["grads"], g["bf16_noise"])


# ---------------------------------------------------------------------------------------------------------------------
# KV-cache decoding on the engine (the multi-kernel step: the one-kernel step is built for 4 streams)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("key", ["semantic_s2", "semantic_s8"])
def test_semantic_generate_on_engine_streams(key):
    from audiolm_pytorch_b200.audiolm import SemanticTransformerWrapper

    m, g = _model(key)
    m.eval()
    ids = g["ids"].to(DEV)
    w = SemanticTransformerWrapper(transformer=m, unique_consecutive=False)
    torch.manual_seed(3)
    out = w.generate(max_length=40, prime_ids=ids[:, :5])
    assert w._engine[1]._graphs
    assert torch.equal(out[:, :5], ids[:, :5]) and 5 < out.shape[1] <= 40
    fast = w.generate(max_length=40, prime_ids=ids[:, :5], temperature=1e-4, filter_thres=0.0)
    with torch.no_grad():
        lg = m(ids=fast[:, :-1].clamp(min=0)).float()
    # argmax-mode tokens of the engine against the teacher-forced full forward on the same prefixes
    seq = fast
    valid = seq != -1
    valid[:, :5] = False
    chosen = lg.gather(-1, seq.clamp(min=0)[..., None])[..., 0]
    top = lg.max(dim=-1).values
    exact = (lg.argmax(-1) == seq)[valid].float().mean().item()
    gap = (top - chosen)[valid]
    print(key, "argmax agreement", exact, "largest gap", gap.max().item())
    assert valid.sum() > 0 and exact >= 0.9 and (gap <= 2e-2 * lg.abs().amax(-1)[valid]).all()


@pytest.mark.parametrize("key", ["semantic_s2", "semantic_s8"])
def test_graph_replay_bitwise_and_fused_flag_streams(key, monkeypatch):
    from audiolm_pytorch_b200 import decode
    from audiolm_pytorch_b200.decode import GraphedStep, StackDecoder

    monkeypatch.setattr(decode, "FUSED_STACK_STEP", True)
    m, g = _model(key)
    m.eval()
    ids = g["ids"].to(DEV)
    b, max_len = ids.shape[0], 64
    with torch.no_grad():
        _, kv = m(ids=ids[:, :9], return_kv_cache=True)
        outs = []
        for use_graph in (False, True):
            dec = StackDecoder(m.transformer, b, max_len)
            assert not dec.fused_ok()   # S != 4: the multi-kernel step
            dec.load_cache(kv)
            x = torch.zeros(b, m.transformer.dim, device=DEV)
            y = torch.zeros(b, m.transformer.dim, device=DEV, dtype=bf16)

            def fn():
                y.copy_(dec.step(x))

            step = GraphedStep(fn, [dec.len, y]) if use_graph else fn
            got = []
            for t in range(9, 15):
                x.copy_(m.semantic_embedding(ids[:, t]))
                step()
                got.append(y.clone())
            outs.append(torch.stack(got))
            assert int(dec.len.item()) == 16
    assert torch.equal(outs[0], outs[1])


# ---------------------------------------------------------------------------------------------------------------------
# training plumbing
# ---------------------------------------------------------------------------------------------------------------------
def test_grad_ready_hook_and_dropout_two_streams():
    from audiolm_pytorch_b200.transformer import Transformer

    torch.manual_seed(0)
    tr = Transformer(dim=128, depth=3, heads=2, flash_attn=True, num_residual_streams=2).to(DEV).train()
    fired = []
    tr.grad_ready_hook = fired.append
    x = torch.randn(2, 64, 128, device=DEV)
    w = torch.randn(2, 64, 128, device=DEV)
    tr.accumulate_into_grad = True
    for p in tr.parameters():
        p.grad = torch.zeros_like(p)
    (tr(x).float() * w).sum().backward()
    assert fired == [2, 1, 0]
    assert all(torch.isfinite(p.grad).all() for p in tr.parameters())

    torch.manual_seed(1)
    trd = Transformer(dim=128, depth=2, heads=2, flash_attn=True, num_residual_streams=2, attn_dropout=0.1,
                      ff_dropout=0.1).to(DEV).train()
    (trd(x).float() * w).sum().backward()
    assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in trd.parameters())
    assert all(p.grad.abs().sum() > 0 for name, p in trd.named_parameters() if name.endswith(".weight"))
