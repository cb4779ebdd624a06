"""ctypes binding of libalm_b200.so (the C ABI declared in include/alm_b200.h).

There is no fallback: if the library is missing or a call fails, we raise.  The only torch
objects that cross this boundary are raw `data_ptr()`s and the current CUDA stream handle.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

import torch

_PKG = Path(__file__).resolve().parent
LIB_PATH = _PKG / "libalm_b200.so"

P = C.c_void_p
I = C.c_int
L = C.c_int64
F = C.c_float
U32 = C.c_uint32
U64 = C.c_uint64
DROP = [F, U64, U32]  # dropout_p, seed, site

# name -> argtypes (stream is always last and always a void*)
SIGNATURES: dict[str, list] = {
    "alm_gemm_bf16": [P, I, L, L, P, I, L, L, P, I, L, L, I, I, I, I, F, P, I, I, P],
    "alm_mqa_attn_fwd": [P, L, P, L, L, P, L, L, P, P, L, P, L, P, L, L, I, I, I, I, I, F, *DROP, P],
    "alm_mqa_attn_bwd": [P, L, P, L, L, P, L, L, P, L, P, P, P, I, P, L, P, P, L, P, L, P, P, L, L, I, I, I, I, I, F, *DROP,
                         P],
    "alm_pack_key_mask": [P, P, I, I, P],
    "alm_embed_gather": [P, I, P, P, I, I, P],
    "alm_embed_scatter": [P, I, P, P, I, I, P],
    "alm_attn_delta": [P, L, P, L, P, L, P, I, I, I, P],
    "alm_kv_append": [P, L, P, P, L, P, I, I, P],
    # the same calls with the head width (dim_head in {32, 64, 128}) as the last argument before the stream
    "alm_mqa_attn_fwd_dh": [P, L, P, L, L, P, L, L, P, P, L, P, L, P, L, L, I, I, I, I, I, F, *DROP, I, P],
    "alm_mqa_attn_bwd_dh": [P, L, P, L, L, P, L, L, P, L, P, P, P, I, P, L, P, P, L, P, L, P, P, L, L, I, I, I, I, I, F,
                            *DROP, I, P],
    "alm_attn_delta_dh": [P, L, P, L, P, L, P, I, I, I, I, P],
    "alm_kv_append_dh": [P, L, P, P, L, P, I, I, I, P],
    "alm_mqa_attn_decode_dh": [P, L, P, P, L, P, I, P, L, P, L, P, L, P, I, I, I, F, I, P],
    "alm_gemv_bf16": [P, L, P, L, P, I, L, P, I, I, I, P],
    "alm_gemm_head_ce": [P, L, P, L, P, P, L, I, P, P, P, P, P, P, L, I, I, I, P],
    "alm_ce_finish": [P, I, P, P, L, P, P, I, P],
    "alm_decode_stack_step": [P, I, P, P, P, P, I, L, P, L, P, L, I, I, I, I, I, F, I, P],
    "alm_mqa_attn_decode": [P, L, P, P, L, P, I, P, L, P, L, P, L, P, I, I, I, F, P],
    "alm_decode_bias_row": [P, I, P, P, P, I, P, I, P, L, I, P],
    "alm_bias_gather_fwd": [P, P, P, P, I, I, I, L, P],
    "alm_bias_gather_bwd": [P, P, P, P, I, I, I, L, P],
    "alm_hc_pre_fwd": [P] * 12 + [P, P, P, P, P, I, I, I, P],
    "alm_hc_pre_bwd": [P] * 12 + [P, P, P, P, P, P, P, P, P, F] + [P] * 8 + [I, I, I, P],
    "alm_hc_post_fwd": [P, P, P, P, P, P, I, I, I, P],
    "alm_hc_post_bwd": [P, P, P, P, P, P, P, P, P, P, I, I, I, P],
    "alm_geglu_ln_fwd": [P, L, I, P, P, L, P, I, I, I, *DROP, P],
    "alm_geglu_ln_bwd": [P, L, I, P, P, P, L, P, P, I, I, I, *DROP, P],
    "alm_dropout_bf16": [P, L, L, I, *DROP, P],
    "alm_ce_fwd_bwd": [P, L, P, L, P, P, L, P, P, I, I, I, P],
    "alm_axpby_bf16": [P, L, F, P, L, F, P, L, L, I, P],
    "alm_cast_pad_bf16": [P, L, P, L, L, I, I, P],
    "alm_cast_pad_multi": [P, I, P],
    "alm_scale_by_scalar_bf16": [P, P, L, P],
    "alm_topk_gumbel_sample": [P, L, P, L, P, I, I, I, F, P],
    "alm_resid_ln_fwd": [P, P, P, P, P, P, P, I, I, P],
    "alm_resid_ln_bwd": [P, P, P, P, P, P, P, P, P, F, I, I, P],
    "alm_residual_unit_fwd": [P, P, P, P, P, P, I, I, I, I, I, P],
    "alm_causal_conv1d_fwd": [P, P, P, P, P, I, I, I, I, I, I, I, I, I, I, P],
    "alm_causal_convT1d_fwd": [P, P, P, P, I, I, I, I, I, P],
    "alm_codec_first_conv": [P, P, P, P, I, I, I, I, I, P],
    "alm_codec_ru_tc": [P, P, P, P, P, I, I, I, I, I, I, P],
    "alm_codec_ru_se_tc": [P, P, P, P, P, P, P, I, I, I, I, I, I, I, P],
    "alm_codec_se_fp32": [P, P, P, P, P, P, P, I, I, I, I, P],
    "alm_codec_conv_tc": [P, P, P, P, I, I, I, I, I, I, I, I, I, I, P],
    "alm_codec_pack_c8s": [P, P, I, I, I, P],
    "alm_codec_last_conv": [P, P, P, P, I, I, I, I, I, P],
    "alm_codec_gate_loop_fp32": [P, P, P, P, I, I, I, P],
    "alm_codec_gate_loop_tc": [P, P, P, P, I, I, I, P],
    "alm_rvq_encode": [P, L, P, P, P, L, P, L, I, I, I, I, P],
    "alm_rvq_pack_codebooks": [P, P, P, L, I, P],
    "alm_rvq_prepare": [P, L, P, P, L, P, I, I, I, P],
    "alm_rvq_select": [P, L, P, P, P, P, L, P, P, L, I, I, I, I, P],
    "alm_rvq_prepare_cos": [P, L, P, P, L, P, I, I, I, P],
    "alm_rvq_select_cos": [P, L, P, P, P, P, L, P, P, L, I, I, I, I, P],
    "alm_split_rows": [P, L, P, I, I, P],
    "alm_rvq_decode": [P, L, P, P, L, I, I, I, I, P],
    "alm_sq_encode": [P, L, I, I, I, I, P, P, P, P, P, P, I, I, P, L, P, I, P],
    "alm_sq_decode": [P, I, I, I, I, I, I, P, P, P, P, I, I, P, L, P],
    "alm_hubert_conv0": [P, P, P, P, I, I, I, I, I, P],
    "alm_hubert_chan_stats": [P, P, I, I, I, P],
    "alm_hubert_norm_act": [P, P, I, P, L, P, P, I, P, P, L, I, P],
    "alm_hubert_add_ln": [P, P, I, I, P, I, P, P, I, P, P, L, I, P],
    "alm_hubert_pos_pack": [P, P, I, I, I, I, I, I, P],
    "alm_hubert_qkv_heads": [P, P, P, P, I, I, I, I, P],
    "alm_hubert_merge_heads": [P, P, I, I, I, I, P],
    "alm_w2v_group_stats": [P, P, P, I, I, I, I, P],
    "alm_w2v_norm_act": [P, P, P, P, I, P, I, I, F, I, P, P, I, I, I, I, P],
    "alm_encodec_pad1d": [P, P, L, I, I, I, P],
    "alm_encodec_resblock_fp32": [P, P, P, P, P, P, P, I, I, I, I, P],
    "alm_encodec_lstm": [P, P, P, P, P, I, I, I, I, P],
    "alm_encodec_resblock_tc": [P, P, P, P, P, I, I, I, I, I, P],
    "alm_resample": [P, L, L, P, L, L, I, P, P, I, I, I, P],
}


class AlmError(RuntimeError):
    pass


_lib = None


def load() -> C.CDLL:
    """Load the shared library (building is explicit: `python -m audiolm_pytorch_b200.build`)."""
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        raise AlmError(
            f"{LIB_PATH} not found. Build it with `python -m audiolm_pytorch_b200.build` "
            "(there is no CPU / PyTorch fallback for the hot path)."
        )
    lib = C.CDLL(str(LIB_PATH), mode=os.RTLD_LOCAL | os.RTLD_NOW)
    lib.alm_version.restype = I
    lib.alm_status_string.restype = C.c_char_p
    lib.alm_status_string.argtypes = [I]
    lib.alm_launch_count.restype = C.c_ulonglong
    lib.alm_reset_launch_count.restype = None
    lib.alm_decode_stack_scratch_bytes.restype = L
    lib.alm_decode_stack_scratch_bytes.argtypes = [I, I, I, I]
    lib.alm_gemm_head_ce_tiles.restype = I
    lib.alm_gemm_head_ce_tiles.argtypes = [I]
    lib.alm_codec_gate_loop_workspace.restype = C.c_longlong
    lib.alm_codec_gate_loop_workspace.argtypes = [I, I, I, I]
    lib.alm_encodec_lstm_workspace.restype = C.c_longlong
    lib.alm_encodec_lstm_workspace.argtypes = [I, I]
    lib.alm_decode_stack_grid.restype = I
    lib.alm_decode_stack_grid.argtypes = []
    lib.alm_decode_stack_plan.restype = I
    lib.alm_decode_stack_plan.argtypes = [I, I, I, I, I, P]
    lib.alm_decode_stack_plan_dh.restype = I
    lib.alm_decode_stack_plan_dh.argtypes = [I, I, I, I, I, I, P]
    lib.alm_decode_stack_trace_offset.restype = L
    lib.alm_decode_stack_trace_offset.argtypes = [I, I, I, I]
    for name, argtypes in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.argtypes = argtypes
        fn.restype = I
    _lib = lib
    return lib


def ptr(t) -> int | None:
    if t is None:
        return None
    return t.data_ptr()


def stream_handle() -> int:
    return torch.cuda.current_stream().cuda_stream


def call(name: str, *args) -> None:
    """Invoke `name(*args, current_stream)`; tensors are passed by address."""
    lib = load()
    conv = []
    for a in args:
        if isinstance(a, torch.Tensor):
            if not a.is_cuda:
                raise AlmError(f"{name}: got a {a.device} tensor; the hot path has no CPU implementation")
            conv.append(a.data_ptr())
        else:
            conv.append(a)
    rc = getattr(lib, name)(*conv, stream_handle())
    if rc != 0:
        raise AlmError(f"{name} failed: {lib.alm_status_string(rc).decode()} ({rc})")


def launch_count() -> int:
    return int(load().alm_launch_count())


def reset_launch_count() -> None:
    load().alm_reset_launch_count()
