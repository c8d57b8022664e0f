"""`torch.ops.hstu.*` registration of the H100 attention: the reference's OWN native operator schema.

The reference's C++ extension declares three operators in the `hstu` namespace
(generative_recommenders/ops/cpp/hstu_attention/flash_api.cpp:275-365): `hstu_mha` (autograd), `hstu_mha_fwd`, `hstu_mha_bwd`,
implemented there for sm80 / sm90.  `register()` defines the same schemas (as a library FRAGMENT, so it coexists with an
already-loaded reference extension only if that one is absent -- a second definition of the same operator is an error) and
routes them to libhstu_b200.so, so code written against `torch.ops.hstu.hstu_mha(...)` runs on H100 unchanged.

Arguments this backend does not implement raise instead of being ignored: `attn_scale` and the dense layout
(`seq_offsets=None`).
`causal=False` (the reference CUDA op's default) runs the non-causal attention under the reference eager path's
causal=False mask (ops/hstu_attention.py `causal=False`), forward and backward; it takes no fp8 inputs.
fp8: with q, k and v of dtype float8_e4m3fn, `hstu_mha_fwd` and `hstu_mha` run the fp8 forward (`hstu_attn_fwd_fp8`) and
return bf16: the attention of q * q_descale[b, h], k * k_descale[b, h], v * v_descale[b, h], each descale an fp32 [B, H]
tensor or None for 1, as in the reference's e4m3 forward.  Head dims: dqk == dv, or dqk < dv (the DLRM-HSTU default
attention_dim 128 / hidden_dim 256 included), both in {32, 64, 128, 256}.  There is no fp8 backward: `hstu_mha` raises when a
gradient is requested through fp8 inputs.  Descales with bf16 / fp16 inputs raise.
`deterministic=True` (or `torch.use_deterministic_algorithms(True)`) makes the backward bitwise reproducible: the wgmma
backward then runs its atomic-free dK / dV and dQ kernels, and shapes it does not cover run the generic kernels, which have
no atomics either.  Otherwise the wgmma backward at d = 64 / 128 accumulates dQ with fp32 atomic adds whose order varies
from run to run (fp32, ~1e-7 relative); at d = 32 it is atomic-free either way.
`sort_by_length` / `sm_margin` are accepted and ignored (the kernels always schedule heavy tiles first and use every SM).
"""
from typing import List, Optional

import torch

from . import _lib
from .ops.hstu_attention import _FP8, _HSTUAttentionFunction, cuda_hstu_attention_bwd, cuda_hstu_attention_fwd

_LIB = None

_MHA = ("hstu_mha(SymInt max_seq_len, float alpha, Tensor q, Tensor k, Tensor v, Tensor? seq_offsets, bool causal, "
        "Tensor? num_targets, Tensor? attn_scale, int max_attn_len, int min_full_attn_seq_len, int contextual_seq_len, "
        "Tensor? q_descale, Tensor? k_descale, Tensor? v_descale, bool sort_by_length, bool deterministic, int sm_margin) -> Tensor")
_FWD = ("hstu_mha_fwd(SymInt max_seq_len, float alpha, Tensor q, Tensor k, Tensor v, Tensor? seq_offsets, bool causal, "
        "Tensor? num_targets, Tensor? attn_scale, int max_attn_len, int min_full_attn_seq_len, int contextual_seq_len, "
        "Tensor? q_descale, Tensor? k_descale, Tensor? v_descale, int sm_margin) -> Tensor")
_BWD = ("hstu_mha_bwd(int max_seq_len, float alpha, Tensor dout, Tensor q, Tensor k, Tensor v, Tensor dq, Tensor dk, Tensor dv, "
        "Tensor? seq_offsets, bool causal, Tensor? num_targets, Tensor? attn_scale, int max_attn_len, int min_full_attn_seq_len, "
        "int contextual_seq_len, bool sort_by_length, bool deterministic, int sm_margin) -> Tensor[]")


def _check(causal, seq_offsets, attn_scale, descales, qkv=()):
    if seq_offsets is None:
        raise RuntimeError("hstu::hstu_mha on H100: the dense (seq_offsets=None) layout is not implemented; pass jagged tensors")
    if attn_scale is not None:
        raise RuntimeError("hstu::hstu_mha on H100: attn_scale is not implemented")
    if any(d is not None for d in descales) and not (qkv and all(t.dtype == _FP8 for t in qkv)):
        raise RuntimeError("hstu::hstu_mha on H100: q,k,v_descale apply to float8_e4m3fn q, k and v only "
                           f"(got {', '.join(str(t.dtype) for t in qkv) or 'no inputs'})")


def _fwd(max_seq_len, alpha, q, k, v, seq_offsets, causal, num_targets, attn_scale, max_attn_len, min_full_attn_seq_len,
         contextual_seq_len, q_descale, k_descale, v_descale, sm_margin):
    descales = (q_descale, k_descale, v_descale)
    _check(causal, seq_offsets, attn_scale, descales, (q, k, v))
    return cuda_hstu_attention_fwd(int(max_seq_len), alpha, q, k, v, seq_offsets, num_targets, max_attn_len, contextual_seq_len,
                                   min_full_attn_seq_len, descales=descales if any(t.dtype == _FP8 for t in (q, k, v)) else None,
                                   causal=bool(causal))


def _bwd(max_seq_len, alpha, dout, q, k, v, dq, dk, dv, seq_offsets, causal, num_targets, attn_scale, max_attn_len,
         min_full_attn_seq_len, contextual_seq_len, sort_by_length, deterministic, sm_margin) -> List[torch.Tensor]:
    _check(causal, seq_offsets, attn_scale, ())
    cuda_hstu_attention_bwd(int(max_seq_len), alpha, dout, q, k, v, dq, dk, dv, seq_offsets, num_targets, max_attn_len,
                            contextual_seq_len, min_full_attn_seq_len, deterministic=_deterministic(deterministic),
                            causal=bool(causal))
    return [dq, dk, dv]


def _deterministic(flag):
    """deterministic=False of the schema leaves the choice to torch.use_deterministic_algorithms."""
    return True if flag else None


def _mha(max_seq_len, alpha, q, k, v, seq_offsets, causal, num_targets, attn_scale, max_attn_len, min_full_attn_seq_len,
         contextual_seq_len, q_descale, k_descale, v_descale, sort_by_length, deterministic, sm_margin):
    descales = (q_descale, k_descale, v_descale)
    _check(causal, seq_offsets, attn_scale, descales, (q, k, v))
    if any(t.dtype == _FP8 for t in (q, k, v)):
        if torch.is_grad_enabled() and any(t.requires_grad for t in (q, k, v)):
            raise RuntimeError("hstu::hstu_mha on H100: fp8 attention is forward only (the reference has no fp8 backward); "
                               "run it under torch.no_grad() or on tensors that do not require grad")
        return cuda_hstu_attention_fwd(int(max_seq_len), alpha, q, k, v, seq_offsets, num_targets, max_attn_len,
                                       contextual_seq_len, min_full_attn_seq_len, descales=descales, causal=bool(causal))
    return _HSTUAttentionFunction.apply(int(max_seq_len), alpha, q, k, v, seq_offsets, num_targets, max_attn_len,
                                        contextual_seq_len, min_full_attn_seq_len, _lib.IMPL_AUTO, bool(causal),
                                        _deterministic(deterministic))


def _fwd_meta(max_seq_len, alpha, q, k, v, *args):
    dt = torch.bfloat16 if v.dtype == _FP8 else v.dtype  # the fp8 forward writes bf16
    return q.new_empty((q.shape[0], q.shape[1], v.shape[2]), dtype=dt)


def register() -> None:
    """Define `hstu::hstu_mha`, `hstu::hstu_mha_fwd`, `hstu::hstu_mha_bwd` with the reference's schemas (idempotent)."""
    global _LIB
    if _LIB is not None:
        return
    lib = torch.library.Library("hstu", "FRAGMENT")
    lib.define(_MHA)
    lib.define(_FWD)
    lib.define(_BWD)
    lib.impl("hstu_mha", _mha, "CompositeImplicitAutograd")  # autograd through _HSTUAttentionFunction; fwd / bwd: raw kernels
    lib.impl("hstu_mha_fwd", _fwd, "CUDA")
    lib.impl("hstu_mha_bwd", _bwd, "CUDA")
    lib.impl("hstu_mha_fwd", _fwd_meta, "Meta")
    _LIB = lib
