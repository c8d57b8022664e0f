"""ctypes binding of libhstu_b200.so -- the only way the Python host layer reaches the CUDA kernels.

The structure layout and prototypes mirror include/hstu_b200.h one to one.  There is no CPU fallback: if the
library is missing or a call fails, an exception is raised.
"""
import ctypes as C
import os
from typing import Optional

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
# HSTU_B200_LIB: another build of the same ABI (compile-time variants for A/B measurements: HSTU_EXP / HSTU_EXP_SRC of build.py)
LIB_PATH = os.environ.get("HSTU_B200_LIB") or os.path.join(_HERE, "lib", "libhstu_b200.so")

ABI_VERSION = 1
F32, BF16, F16, E4M3 = 0, 1, 2, 3
IMPL_AUTO, IMPL_GENERIC, IMPL_UMMA = 0, 1, 2

_DTYPES = {torch.float32: F32, torch.bfloat16: BF16, torch.float16: F16, torch.float8_e4m3fn: E4M3}


class AttnParams(C.Structure):
    _fields_ = [
        ("abi_version", C.c_int32), ("dtype", C.c_int32), ("impl", C.c_int32), ("batch", C.c_int32),
        ("heads", C.c_int32), ("dqk", C.c_int32), ("dv", C.c_int32), ("max_seq_len", C.c_int32),
        ("total_rows", C.c_int64), ("alpha", C.c_float), ("max_attn_len", C.c_int32),
        ("min_full_attn_seq_len", C.c_int32), ("contextual_seq_len", C.c_int32), ("delta_q_len", C.c_int32),
        ("offsets_are_i64", C.c_int32), ("num_targets_are_i64", C.c_int32),
        ("seq_offsets", C.c_void_p), ("num_targets", C.c_void_p), ("q", C.c_void_p), ("k", C.c_void_p),
        ("v", C.c_void_p), ("out", C.c_void_p),
        ("q_row_stride", C.c_int64), ("q_head_stride", C.c_int64), ("k_row_stride", C.c_int64),
        ("k_head_stride", C.c_int64), ("v_row_stride", C.c_int64), ("v_head_stride", C.c_int64),
        ("o_row_stride", C.c_int64), ("o_head_stride", C.c_int64),
        ("dout", C.c_void_p), ("dq", C.c_void_p), ("dk", C.c_void_p), ("dv_out", C.c_void_p),
        ("do_row_stride", C.c_int64), ("do_head_stride", C.c_int64), ("dq_row_stride", C.c_int64),
        ("dq_head_stride", C.c_int64), ("dk_row_stride", C.c_int64), ("dk_head_stride", C.c_int64),
        ("dv_row_stride", C.c_int64), ("dv_head_stride", C.c_int64),
        ("pos_w", C.c_void_p), ("ts_w", C.c_void_p), ("timestamps", C.c_void_p), ("num_ts_buckets", C.c_int32),
        ("deterministic", C.c_int32), ("dpos_w", C.c_void_p), ("dts_w", C.c_void_p),
        ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t),
    ]


class Descales(C.Structure):
    """hstu_attn_descales: per (sequence, head) fp32 scales of the fp8 forward's q, k, v (NULL = 1)."""
    _fields_ = [
        ("q", C.c_void_p), ("k", C.c_void_p), ("v", C.c_void_p),
        ("q_batch_stride", C.c_int64), ("q_head_stride", C.c_int64), ("k_batch_stride", C.c_int64),
        ("k_head_stride", C.c_int64), ("v_batch_stride", C.c_int64), ("v_head_stride", C.c_int64),
    ]


class SslParams(C.Structure):
    _fields_ = [
        ("abi_version", C.c_int32), ("dtype", C.c_int32), ("N", C.c_int64), ("R", C.c_int32), ("D", C.c_int32),
        ("l2_norm", C.c_int32), ("l2_eps", C.c_float), ("temperature", C.c_float), ("reserved0", C.c_int32),
        ("q", C.c_void_p), ("pos_emb", C.c_void_p), ("table", C.c_void_p), ("pos_ids", C.c_void_p), ("neg_ids", C.c_void_p),
        ("logits", C.c_void_p), ("rnorm", C.c_void_p), ("lse", C.c_void_p), ("loss_rows", C.c_void_p),
        ("row_coef", C.c_void_p), ("d_q", C.c_void_p), ("d_pos_emb", C.c_void_p), ("d_table", C.c_void_p),
    ]


_lib: Optional[C.CDLL] = None

_i32, _i64, _f32, _u64, _vp = C.c_int32, C.c_int64, C.c_float, C.c_uint64, C.c_void_p

_PROTOS = {
    "hstu_last_error": (C.c_char_p, []),
    "hstu_abi_version": (C.c_int, []),
    "hstu_attn_workspace_bytes": (C.c_size_t, [C.POINTER(AttnParams), C.c_int]),
    "hstu_attn_fwd": (C.c_int, [C.POINTER(AttnParams), _vp]),
    "hstu_attn_bwd": (C.c_int, [C.POINTER(AttnParams), _vp]),
    "hstu_attn_fwd_fp8": (C.c_int, [C.POINTER(AttnParams), C.POINTER(Descales), _vp]),
    "hstu_attn_fwd_delta_fp8_kv": (C.c_int, [C.POINTER(AttnParams), C.POINTER(Descales), _vp]),
    "hstu_attn_fp8_kv_workspace_bytes": (C.c_size_t, [C.POINTER(AttnParams)]),
    "hstu_attn_select_impl": (C.c_int, [C.POINTER(AttnParams), C.c_int]),
    "hstu_attn_fp16_operands_bytes": (C.c_size_t, [C.POINTER(AttnParams)]),
    "hstu_attn_fwd_keep_fp16_operands": (C.c_int, [C.POINTER(AttnParams), _vp, C.c_size_t, _vp]),
    "hstu_attn_bwd_fp16_operands_workspace_bytes": (C.c_size_t, [C.POINTER(AttnParams)]),
    "hstu_attn_bwd_on_fp16_operands": (C.c_int, [C.POINTER(AttnParams), _vp, C.c_size_t, _vp]),
    "hstu_attn_fwd_bidir": (C.c_int, [C.POINTER(AttnParams), _vp]),
    "hstu_attn_bwd_bidir": (C.c_int, [C.POINTER(AttnParams), _vp]),
    "hstu_attn_bidir_workspace_bytes": (C.c_size_t, [C.POINTER(AttnParams), C.c_int]),
    "hstu_attn_bidir_select_impl": (C.c_int, [C.POINTER(AttnParams), C.c_int]),
    "hstu_mask_valid": (C.c_int, [_i32] * 7),
    "hstu_kv_range_for_q_rows": (C.c_int, [_i32] * 7 + [C.POINTER(_i32)] * 2),
    "hstu_q_range_for_kv_rows": (C.c_int, [_i32] * 7 + [C.POINTER(_i32)] * 3),
    "hstu_mask_valid_bidir": (C.c_int, [_i32] * 7),
    "hstu_kv_range_for_q_rows_bidir": (C.c_int, [_i32] * 7 + [C.POINTER(_i32)] * 2),
    "hstu_q_range_for_kv_rows_bidir": (C.c_int, [_i32] * 7 + [C.POINTER(_i32)] * 3),
    "hstu_layer_norm_fwd": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _i64, _i32, _i64, _i64, _f32, _i32, _i32, _vp]),
    "hstu_layer_norm_bwd": (C.c_int, [_vp] * 10 + [_i64, _i32, _i64, _i64, _i64, _i32, _i32, _vp]),
    "hstu_norm_bwd_partial_rows": (_i32, []),
    "hstu_rms_norm_fwd": (C.c_int, [_vp, _vp, _vp, _vp, _i64, _i32, _f32, _i32, _vp]),
    "hstu_rms_norm_bwd": (C.c_int, [_vp] * 7 + [_i64, _i32, _i32, _vp]),
    "hstu_norm_mul_dropout_fwd": (C.c_int, [_vp] * 7 + [_i64, _i32, _i32, _i64, _i64, _f32, _f32, _u64, _i32, _i32, _i32, _i32, _vp]),
    "hstu_norm_mul_dropout_bwd": (C.c_int, [_vp] * 12 + [_i64, _i32, _i32, _i64, _i64, _i64, _i64, _f32, _u64, _i32, _i32, _i32, _i32, _vp]),
    "hstu_silu_fwd": (C.c_int, [_vp, _vp, _i64, _i32, _i64, _i64, _i32, _vp]),
    "hstu_silu_bwd": (C.c_int, [_vp, _vp, _vp, _i64, _i32, _i64, _i64, _i64, _i32, _vp]),
    "hstu_jagged_concat": (C.c_int, [_vp] * 5 + [_i32] * 8 + [_vp]),
    "hstu_jagged_split": (C.c_int, [_vp] * 5 + [_i32] * 8 + [_vp]),
    "hstu_position_embeddings_fwd": (C.c_int, [_vp] * 10 + [_i64, _i32, _i32, _i32, _i32, _i32, _f32, _i32, _i32, _i32, _i32, _i32, _i32, _vp]),
    "hstu_position_embeddings_bwd": (C.c_int, [_vp] * 6 + [_i64, _i32, _f32, _i32, _vp]),
    "hstu_jagged_dense_bmm_broadcast_add": (C.c_int, [_vp] * 5 + [_i32] * 7 + [_vp]),
    "hstu_jagged_dense_bmm_wgrad": (C.c_int, [_vp] * 5 + [_i32] * 6 + [_vp]),
    "hstu_sampled_softmax_fwd": (C.c_int, [C.POINTER(SslParams), _vp]),
    "hstu_sampled_softmax_bwd": (C.c_int, [C.POINTER(SslParams), _vp]),
}

EXPORTED_SYMBOLS = tuple(_PROTOS.keys())


def lib() -> C.CDLL:
    """Load (once) and return the shared library; raises if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: build it with `python -m generative_recommenders_b200.build` "
                "(there is no CPU / eager fallback for HammerKernel.CUDA)"
            )
        l = C.CDLL(LIB_PATH)
        for name, (res, args) in _PROTOS.items():
            fn = getattr(l, name)
            fn.restype = res
            fn.argtypes = args
        if l.hstu_abi_version() != ABI_VERSION:
            raise RuntimeError("libhstu_b200.so ABI version mismatch")
        _lib = l
    return _lib


_selftest: Optional[C.CDLL] = None


def selftest_lib() -> C.CDLL:
    """The TEST library with the wgmma / TMA self test (include/hstu_b200_selftest.h); not used by any product code path."""
    global _selftest
    if _selftest is None:
        path = os.path.join(_HERE, "lib", "libhstu_b200_selftest.so")
        if not os.path.exists(path):
            raise RuntimeError(f"{path} is missing: build it with `python -m generative_recommenders_b200.build`")
        l = C.CDLL(path)
        l.hstu_umma_selftest.restype = C.c_int
        l.hstu_umma_selftest.argtypes = [C.c_char_p, C.c_size_t]
        _selftest = l
    return _selftest


# ---- instrumentation used by bench.py: kernel-launch counter and optional CUDA-event timing per C-ABI call ----
LAUNCHES = 0
_TIMED = None  # None, or dict: name -> list[(start_event, end_event)]


def note_launch(n: int = 1) -> None:
    global LAUNCHES
    LAUNCHES += n


def enable_timing(on: bool) -> None:
    global _TIMED
    _TIMED = {} if on else None


def timed_events():
    return _TIMED


class timed:
    """`with timed("attn_fwd", device):` brackets the enqueued kernels with CUDA events on the current stream."""

    def __init__(self, name: str, device):
        self.name, self.device = name, device

    def __enter__(self):
        if _TIMED is not None:
            self.e0 = torch.cuda.Event(enable_timing=True)
            self.e1 = torch.cuda.Event(enable_timing=True)
            self.e0.record(torch.cuda.current_stream(self.device))
        return self

    def __exit__(self, *exc):
        if _TIMED is not None:
            self.e1.record(torch.cuda.current_stream(self.device))
            _TIMED.setdefault(self.name, []).append((self.e0, self.e1))
        return False


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = lib().hstu_last_error().decode(errors="replace")
        raise RuntimeError(f"{what} failed (code {rc}): {msg}")


def dtype_code(t: torch.Tensor) -> int:
    try:
        return _DTYPES[t.dtype]
    except KeyError:
        raise RuntimeError(f"unsupported dtype {t.dtype} for the CUDA HSTU kernels") from None


def ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def stream_ptr(device: torch.device) -> int:
    return torch.cuda.current_stream(device).cuda_stream


def require_cuda(*tensors: Optional[torch.Tensor]) -> torch.device:
    dev = None
    for t in tensors:
        if t is None:
            continue
        if not t.is_cuda:
            raise RuntimeError("HammerKernel.CUDA ops need CUDA tensors (no CPU fallback)")
        if dev is None:
            dev = t.device
        elif t.device != dev:
            raise RuntimeError("all tensors must be on the same CUDA device")
    assert dev is not None
    return dev
