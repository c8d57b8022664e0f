"""Jagged HSTU attention on H100 -- host side of `hstu_attn_fwd` / `hstu_attn_bwd` (include/hstu_b200.h).

Same call surface as the reference facade generative_recommenders/ops/hstu_attention.py:44-203
(`hstu_mha`, `delta_hstu_mha`), same argument meaning and assertions; `kernel` must be HammerKernel.CUDA.
`cuda_hstu_attention_fwd/bwd` are the raw (non-autograd) entry points used by the fused block op; their
dq/dk/dv are caller-allocated and may be strided views of one `duvqk` buffer, as in the reference's
ops/cpp/cuda_hstu_preprocess_and_attention.py:254-306.
`causal=False` runs the non-causal attention (`hstu_attn_fwd_bidir` / `hstu_attn_bwd_bidir`) under the reference eager
path's causal=False mask; it takes no delta-q, fp8 input, relative bias or kept fp16 operands.
"""
import ctypes as C
from typing import Optional, Tuple

import torch

from .. import _lib
from ..common import HammerKernel, require_cuda_kernel, switch_to_contiguous_if_needed

_FP8 = torch.float8_e4m3fn


def _fill_common(p, max_seq_len, alpha, q, k, v, seq_offsets, num_targets, max_attn_len, contextual_seq_len,
                 min_full_attn_seq_len, impl, delta_q_len=0):
    if seq_offsets.dtype not in (torch.int32, torch.int64):
        raise RuntimeError("seq_offsets must be int32 or int64")
    if num_targets is not None and num_targets.dtype not in (torch.int32, torch.int64):
        raise RuntimeError("num_targets must be int32 or int64")
    p.abi_version = _lib.ABI_VERSION
    p.dtype = _lib.dtype_code(q)
    p.impl = impl
    p.batch = seq_offsets.numel() - 1
    p.heads = q.shape[1]
    p.dqk = q.shape[2]
    p.dv = v.shape[2]
    p.max_seq_len = int(max_seq_len)
    p.total_rows = k.shape[0]
    p.alpha = float(alpha)
    p.max_attn_len = int(max_attn_len)
    p.min_full_attn_seq_len = int(min_full_attn_seq_len)
    p.contextual_seq_len = int(contextual_seq_len)
    p.delta_q_len = int(delta_q_len)
    p.offsets_are_i64 = int(seq_offsets.dtype == torch.int64)
    p.num_targets_are_i64 = int(num_targets is not None and num_targets.dtype == torch.int64)
    p.seq_offsets = seq_offsets.data_ptr()
    p.num_targets = _lib.ptr(num_targets)
    p.q, p.k, p.v = q.data_ptr(), k.data_ptr(), v.data_ptr()
    p.q_row_stride, p.q_head_stride = q.stride(0), q.stride(1)
    p.k_row_stride, p.k_head_stride = k.stride(0), k.stride(1)
    p.v_row_stride, p.v_head_stride = v.stride(0), v.stride(1)


def _aligned_buffer(nbytes: int, device):
    """(buffer, base): a uint8 tensor holding nbytes from a 256-byte aligned base address, as the library's workspaces and
    kept operands need; (None, None) for 0 bytes."""
    if nbytes == 0:
        return None, None
    buf = torch.empty(nbytes + 256, dtype=torch.uint8, device=device)
    return buf, (buf.data_ptr() + 255) // 256 * 256


def _workspace(p, bwd: bool, device, causal: bool = True):
    size = _lib.lib().hstu_attn_workspace_bytes if causal else _lib.lib().hstu_attn_bidir_workspace_bytes
    p.workspace_bytes = size(C.byref(p), int(bwd))
    ws, p.workspace = _aligned_buffer(p.workspace_bytes, device)
    return ws


def _fwd_params(max_seq_len, alpha, q, k, v, seq_offsets, num_targets, max_attn_len, contextual_seq_len,
                min_full_attn_seq_len, impl, delta_q_len, out, out_dtype):
    """(p, out, device) of a forward: q, k, v, seq_offsets, num_targets on one CUDA device and contiguous where the kernels
    need it, and out, allocated [rows of q, H, dv] in out_dtype if None."""
    dev = _lib.require_cuda(q, k, v, seq_offsets, num_targets)
    q, k, v = _prep(q, k, v)
    seq_offsets = seq_offsets.contiguous()
    if num_targets is not None:
        num_targets = num_targets.contiguous()
    if out is None:
        out = torch.empty((q.shape[0], q.shape[1], v.shape[2]), dtype=out_dtype, device=dev)
    p = _lib.AttnParams()
    _fill_common(p, max_seq_len, alpha, q, k, v, seq_offsets, num_targets, max_attn_len, contextual_seq_len,
                 min_full_attn_seq_len, impl, delta_q_len)
    p.out = out.data_ptr()
    p.o_row_stride, p.o_head_stride = out.stride(0), out.stride(1)
    return p, out, dev


def _prep(*ts):
    return tuple(switch_to_contiguous_if_needed(t) for t in ts)


def _wgmma_view(t: torch.Tensor) -> torch.Tensor:
    """t, or a contiguous copy of it where the wgmma kernels could not take it (a 16-byte base, row / head strides of whole
    16-byte units)."""
    ok = t.data_ptr() % 16 == 0 and t.stride(0) % 8 == 0 and t.stride(1) % 8 == 0
    return t if ok else t.clone(memory_format=torch.contiguous_format)


class Fp16Operands:
    """The scaled fp16 copies of q, k, v and their per (sequence, head) amax that a bf16 attention at dqk == dv == 32 runs on
    (include/hstu_b200.h, hstu_attn_fwd_keep_fp16_operands).  Pass an empty one to `cuda_hstu_attention_fwd` and the same one
    to the backward of the same q, k, v: the forward fills it, and the backward then converts dO alone and reads neither q,
    k nor v.  A forward that does not run on such operands leaves it empty, and the backward then takes q, k, v as usual."""

    def __init__(self):
        self.buf: Optional[torch.Tensor] = None  # uint8, the library's layout from a 256-byte aligned `base`
        self.base = 0
        self.nbytes = 0  # from `base`: the backward checks it against what its sizes need


def cuda_hstu_attention_fwd(
    max_seq_len: int, alpha: float, q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, seq_offsets: torch.Tensor,
    num_targets: Optional[torch.Tensor] = None, max_attn_len: int = 0, contextual_seq_len: int = 0,
    min_full_attn_seq_len: int = 0, impl: int = _lib.IMPL_AUTO, delta_q_len: int = 0,
    out: Optional[torch.Tensor] = None, bias: Optional[Tuple[torch.Tensor, torch.Tensor, torch.Tensor]] = None,
    descales: Optional[Tuple[Optional[torch.Tensor], Optional[torch.Tensor], Optional[torch.Tensor]]] = None,
    fp16_operands: Optional[Fp16Operands] = None, causal: bool = True,
) -> torch.Tensor:
    """descales: (q_descale, k_descale, v_descale) of fp8 inputs -- see cuda_hstu_attention_fwd_fp8.  q, k, v of dtype
    torch.float8_e4m3fn take that path with or without descales.  fp16_operands: an empty Fp16Operands that keeps the
    call's fp16 operands for its backward, if it runs on them (a non-causal call leaves it empty).  causal=False: the
    non-causal attention (bf16 / fp16 / fp32, no delta_q, fp8 or bias)."""
    if not causal:
        _refuse_bidir(q, k, v, delta_q_len, bias, descales)
        fp16_operands = None
    elif delta_q_len and q.dtype in (torch.bfloat16, torch.float16) and k.dtype == _FP8 and v.dtype == _FP8:
        if bias is not None:
            raise RuntimeError("delta-q attention on an fp8 K / V cache: the relative bias is not supported")
        if descales is not None and descales[0] is not None:
            raise RuntimeError("delta-q attention on an fp8 K / V cache: q is bf16 / fp16 and takes no descale")
        return cuda_hstu_attention_fwd_delta_fp8_kv(max_seq_len, alpha, q, k, v, seq_offsets, delta_q_len,
                                                    None if descales is None else tuple(descales[1:]), num_targets,
                                                    max_attn_len, contextual_seq_len, min_full_attn_seq_len, impl, out)
    elif descales is not None or any(t.dtype == _FP8 for t in (q, k, v)):
        if bias is not None or delta_q_len:
            raise RuntimeError("fp8 attention: the relative bias and delta_q are not supported")
        return cuda_hstu_attention_fwd_fp8(max_seq_len, alpha, q, k, v, seq_offsets, descales, num_targets, max_attn_len,
                                           contextual_seq_len, min_full_attn_seq_len, impl, out)
    p, out, dev = _fwd_params(max_seq_len, alpha, q, k, v, seq_offsets, num_targets, max_attn_len, contextual_seq_len,
                              min_full_attn_seq_len, impl, delta_q_len, out, v.dtype)
    keep = _fill_bias(p, bias, None)
    kept = _lib.lib().hstu_attn_fp16_operands_bytes(C.byref(p)) if fp16_operands is not None else 0
    if kept:
        fp16_operands.buf, fp16_operands.base = _aligned_buffer(kept, dev)
        fp16_operands.nbytes = kept
        ws = None  # the pre-pass writes into the operands buffer instead of a workspace
        with torch.cuda.device(dev), _lib.timed("attn_fwd", dev):
            _lib.check(_lib.lib().hstu_attn_fwd_keep_fp16_operands(C.byref(p), fp16_operands.base, kept, _lib.stream_ptr(dev)),
                       "hstu_attn_fwd_keep_fp16_operands")
    else:
        ws = _workspace(p, False, dev) if causal else _workspace(p, False, dev, causal=False)
        run, name = (_lib.lib().hstu_attn_fwd, "attn_fwd") if causal else (_lib.lib().hstu_attn_fwd_bidir, "attn_fwd_bidir")
        with torch.cuda.device(dev), _lib.timed(name, dev):
            _lib.check(run(C.byref(p), _lib.stream_ptr(dev)), run.__name__)
    if delta_q_len:  # a workspace holds the partials of split key chunks: the attention kernel, then their reduction
        _lib.note_launch(2 if ws is not None else 1)
    else:  # bf16 at d = 32: amax and convert kernels before the attention kernel (into the workspace or the operands buffer)
        _lib.note_launch(3 if ws is not None or kept else 1)
    del ws, keep
    return out


def _refuse_bidir(q, k, v, delta_q_len=0, bias=None, descales=None):
    if delta_q_len:
        raise RuntimeError("non-causal attention: delta_q (the KV-cached forward) is causal only")
    if descales is not None or any(t is not None and t.dtype == _FP8 for t in (q, k, v)):
        raise RuntimeError("non-causal attention: fp8 (float8_e4m3fn) inputs are not supported")
    if bias is not None:
        raise RuntimeError("non-causal attention: the relative bias is not supported")


def cuda_hstu_attention_fwd_fp8(
    max_seq_len: int, alpha: float, q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, seq_offsets: torch.Tensor,
    descales: Optional[Tuple[Optional[torch.Tensor], Optional[torch.Tensor], Optional[torch.Tensor]]] = None,
    num_targets: Optional[torch.Tensor] = None, max_attn_len: int = 0, contextual_seq_len: int = 0,
    min_full_attn_seq_len: int = 0, impl: int = _lib.IMPL_AUTO, out: Optional[torch.Tensor] = None,
) -> torch.Tensor:
    """Forward of attention on float8_e4m3fn q, k, v (`hstu_attn_fwd_fp8`): the bf16 result of the attention of
    q * q_descale[b, h], k * k_descale[b, h] and v * v_descale[b, h], every mask option of the bf16 path included.  Each
    descale is an fp32 [B, H] tensor (any strides) or None for 1.  There is no fp8 backward.  The wgmma kernels take
    dqk == dv, or dqk < dv, with both in {32, 64, 128, 256} (the output has dv columns), 16-byte aligned views with row /
    head strides that are multiples of 16 elements."""
    if not all(t.dtype == _FP8 for t in (q, k, v)):
        raise RuntimeError(f"fp8 attention: q, k and v must all be torch.float8_e4m3fn (got {q.dtype}, {k.dtype}, {v.dtype}); "
                           "descales apply to fp8 inputs only")
    if out is not None and out.dtype != torch.bfloat16:
        raise RuntimeError(f"fp8 attention: out must be bf16 (got {out.dtype})")
    p, out, dev = _fwd_params(max_seq_len, alpha, q, k, v, seq_offsets, num_targets, max_attn_len, contextual_seq_len,
                              min_full_attn_seq_len, impl, 0, out, torch.bfloat16)
    ds = _lib.Descales()
    _fill_descales(ds, "qkv", descales if descales is not None else (None, None, None), p.batch, p.heads, dev,
                   "fp8 attention")
    ws = _workspace(p, False, dev)
    with torch.cuda.device(dev), _lib.timed("attn_fwd_fp8", dev):
        _lib.check(_lib.lib().hstu_attn_fwd_fp8(C.byref(p), C.byref(ds), _lib.stream_ptr(dev)), "hstu_attn_fwd_fp8")
    _lib.note_launch(2)  # the fp16 copy of v, then the attention kernel
    del ws
    return out


def _fill_descales(ds, names, descales, B, H, dev, what):
    for name, d in zip(names, descales):
        if d is None:
            continue
        if d.dtype != torch.float32 or tuple(d.shape) != (B, H):
            raise RuntimeError(f"{what}: {name}_descale must be an fp32 [B, H] = [{B}, {H}] tensor "
                               f"(got {d.dtype} {tuple(d.shape)})")
        if d.device != dev:
            raise RuntimeError(f"{what}: {name}_descale is on {d.device}, the inputs on {dev}")
        setattr(ds, name, d.data_ptr())
        setattr(ds, f"{name}_batch_stride", d.stride(0))
        setattr(ds, f"{name}_head_stride", d.stride(1))


def cuda_hstu_attention_fwd_delta_fp8_kv(
    max_seq_len: int, alpha: float, delta_q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, seq_offsets: torch.Tensor,
    delta_q_len: int, kv_descales: Optional[Tuple[Optional[torch.Tensor], Optional[torch.Tensor]]] = None,
    num_targets: Optional[torch.Tensor] = None, max_attn_len: int = 0, contextual_seq_len: int = 0,
    min_full_attn_seq_len: int = 0, impl: int = _lib.IMPL_AUTO, out: Optional[torch.Tensor] = None,
) -> torch.Tensor:
    """KV-cached (delta-q) forward with bf16 / fp16 queries over a float8_e4m3fn K / V cache (`hstu_attn_fwd_delta_fp8_kv`):
    the attention of delta_q [B * delta_q_len, H, dqk] over k * k_descale[b, h] and v * v_descale[b, h], in the dtype of
    delta_q.  kv_descales: (k_descale, v_descale), each an fp32 [B, H] tensor (any strides) or None for 1.  The wgmma
    kernels widen K / V to the query dtype inside the kernel; they take dqk == dv, or dqk < dv, with both in {32, 64, 128,
    256}, and k / v views with row / head strides that are multiples of 16 elements.  There is no generic kernel for it."""
    what = "delta-q attention on an fp8 K / V cache"
    if delta_q.dtype not in (torch.bfloat16, torch.float16) or k.dtype != _FP8 or v.dtype != _FP8:
        raise RuntimeError(f"{what}: delta_q must be bf16 / fp16 and k, v torch.float8_e4m3fn "
                           f"(got {delta_q.dtype}, {k.dtype}, {v.dtype})")
    if delta_q_len <= 0:
        raise RuntimeError(f"{what}: delta_q_len must be > 0 (got {delta_q_len})")
    if impl == _lib.IMPL_GENERIC:
        raise RuntimeError(f"{what}: runs on the wgmma kernels only (the generic kernels take no fp8 input)")
    if out is not None and out.dtype != delta_q.dtype:
        raise RuntimeError(f"{what}: out must have the dtype of delta_q ({delta_q.dtype}, got {out.dtype})")
    p, out, dev = _fwd_params(max_seq_len, alpha, delta_q, k, v, seq_offsets, num_targets, max_attn_len, contextual_seq_len,
                              min_full_attn_seq_len, impl, delta_q_len, out, delta_q.dtype)
    ds = _lib.Descales()
    _fill_descales(ds, "kv", kv_descales if kv_descales is not None else (None, None), p.batch, p.heads, dev, what)
    p.workspace_bytes = _lib.lib().hstu_attn_fp8_kv_workspace_bytes(C.byref(p))
    ws, p.workspace = _aligned_buffer(p.workspace_bytes, dev)
    with torch.cuda.device(dev), _lib.timed("attn_fwd_delta_fp8_kv", dev):
        _lib.check(_lib.lib().hstu_attn_fwd_delta_fp8_kv(C.byref(p), C.byref(ds), _lib.stream_ptr(dev)),
                   "hstu_attn_fwd_delta_fp8_kv")
    _lib.note_launch(2 if ws is not None else 1)  # the attention kernel, and the reduction of split key chunks
    del ws
    return out


def cuda_hstu_attention_bwd(
    max_seq_len: int, alpha: float, dout: torch.Tensor, q: torch.Tensor, k: torch.Tensor, v: torch.Tensor,
    dq: torch.Tensor, dk: torch.Tensor, dv: torch.Tensor, seq_offsets: torch.Tensor,
    num_targets: Optional[torch.Tensor] = None, max_attn_len: int = 0, contextual_seq_len: int = 0,
    min_full_attn_seq_len: int = 0, impl: int = _lib.IMPL_AUTO,
    bias: Optional[Tuple[torch.Tensor, torch.Tensor, torch.Tensor]] = None,
    dbias: Optional[Tuple[torch.Tensor, torch.Tensor]] = None,
    deterministic: Optional[bool] = None,
    fp16_operands: Optional[Fp16Operands] = None, causal: bool = True,
) -> None:
    """Writes dq, dk, dv in place (last-dim stride 1 required; row/head strides arbitrary).

    causal=False: the backward of the non-causal attention.  It runs atomic-free kernels on every path, so it is bitwise
    reproducible whatever `deterministic` says; it takes no relative bias and no kept fp16 operands.

    fp16_operands: what the forward of these q, k, v kept (Fp16Operands).  If it holds operands, q, k, v are not read and may
    be None; that backward runs on the wgmma kernels only, so a dout or dq / dk / dv view they cannot take goes through a
    contiguous copy.

    deterministic: dq / dk / dv bitwise reproducible from run to run (the wgmma backward then runs its atomic-free dK / dV
    and dQ kernels at every head dim); None follows torch.are_deterministic_algorithms_enabled().  Not available with a
    relative bias, whose table gradients are added with atomics.
    """
    if deterministic is None:
        deterministic = torch.are_deterministic_algorithms_enabled()
    kept = fp16_operands is not None and fp16_operands.buf is not None
    if not causal:
        if kept:
            raise RuntimeError("non-causal attention: a non-causal forward keeps no fp16 operands; pass q, k, v")
        _refuse_bidir(q, k, v, bias=bias)
    if kept and q is None:  # dqk == dv: dout has the shape and dtype of q, k and v
        q = k = v = dout
    dev = _lib.require_cuda(dout, q, k, v, dq, dk, dv, seq_offsets, num_targets)
    q, k, v, dout = _prep(q, k, v, dout)
    for g in (dq, dk, dv):
        if g.stride(-1) != 1:
            raise RuntimeError("dq/dk/dv must have a dense last dimension")
    grads = (dq, dk, dv)
    if kept:  # no generic fallback without q, k, v
        dout = _wgmma_view(dout)
        dq, dk, dv = (_wgmma_view(g) for g in grads)
    seq_offsets = seq_offsets.contiguous()
    if num_targets is not None:
        num_targets = num_targets.contiguous()
    p = _lib.AttnParams()
    _fill_common(p, max_seq_len, alpha, q, k, v, seq_offsets, num_targets, max_attn_len, contextual_seq_len,
                 min_full_attn_seq_len, impl)
    p.dout, p.dq, p.dk, p.dv_out = dout.data_ptr(), dq.data_ptr(), dk.data_ptr(), dv.data_ptr()
    p.do_row_stride, p.do_head_stride = dout.stride(0), dout.stride(1)
    p.dq_row_stride, p.dq_head_stride = dq.stride(0), dq.stride(1)
    p.dk_row_stride, p.dk_head_stride = dk.stride(0), dk.stride(1)
    p.dv_row_stride, p.dv_head_stride = dv.stride(0), dv.stride(1)
    p.deterministic = int(bool(deterministic))
    keep = _fill_bias(p, bias, dbias)
    if kept:  # the amax and convert kernels over dO alone, then the dK/dV and dQ kernels
        p.q = p.k = p.v = None
        p.workspace_bytes = _lib.lib().hstu_attn_bwd_fp16_operands_workspace_bytes(C.byref(p))
        ws, p.workspace = _aligned_buffer(p.workspace_bytes, dev)
        with torch.cuda.device(dev), _lib.timed("attn_bwd", dev):
            _lib.check(_lib.lib().hstu_attn_bwd_on_fp16_operands(C.byref(p), fp16_operands.base, fp16_operands.nbytes,
                                                                 _lib.stream_ptr(dev)), "hstu_attn_bwd_on_fp16_operands")
        _lib.note_launch(4)
        for g, w in zip(grads, (dq, dk, dv)):
            if w is not g:
                g.copy_(w)
        del ws, keep
        return
    ws = _workspace(p, True, dev) if causal else _workspace(p, True, dev, causal=False)
    run, name = (_lib.lib().hstu_attn_bwd, "attn_bwd") if causal else (_lib.lib().hstu_attn_bwd_bidir, "attn_bwd_bidir")
    with torch.cuda.device(dev), _lib.timed(name, dev):
        _lib.check(run(C.byref(p), _lib.stream_ptr(dev)), run.__name__)
    # wgmma path: dK/dV kernel + dQ kernel (d = 32, after the amax and convert kernels for bf16; deterministic d = 64 / 128
    # and every non-causal call: no workspace, no memset, no convert) or main kernel + dQ convert; generic path: dK/dV
    # kernel + dQ kernel
    _lib.note_launch(4 if ws is not None and p.dtype == _lib.BF16 and p.dqk == 32 else 2)
    del ws, keep


def _fill_bias(p, bias, dbias):
    if bias is None:
        return None
    pos_w, ts_w, timestamps = bias
    keep = []
    n, B = int(p.max_seq_len), int(p.batch)
    # the kernels index pos_w[n - 1 + j - i] and timestamps[b * n + i] without bounds checks: the shapes are the contract
    if pos_w is not None and pos_w.numel() != 2 * n - 1:
        raise RuntimeError(f"relative position bias: pos_w must have 2 * max_seq_len - 1 = {2 * n - 1} entries, got {pos_w.numel()}")
    if (ts_w is None) != (timestamps is None):
        raise RuntimeError("relative time bias: ts_w and timestamps must be given together")
    if ts_w is not None:
        if tuple(timestamps.shape) != (B, n):
            raise RuntimeError(f"relative time bias: timestamps must be [B, max_seq_len] = [{B}, {n}], got {tuple(timestamps.shape)}")
        if ts_w.numel() < 2:
            raise RuntimeError("relative time bias: ts_w must have num_buckets + 1 >= 2 entries")
    if pos_w is not None:
        pos_w = pos_w.detach().float().contiguous()
        p.pos_w = pos_w.data_ptr()
        keep.append(pos_w)
    if ts_w is not None:
        ts_w = ts_w.detach().float().contiguous()
        timestamps = timestamps.to(torch.int64).contiguous()
        p.ts_w, p.timestamps = ts_w.data_ptr(), timestamps.data_ptr()
        p.num_ts_buckets = ts_w.numel() - 1
        keep += [ts_w, timestamps]
    if dbias is not None:
        dpos_w, dts_w = dbias
        p.dpos_w = _lib.ptr(dpos_w)
        p.dts_w = _lib.ptr(dts_w)
    return keep


class _HSTUAttentionFunction(torch.autograd.Function):
    """The autograd of hstu_mha and torch.ops.hstu.hstu_mha.  deterministic: that of cuda_hstu_attention_bwd (None follows
    torch.are_deterministic_algorithms_enabled() when the backward runs)."""

    @staticmethod
    def forward(ctx, max_seq_len, alpha, q, k, v, seq_offsets, num_targets, max_attn_len, contextual_seq_len,
                min_full_attn_seq_len, impl, causal, deterministic):
        # no Fp16Operands here: q, k, v are saved anyway, so the copies would double the saved bytes to spare only the
        # backward's pre-pass over q, k, v
        out = cuda_hstu_attention_fwd(max_seq_len, alpha, q, k, v, seq_offsets, num_targets, max_attn_len,
                                      contextual_seq_len, min_full_attn_seq_len, impl, causal=causal)
        ctx.save_for_backward(q, k, v, seq_offsets, num_targets)
        ctx.args = (max_seq_len, alpha, max_attn_len, contextual_seq_len, min_full_attn_seq_len, impl, causal, deterministic)
        return out

    @staticmethod
    def backward(ctx, dout):
        q, k, v, seq_offsets, num_targets = ctx.saved_tensors
        max_seq_len, alpha, max_attn_len, contextual_seq_len, min_full, impl, causal, deterministic = ctx.args
        dq = torch.empty(q.shape, dtype=q.dtype, device=q.device)
        dk = torch.empty(k.shape, dtype=k.dtype, device=k.device)
        dv = torch.empty(v.shape, dtype=v.dtype, device=v.device)
        cuda_hstu_attention_bwd(max_seq_len, alpha, dout, q, k, v, dq, dk, dv, seq_offsets, num_targets, max_attn_len,
                                contextual_seq_len, min_full, impl, deterministic=deterministic, causal=causal)
        return None, None, dq, dk, dv, None, None, None, None, None, None, None, None


def hstu_mha(
    max_seq_len: int,
    alpha: float,
    q: torch.Tensor,
    k: torch.Tensor,
    v: torch.Tensor,
    seq_offsets: torch.Tensor,
    causal: bool = True,
    dropout_pr: float = 0.0,
    training: bool = True,
    num_targets: Optional[torch.Tensor] = None,
    max_attn_len: int = 0,
    contextual_seq_len: int = 0,
    min_full_attn_seq_len: int = 0,
    sort_by_length: bool = False,
    kernel: HammerKernel = HammerKernel.CUDA,
    enable_tma: bool = False,
    impl: int = _lib.IMPL_AUTO,
) -> torch.Tensor:
    """Drop-in for generative_recommenders.ops.hstu_attention.hstu_mha (hstu_attention.py:44-128).

    `sort_by_length` and `enable_tma` are accepted for call compatibility: the kernels always schedule heavy tiles
    first and always use TMA where the shape allows.  Precondition (as for the reference Triton backend): every
    sequence length is <= max_seq_len.  causal=False runs the non-causal attention (the reference eager path's
    causal=False mask), forward and backward.
    """
    _, H, _ = q.shape
    torch._assert(max_seq_len > 0, "max_seq_len must be larger than 0")
    torch._assert(q.dim() == 3, "q must be 3-D")
    torch._assert(k.shape == q.shape, "k must be the same shape as q")
    torch._assert(v.dim() == 3, "v must be 3-D")
    torch._assert(v.shape[0] == q.shape[0], "wrong v shape[0]")
    torch._assert(v.shape[1] == H, "wrong v shape[1]")
    require_cuda_kernel(kernel, "hstu_mha")
    torch._assert(dropout_pr < 1e-6, "dropout for the CUDA path is not implemented")
    return _HSTUAttentionFunction.apply(max_seq_len, alpha, q, k, v, seq_offsets, num_targets, max_attn_len,
                                        contextual_seq_len, min_full_attn_seq_len, impl, bool(causal), None)


def delta_hstu_mha(
    max_seq_len: int,
    alpha: float,
    delta_q: torch.Tensor,
    k: torch.Tensor,
    v: torch.Tensor,
    seq_offsets: torch.Tensor,
    num_targets: Optional[torch.Tensor] = None,
    max_attn_len: int = 0,
    contextual_seq_len: int = 0,
    kernel: HammerKernel = HammerKernel.CUDA,
    enable_tma: bool = False,
    kv_descales: Optional[Tuple[Optional[torch.Tensor], Optional[torch.Tensor]]] = None,
) -> torch.Tensor:
    """Drop-in for delta_hstu_mha (hstu_attention.py:131-203): the last L//B query rows of each sequence.

    k and v may be a float8_e4m3fn cache under bf16 / fp16 queries (cuda_hstu_attention_fwd_delta_fp8_kv), with
    kv_descales = (k_descale, v_descale), fp32 [B, H] tensors or None for 1."""
    L, H, D = delta_q.shape
    B = seq_offsets.size(0) - 1
    torch._assert(max_seq_len > 0, "max_seq_len must be larger than 0")
    torch._assert(delta_q.dim() == 3, "delta_q must be 3-D")
    torch._assert(L % B == 0, "delta_q must be padded")
    torch._assert(k.dim() == 3, "k must be 3-D")
    torch._assert(k.shape[1] == H, "wrong k shape[1]")
    torch._assert(k.shape[2] == D, "wrong k shape[2]")
    torch._assert(v.dim() == 3, "v must be 3-D")
    torch._assert(v.shape[1] == H, "wrong v shape[1]")
    require_cuda_kernel(kernel, "delta_hstu_mha")
    return cuda_hstu_attention_fwd(max_seq_len, alpha, delta_q, k, v, seq_offsets, num_targets, max_attn_len,
                                   contextual_seq_len, 0, _lib.IMPL_AUTO, delta_q_len=L // B,
                                   descales=None if kv_descales is None else (None, *kv_descales))


class _RelBiasAttentionFunction(torch.autograd.Function):
    """Research-path attention: silu(QK^T + rel_bias)/n under a plain causal mask (research hstu.py:150-223)."""

    @staticmethod
    def forward(ctx, n, q, k, v, seq_offsets, pos_w, ts_w, timestamps):
        out = cuda_hstu_attention_fwd(n, 1.0, q, k, v, seq_offsets, impl=_lib.IMPL_GENERIC,
                                      bias=(pos_w, ts_w, timestamps))
        ctx.save_for_backward(q, k, v, seq_offsets, pos_w, ts_w, timestamps)
        ctx.n = n
        return out

    @staticmethod
    def backward(ctx, dout):
        q, k, v, seq_offsets, pos_w, ts_w, timestamps = ctx.saved_tensors
        dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
        dpos = torch.zeros(pos_w.shape, dtype=torch.float32, device=q.device)
        dts = torch.zeros(ts_w.shape, dtype=torch.float32, device=q.device) if ts_w is not None else None
        # the bias-table gradients are added with atomics, so this backward is not reproducible whatever the global flag says
        cuda_hstu_attention_bwd(ctx.n, 1.0, dout, q, k, v, dq, dk, dv, seq_offsets, impl=_lib.IMPL_GENERIC,
                                bias=(pos_w, ts_w, timestamps), dbias=(dpos, dts), deterministic=False)
        return (None, dq, dk, dv, None, dpos.to(pos_w.dtype), None if dts is None else dts.to(ts_w.dtype), None)


def hstu_rel_bias_attention(n: int, q, k, v, seq_offsets, pos_w, ts_w=None, timestamps=None) -> torch.Tensor:
    """q,k [L,H,dqk], v [L,H,dv]; pos_w [2n-1]; ts_w [num_buckets+1], timestamps [B,n] int64 (both or neither)."""
    return _RelBiasAttentionFunction.apply(n, q, k, v, seq_offsets, pos_w, ts_w, timestamps)
