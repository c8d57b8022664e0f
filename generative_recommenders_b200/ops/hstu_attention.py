"""Jagged HSTU attention on H100 -- host side of `hstu_attn_fwd` / `hstu_attn_bwd` (include/hstu_b200.h).

Same call surface as the reference facade generative_recommenders/ops/hstu_attention.py:44-203
(`hstu_mha`, `delta_hstu_mha`), same argument meaning and assertions; `kernel` must be HammerKernel.CUDA.
`cuda_hstu_attention_fwd/bwd` are the raw (non-autograd) entry points used by the fused block op; their
dq/dk/dv are caller-allocated and may be strided views of one `duvqk` buffer, as in the reference's
ops/cpp/cuda_hstu_preprocess_and_attention.py:254-306.
"""
import ctypes as C
from typing import Optional, Tuple

import torch

from .. import _lib
from ..common import HammerKernel, require_cuda_kernel, switch_to_contiguous_if_needed


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


def _workspace(p, bwd: bool, device):
    nbytes = _lib.lib().hstu_attn_workspace_bytes(C.byref(p), int(bwd))
    if nbytes == 0:
        p.workspace, p.workspace_bytes = None, 0
        return None
    ws = torch.empty(nbytes + 256, dtype=torch.uint8, device=device)
    base = (ws.data_ptr() + 255) // 256 * 256
    p.workspace, p.workspace_bytes = base, nbytes
    return ws


def _prep(*ts):
    return tuple(switch_to_contiguous_if_needed(t) for t in ts)


def cuda_hstu_attention_fwd(
    max_seq_len: int, alpha: float, q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, seq_offsets: torch.Tensor,
    num_targets: Optional[torch.Tensor] = None, max_attn_len: int = 0, contextual_seq_len: int = 0,
    min_full_attn_seq_len: int = 0, impl: int = _lib.IMPL_AUTO, delta_q_len: int = 0,
    out: Optional[torch.Tensor] = None, bias: Optional[Tuple[torch.Tensor, torch.Tensor, torch.Tensor]] = None,
) -> torch.Tensor:
    dev = _lib.require_cuda(q, k, v, seq_offsets, num_targets)
    q, k, v = _prep(q, k, v)
    seq_offsets = seq_offsets.contiguous()
    if num_targets is not None:
        num_targets = num_targets.contiguous()
    if out is None:
        out = torch.empty((q.shape[0], q.shape[1], v.shape[2]), dtype=v.dtype, device=dev)
    p = _lib.AttnParams()
    _fill_common(p, max_seq_len, alpha, q, k, v, seq_offsets, num_targets, max_attn_len, contextual_seq_len,
                 min_full_attn_seq_len, impl, delta_q_len)
    p.out = out.data_ptr()
    p.o_row_stride, p.o_head_stride = out.stride(0), out.stride(1)
    keep = _fill_bias(p, bias, None)
    ws = _workspace(p, False, dev)
    with torch.cuda.device(dev), _lib.timed("attn_fwd", dev):
        _lib.check(_lib.lib().hstu_attn_fwd(C.byref(p), _lib.stream_ptr(dev)), "hstu_attn_fwd")
    # bf16 at d = 32: amax and convert kernels before the attention kernel (the forward's only workspace: the fp16 copies)
    _lib.note_launch(3 if ws is not None else 1)
    del ws, keep
    return out


def cuda_hstu_attention_bwd(
    max_seq_len: int, alpha: float, dout: torch.Tensor, q: torch.Tensor, k: torch.Tensor, v: torch.Tensor,
    dq: torch.Tensor, dk: torch.Tensor, dv: torch.Tensor, seq_offsets: torch.Tensor,
    num_targets: Optional[torch.Tensor] = None, max_attn_len: int = 0, contextual_seq_len: int = 0,
    min_full_attn_seq_len: int = 0, impl: int = _lib.IMPL_AUTO,
    bias: Optional[Tuple[torch.Tensor, torch.Tensor, torch.Tensor]] = None,
    dbias: Optional[Tuple[torch.Tensor, torch.Tensor]] = None,
    deterministic: Optional[bool] = None,
) -> None:
    """Writes dq, dk, dv in place (last-dim stride 1 required; row/head strides arbitrary).

    deterministic: dq / dk / dv bitwise reproducible from run to run (the wgmma backward then runs its atomic-free dK / dV
    and dQ kernels at every head dim); None follows torch.are_deterministic_algorithms_enabled().  Not available with a
    relative bias, whose table gradients are added with atomics.
    """
    if deterministic is None:
        deterministic = torch.are_deterministic_algorithms_enabled()
    dev = _lib.require_cuda(dout, q, k, v, dq, dk, dv, seq_offsets, num_targets)
    q, k, v, dout = _prep(q, k, v, dout)
    for g in (dq, dk, dv):
        if g.stride(-1) != 1:
            raise RuntimeError("dq/dk/dv must have a dense last dimension")
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
    ws = _workspace(p, True, dev)
    with torch.cuda.device(dev), _lib.timed("attn_bwd", dev):
        _lib.check(_lib.lib().hstu_attn_bwd(C.byref(p), _lib.stream_ptr(dev)), "hstu_attn_bwd")
    # wgmma path: dK/dV kernel + dQ kernel (d = 32, after the amax and convert kernels for bf16; deterministic d = 64 / 128:
    # no workspace, no memset, no convert) or main kernel + dQ convert; generic path: dK/dV kernel + dQ kernel
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
    @staticmethod
    def forward(ctx, max_seq_len, alpha, q, k, v, seq_offsets, num_targets, max_attn_len, contextual_seq_len,
                min_full_attn_seq_len, impl):
        out = cuda_hstu_attention_fwd(max_seq_len, alpha, q, k, v, seq_offsets, num_targets, max_attn_len,
                                      contextual_seq_len, min_full_attn_seq_len, impl)
        ctx.save_for_backward(q, k, v, seq_offsets, num_targets)
        ctx.args = (max_seq_len, alpha, max_attn_len, contextual_seq_len, min_full_attn_seq_len, impl)
        return out

    @staticmethod
    def backward(ctx, dout):
        q, k, v, seq_offsets, num_targets = ctx.saved_tensors
        max_seq_len, alpha, max_attn_len, contextual_seq_len, min_full, impl = ctx.args
        dq = torch.empty(q.shape, dtype=q.dtype, device=q.device)
        dk = torch.empty(k.shape, dtype=k.dtype, device=k.device)
        dv = torch.empty(v.shape, dtype=v.dtype, device=v.device)
        cuda_hstu_attention_bwd(max_seq_len, alpha, dout, q, k, v, dq, dk, dv, seq_offsets, num_targets, max_attn_len,
                                contextual_seq_len, min_full, impl)
        return None, None, dq, dk, dv, None, None, None, None, None, None


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
    sequence length is <= max_seq_len.
    """
    _, H, _ = q.shape
    torch._assert(max_seq_len > 0, "max_seq_len must be larger than 0")
    torch._assert(q.dim() == 3, "q must be 3-D")
    torch._assert(k.shape == q.shape, "k must be the same shape as q")
    torch._assert(v.dim() == 3, "v must be 3-D")
    torch._assert(v.shape[0] == q.shape[0], "wrong v shape[0]")
    torch._assert(v.shape[1] == H, "wrong v shape[1]")
    torch._assert(causal, "only support causal attention")
    require_cuda_kernel(kernel, "hstu_mha")
    torch._assert(dropout_pr < 1e-6, "dropout for the CUDA path is not implemented")
    return _HSTUAttentionFunction.apply(max_seq_len, alpha, q, k, v, seq_offsets, num_targets, max_attn_len,
                                        contextual_seq_len, min_full_attn_seq_len, impl)


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
) -> torch.Tensor:
    """Drop-in for delta_hstu_mha (hstu_attention.py:131-203): the last L//B query rows of each sequence."""
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
                                   contextual_seq_len, 0, _lib.IMPL_AUTO, delta_q_len=L // B)


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
