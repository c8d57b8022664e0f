"""Jagged concat / split on H100 -- host side of hstu_jagged_concat / hstu_jagged_split.

Same surface as generative_recommenders/ops/jagged_tensors.py:55-207.  Row routing is integer-exact; the backward of
concat is split and vice versa (as in ops/triton/triton_jagged_tensors.py:213-244,329-359).
"""
from typing import Optional, Tuple

import torch

from .. import _lib
from ..common import HammerKernel, require_cuda_kernel


def _off(o: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
    if o is None:
        return None
    if o.dtype not in (torch.int32, torch.int64):
        raise RuntimeError("offsets must be int32 or int64")
    return o.contiguous()


def _same_width(ol, orr):
    if ol is not None and orr is not None and ol.dtype != orr.dtype:
        return ol.to(torch.int64), orr.to(torch.int64)
    return ol, orr


def _batch(ol, orr, n_left, n_right, max_len_left, max_len_right) -> int:
    if ol is not None:
        return ol.numel() - 1
    if orr is not None:
        return orr.numel() - 1
    raise RuntimeError("offsets_left and offsets_right cannot be None at the same time")


def cuda_concat_2D_jagged(max_seq_len, values_left, values_right, max_len_left, max_len_right, offsets_left,
                          offsets_right, n_prefix_from_right: int = 0) -> torch.Tensor:
    dev = _lib.require_cuda(values_left, values_right, offsets_left, offsets_right)
    vl, vr = values_left.contiguous(), values_right.contiguous()
    ol, orr = _same_width(_off(offsets_left), _off(offsets_right))
    B = _batch(ol, orr, vl.shape[0], vr.shape[0], max_len_left, max_len_right)
    D = vl.shape[1]
    out = torch.empty((vl.shape[0] + vr.shape[0], D), dtype=vl.dtype, device=dev)
    i64 = int((ol if ol is not None else orr).dtype == torch.int64)
    with torch.cuda.device(dev):
        _lib.check(
            _lib.lib().hstu_jagged_concat(vl.data_ptr(), vr.data_ptr(), out.data_ptr(), _lib.ptr(ol), _lib.ptr(orr), i64, B,
                                          int(max_len_left or 0), int(max_len_right or 0), int(n_prefix_from_right), D,
                                          vl.element_size(), int(max_seq_len), _lib.stream_ptr(dev)),
            "hstu_jagged_concat")
        _lib.note_launch(1)
    return out


def cuda_split_2D_jagged(max_seq_len, values, total_len_left, total_len_right, max_len_left, max_len_right, offsets_left,
                         offsets_right, n_prefix_to_right: int = 0) -> Tuple[torch.Tensor, torch.Tensor]:
    dev = _lib.require_cuda(values, offsets_left, offsets_right)
    v = values.contiguous()
    ol, orr = _same_width(_off(offsets_left), _off(offsets_right))
    B = _batch(ol, orr, 0, 0, max_len_left, max_len_right)
    D = v.shape[1]
    # sizes of the two sides: given, or derived (a dense side has B * max_len rows; the last offset needs a sync,
    # exactly like the reference triton path, triton_jagged_tensors.py:288)
    if ol is None:
        n_left = B * int(max_len_left)
        n_right = v.shape[0] - n_left
    elif orr is None:
        n_right = B * int(max_len_right)
        n_left = v.shape[0] - n_right
    else:
        if total_len_left is not None and total_len_right is not None:
            n_left, n_right = int(total_len_left), int(total_len_right)
        else:
            n_left = int(ol[-1].item())
            n_right = v.shape[0] - n_left
    left = torch.empty((n_left, D), dtype=v.dtype, device=dev)
    right = torch.empty((n_right, D), dtype=v.dtype, device=dev)
    i64 = int((ol if ol is not None else orr).dtype == torch.int64)
    with torch.cuda.device(dev):
        _lib.check(
            _lib.lib().hstu_jagged_split(v.data_ptr(), left.data_ptr(), right.data_ptr(), _lib.ptr(ol), _lib.ptr(orr), i64, B,
                                         int(max_len_left or 0), int(max_len_right or 0), int(n_prefix_to_right), D,
                                         v.element_size(), int(max_seq_len), _lib.stream_ptr(dev)),
            "hstu_jagged_split")
        _lib.note_launch(1)
    return left, right


class _Concat2DJaggedFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, max_seq_len, values_left, values_right, max_len_left, max_len_right, offsets_left, offsets_right,
                n_prefix):
        ctx.save_for_backward(offsets_left, offsets_right)
        ctx.args = (max_seq_len, max_len_left, max_len_right, n_prefix, values_left.shape[0], values_right.shape[0])
        return cuda_concat_2D_jagged(max_seq_len, values_left, values_right, max_len_left, max_len_right, offsets_left,
                                     offsets_right, n_prefix)

    @staticmethod
    def backward(ctx, dout):
        offsets_left, offsets_right = ctx.saved_tensors
        max_seq_len, max_len_left, max_len_right, n_prefix, nl, nr = ctx.args
        dl, dr = cuda_split_2D_jagged(max_seq_len, dout, nl, nr, max_len_left, max_len_right, offsets_left, offsets_right,
                                      n_prefix)
        return None, dl, dr, None, None, None, None, None


class _Split2DJaggedFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, max_seq_len, values, total_len_left, total_len_right, max_len_left, max_len_right, offsets_left,
                offsets_right, n_prefix):
        ctx.save_for_backward(offsets_left, offsets_right)
        ctx.args = (max_seq_len, max_len_left, max_len_right, n_prefix)
        return cuda_split_2D_jagged(max_seq_len, values, total_len_left, total_len_right, max_len_left, max_len_right,
                                    offsets_left, offsets_right, n_prefix)

    @staticmethod
    def backward(ctx, dleft, dright):
        offsets_left, offsets_right = ctx.saved_tensors
        max_seq_len, max_len_left, max_len_right, n_prefix = ctx.args
        dv = cuda_concat_2D_jagged(max_seq_len, dleft, dright, max_len_left, max_len_right, offsets_left, offsets_right,
                                   n_prefix)
        return None, dv, None, None, None, None, None, None, None


def concat_2D_jagged(
    max_seq_len: int,
    values_left: torch.Tensor,
    values_right: torch.Tensor,
    max_len_left: Optional[int] = None,
    max_len_right: Optional[int] = None,
    offsets_left: Optional[torch.Tensor] = None,
    offsets_right: Optional[torch.Tensor] = None,
    kernel: HammerKernel = HammerKernel.CUDA,
) -> torch.Tensor:
    torch._assert(values_left.dim() == 2, "values_left must be 2D")
    torch._assert(values_right.dim() == 2, "values_right must be 2D")
    torch._assert(values_right.shape[1] == values_left.shape[1],
                  f"values_left shape[1] must be equal to values_right shape[1] {values_left.shape[1]} vs {values_right.shape[1]}")
    require_cuda_kernel(kernel, "concat_2D_jagged")
    return _Concat2DJaggedFunction.apply(max_seq_len, values_left, values_right, max_len_left, max_len_right,
                                         offsets_left, offsets_right, 0)


def split_2D_jagged(
    max_seq_len: int,
    values: torch.Tensor,
    total_len_left: Optional[int] = None,
    total_len_right: Optional[int] = None,
    max_len_left: Optional[int] = None,
    max_len_right: Optional[int] = None,
    offsets_left: Optional[torch.Tensor] = None,
    offsets_right: Optional[torch.Tensor] = None,
    kernel: HammerKernel = HammerKernel.CUDA,
) -> Tuple[torch.Tensor, torch.Tensor]:
    torch._assert(values.dim() == 2, "values must be 2D")
    torch._assert(offsets_left is not None or offsets_right is not None,
                  "offsets_left and offsets_right cannot be None at the same time")
    if offsets_left is None:
        torch._assert(max_len_left is not None, "max_len_left must be provided when offsets_left is None")
    if offsets_right is None:
        torch._assert(max_len_right is not None, "max_len_right must be provided when offsets_right is None")
    if offsets_left is not None and offsets_right is not None:
        torch._assert(offsets_left.shape[0] == offsets_right.shape[0],
                      "offsets_left shape[0] must be equal to offsets_right shape[0]")
    require_cuda_kernel(kernel, "split_2D_jagged")
    return _Split2DJaggedFunction.apply(max_seq_len, values, total_len_left, total_len_right, max_len_left, max_len_right,
                                        offsets_left, offsets_right, 0)


def hstu_split_l2_embeddings(max_seq_len: int, x: torch.Tensor, prefix_offsets: torch.Tensor, l2_offsets: torch.Tensor,
                             contextual_seq_len: int, kernel: HammerKernel = HammerKernel.CUDA):
    require_cuda_kernel(kernel, "hstu_split_l2_embeddings")
    return _Split2DJaggedFunction.apply(max_seq_len, x, None, None, None, None, prefix_offsets, l2_offsets,
                                        contextual_seq_len)


def hstu_concat_l2_embeddings(max_prefix_len: int, prefix_x: torch.Tensor, prefix_offsets: torch.Tensor, max_l2_len: int,
                              l2_x: torch.Tensor, l2_offsets: torch.Tensor, contextual_seq_len: int,
                              kernel: HammerKernel = HammerKernel.CUDA) -> torch.Tensor:
    require_cuda_kernel(kernel, "hstu_concat_l2_embeddings")
    return _Concat2DJaggedFunction.apply(max_prefix_len + max_l2_len, prefix_x, l2_x, max_prefix_len, max_l2_len,
                                         prefix_offsets, l2_offsets, contextual_seq_len)


# ------------------------------------------------------------------------------------------------------------------
# jagged x dense batched matmul + broadcast bias  (ops/jagged_tensors.py:210-253 of the reference)
# ------------------------------------------------------------------------------------------------------------------
def _bmm(jagged, dense, bias, seq_offsets, max_seq_len, n_out, transposed):
    dev = jagged.device
    B = dense.shape[0]
    K = jagged.shape[1]
    out = torch.empty((jagged.shape[0], n_out), dtype=jagged.dtype, device=dev)
    with torch.cuda.device(dev), _lib.timed("jagged_bmm", dev):
        _lib.check(_lib.lib().hstu_jagged_dense_bmm_broadcast_add(
            jagged.data_ptr(), dense.data_ptr(), _lib.ptr(bias), out.data_ptr(), seq_offsets.data_ptr(),
            int(seq_offsets.dtype == torch.int64), B, K, n_out, int(max_seq_len), int(transposed), _lib.dtype_code(jagged),
            _lib.stream_ptr(dev)), "hstu_jagged_dense_bmm_broadcast_add")
        _lib.note_launch(1)
    return out


class _JaggedDenseBmmBroadcastAddFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, max_seq_len, seq_offsets, jagged, dense, bias):
        _lib.require_cuda(jagged, dense, bias, seq_offsets)
        if not (jagged.dtype == dense.dtype == bias.dtype):
            raise RuntimeError("jagged_dense_bmm_broadcast_add: jagged, dense and bias must share a dtype")
        jagged, dense, bias = jagged.contiguous(), dense.contiguous(), bias.contiguous()
        seq_offsets = _off(seq_offsets)
        ctx.save_for_backward(seq_offsets, jagged, dense)
        ctx.max_seq_len = int(max_seq_len)
        return _bmm(jagged, dense, bias, seq_offsets, max_seq_len, dense.shape[2], False)

    @staticmethod
    def backward(ctx, dout):
        seq_offsets, jagged, dense = ctx.saved_tensors
        dev = dout.device
        dout = dout.contiguous()
        B, K, N = dense.shape
        # d_jagged[rows of b] = dout[rows of b] @ dense[b]^T : the same kernel with the dense operand read transposed
        d_jagged = _bmm(dout, dense, None, seq_offsets, ctx.max_seq_len, K, True)
        d_dense = torch.empty_like(dense)
        d_bias = torch.empty((B, N), dtype=dense.dtype, device=dev)
        with torch.cuda.device(dev), _lib.timed("jagged_bmm_wgrad", dev):
            _lib.check(_lib.lib().hstu_jagged_dense_bmm_wgrad(
                jagged.data_ptr(), dout.data_ptr(), d_dense.data_ptr(), d_bias.data_ptr(), seq_offsets.data_ptr(),
                int(seq_offsets.dtype == torch.int64), B, K, N, ctx.max_seq_len, _lib.dtype_code(jagged), _lib.stream_ptr(dev)),
                "hstu_jagged_dense_bmm_wgrad")
            _lib.note_launch(1)
        return None, None, d_jagged, d_dense, d_bias


def jagged_dense_bmm_broadcast_add(
    max_seq_len: int,
    seq_offsets: torch.Tensor,
    jagged: torch.Tensor,
    dense: torch.Tensor,
    bias: torch.Tensor,
    kernel: HammerKernel = HammerKernel.CUDA,
) -> torch.Tensor:
    """Drop-in for generative_recommenders.ops.jagged_tensors.jagged_dense_bmm_broadcast_add (jagged_tensors.py:210-253):
    out = jagged x dense + bias with jagged (sum_B(M_i), K), dense (B, K, N), bias (B, N) -> (sum_B(M_i), N)."""
    _, K = jagged.shape
    B, _, N = dense.shape
    torch._assert(dense.shape[1] == K, "wrong dense shape[1]")
    torch._assert(seq_offsets.shape[0] == B + 1, "wrong seq_offsets shape[0]")
    torch._assert(bias.shape[0] == B, "wrong bias shape[0]")
    torch._assert(bias.shape[1] == N, "wrong bias shape[1]")
    require_cuda_kernel(kernel, "jagged_dense_bmm_broadcast_add")
    return _JaggedDenseBmmBroadcastAddFunction.apply(max_seq_len, seq_offsets, jagged, dense, bias)
