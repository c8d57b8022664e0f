"""Block-level fused ops of one HSTU layer on H100.

Same surface as generative_recommenders/ops/hstu_compute.py:50-259:
  hstu_compute_uqvk              LN -> addmm -> split [u|v|q|k] -> silu(u)
  hstu_compute_output            y = u * Norm(attn) [concat(u, attn, y)] -> dropout -> x + y W_o
  hstu_preprocess_and_attention  the first one fused with the jagged attention under ONE autograd node; q/k/v are strided
                                 views of `uvqk` and dq/dk/dv are written in place into `duvqk`
                                 (layout contract of ops/cpp/cuda_hstu_preprocess_and_attention.py:98-131,254-306).
Dense GEMMs go through torch.addmm / torch.mm (cuBLAS); everything else is a kernel of libhstu_b200.so.
"""
from typing import Optional, Tuple

import torch

from .. import _lib
from ..common import HammerKernel, require_cuda_kernel
from .hstu_attention import cuda_hstu_attention_bwd, cuda_hstu_attention_fwd, hstu_mha
from .layer_norm import _partial, cuda_layer_norm_bwd, cuda_layer_norm_fwd, layer_norm


# ------------------------------------------------------------------------------------------------------------------
# SiLU on a strided column block
# ------------------------------------------------------------------------------------------------------------------
def cuda_silu_fwd(x: torch.Tensor) -> torch.Tensor:
    dev = _lib.require_cuda(x)
    n, c = x.shape
    y = torch.empty((n, c), dtype=x.dtype, device=dev)
    with torch.cuda.device(dev), _lib.timed("silu_fwd", dev):
        _lib.check(_lib.lib().hstu_silu_fwd(x.data_ptr(), y.data_ptr(), n, c, x.stride(0), y.stride(0), _lib.dtype_code(x),
                                            _lib.stream_ptr(dev)), "hstu_silu_fwd")
        _lib.note_launch(1)
    return y


def cuda_silu_bwd(dy: torch.Tensor, x: torch.Tensor, dx: torch.Tensor) -> None:
    dev = x.device
    n, c = x.shape
    dy = dy if dy.stride(-1) == 1 else dy.contiguous()
    with torch.cuda.device(dev), _lib.timed("silu_bwd", dev):
        _lib.check(_lib.lib().hstu_silu_bwd(dy.data_ptr(), x.data_ptr(), dx.data_ptr(), n, c, dy.stride(0), x.stride(0),
                                            dx.stride(0), _lib.dtype_code(x), _lib.stream_ptr(dev)), "hstu_silu_bwd")
        _lib.note_launch(1)


class _SiluFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        ctx.save_for_backward(x)
        return cuda_silu_fwd(x)

    @staticmethod
    def backward(ctx, dy):
        (x,) = ctx.saved_tensors
        dx = torch.empty(x.shape, dtype=x.dtype, device=x.device)
        cuda_silu_bwd(dy, x, dx)
        return dx


def hstu_compute_uqvk(
    x: torch.Tensor, norm_weight: torch.Tensor, norm_bias: torch.Tensor, norm_eps: float, num_heads: int, attn_dim: int,
    hidden_dim: int, uvqk_weight: torch.Tensor, uvqk_bias: torch.Tensor, kernel: HammerKernel = HammerKernel.CUDA,
) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
    require_cuda_kernel(kernel, "hstu_compute_uqvk")
    normed_x = layer_norm(x, weight=norm_weight, bias=norm_bias, eps=norm_eps, kernel=kernel)
    uvqk = torch.addmm(uvqk_bias, normed_x, uvqk_weight)
    u, v, q, k = torch.split(
        uvqk, [hidden_dim * num_heads, hidden_dim * num_heads, attn_dim * num_heads, attn_dim * num_heads], dim=1)
    u = _SiluFunction.apply(u)
    return (u, q.view(-1, num_heads, attn_dim), k.view(-1, num_heads, attn_dim), v.view(-1, num_heads, hidden_dim))


# ------------------------------------------------------------------------------------------------------------------
# output stage
# ------------------------------------------------------------------------------------------------------------------
def cuda_norm_mul_dropout_fwd(attn, u, w, b, eps, p, seed, silu_u, concat_ux, group_norm, num_heads, linear_dim):
    dev = _lib.require_cuda(attn, u, w, b)
    n = attn.shape[0]
    width = num_heads * linear_dim
    out = torch.empty((n, width * (3 if concat_ux else 1)), dtype=attn.dtype, device=dev)
    nstat = n * (num_heads if group_norm else 1)
    mean = torch.empty(nstat, dtype=torch.float32, device=dev)
    rstd = torch.empty(nstat, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev), _lib.timed("nmd_fwd", dev):
        _lib.check(
            _lib.lib().hstu_norm_mul_dropout_fwd(attn.data_ptr(), u.data_ptr(), w.data_ptr(), b.data_ptr(), out.data_ptr(),
                                                 mean.data_ptr(), rstd.data_ptr(), n, num_heads, linear_dim, attn.stride(0),
                                                 u.stride(0), eps, p, seed, _lib.dtype_code(attn), int(silu_u),
                                                 int(concat_ux), int(group_norm), _lib.stream_ptr(dev)),
            "hstu_norm_mul_dropout_fwd")
        _lib.note_launch(1)
    return out, mean, rstd


def cuda_norm_mul_dropout_bwd(dy, attn, u, w, b, mean, rstd, p, seed, silu_u, concat_ux, group_norm, num_heads,
                              linear_dim):
    dev = attn.device
    n = attn.shape[0]
    width = num_heads * linear_dim
    np_ = num_heads if group_norm else width
    dattn = torch.empty((n, width), dtype=attn.dtype, device=dev)
    du = torch.empty((n, width), dtype=attn.dtype, device=dev)
    dw = torch.empty(np_, dtype=torch.float32, device=dev)
    db = torch.empty(np_, dtype=torch.float32, device=dev)
    part = _partial(np_, dev)
    dy = dy.contiguous()
    with torch.cuda.device(dev), _lib.timed("nmd_bwd", dev):
        _lib.check(
            _lib.lib().hstu_norm_mul_dropout_bwd(dy.data_ptr(), attn.data_ptr(), u.data_ptr(), w.data_ptr(), b.data_ptr(),
                                                 mean.data_ptr(), rstd.data_ptr(), dattn.data_ptr(), du.data_ptr(),
                                                 dw.data_ptr(), db.data_ptr(), part.data_ptr(), n, num_heads, linear_dim,
                                                 attn.stride(0), u.stride(0), dattn.stride(0), du.stride(0), p, seed,
                                                 _lib.dtype_code(attn), int(silu_u), int(concat_ux), int(group_norm),
                                                 _lib.stream_ptr(dev)),
            "hstu_norm_mul_dropout_bwd")
        _lib.note_launch(2)
    return dattn, du, dw, db


def _next_dropout_seed(dev: torch.device, numel: int) -> int:
    """Seed of the counter-based dropout generator, drawn from the CUDA generator of `dev` the way torch's own dropout consumes
    it: (initial seed, philox offset) identify the call and the offset advances by the number of random words used.  So
    `torch.cuda.manual_seed(s)` makes the masks reproducible, ranks seeded differently get different masks, and the CPU RNG
    stream of the caller is left alone."""
    gen = torch.cuda.default_generators[dev.index if dev.index is not None else torch.cuda.current_device()]
    off = gen.get_offset()
    gen.set_offset(off + ((numel + 3) // 4 + 3) // 4 * 4)
    return (gen.initial_seed() * 0x9E3779B97F4A7C15 + off * 0xD1B54A32D192ED03 + 0x2545F4914F6CDD1D) & (2**64 - 1)


def _row_major(t: torch.Tensor) -> torch.Tensor:
    return t if t.stride(-1) == 1 else t.contiguous()


class _HSTUComputeOutputFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, attn, u, x, norm_weight, norm_bias, output_weight, eps, dropout_ratio, training, concat_ux,
                group_norm, num_heads, linear_dim, silu_u, recompute_y):
        attn, u = _row_major(attn), _row_major(u)
        w = norm_weight.to(attn.dtype).contiguous()
        b = norm_bias.to(attn.dtype).contiguous()
        p = float(dropout_ratio) if training else 0.0
        seed = _next_dropout_seed(attn.device, attn.numel() * (3 if concat_ux else 1)) if p > 0.0 else 0
        y, mean, rstd = cuda_norm_mul_dropout_fwd(attn, u, w, b, eps, p, seed, silu_u, concat_ux, group_norm, num_heads,
                                                  linear_dim)
        out = torch.addmm(x, y, output_weight.to(x.dtype))
        ctx.save_for_backward(attn, u, norm_weight, norm_bias, output_weight, mean, rstd, None if recompute_y else y)
        ctx.cfg = (eps, p, seed, silu_u, concat_ux, group_norm, num_heads, linear_dim)
        return out

    @staticmethod
    def backward(ctx, dout):
        attn, u, norm_weight, norm_bias, output_weight, mean, rstd, y = ctx.saved_tensors
        eps, p, seed, silu_u, concat_ux, group_norm, num_heads, linear_dim = ctx.cfg
        w = norm_weight.to(attn.dtype).contiguous()
        b = norm_bias.to(attn.dtype).contiguous()
        if y is None:
            y, _, _ = cuda_norm_mul_dropout_fwd(attn, u, w, b, eps, p, seed, silu_u, concat_ux, group_norm, num_heads,
                                                linear_dim)
        wo = output_weight.to(dout.dtype)
        dy = torch.mm(dout, wo.t())
        dwo = torch.mm(y.t(), dout)
        dattn, du, dw, db = cuda_norm_mul_dropout_bwd(dy, attn, u, w, b, mean, rstd, p, seed, silu_u, concat_ux,
                                                      group_norm, num_heads, linear_dim)
        return (dattn, du, dout, dw.to(norm_weight.dtype), db.to(norm_bias.dtype), dwo.to(output_weight.dtype), None, None,
                None, None, None, None, None, None, None)


def hstu_compute_output(
    attn: torch.Tensor, u: torch.Tensor, x: torch.Tensor, norm_weight: torch.Tensor, norm_bias: torch.Tensor,
    norm_eps: float, output_weight: torch.Tensor, num_heads: int, linear_dim: int, dropout_ratio: float, training: bool,
    concat_ux: bool, group_norm: bool, recompute_y_in_backward: bool, kernel: HammerKernel = HammerKernel.CUDA,
    silu_u: bool = False,
) -> torch.Tensor:
    require_cuda_kernel(kernel, "hstu_compute_output")
    return _HSTUComputeOutputFunction.apply(attn, u, x, norm_weight, norm_bias, output_weight, norm_eps, dropout_ratio,
                                            training, concat_ux, group_norm, num_heads, linear_dim, silu_u,
                                            recompute_y_in_backward)


# ------------------------------------------------------------------------------------------------------------------
# LN -> uvqk GEMM -> silu(u) -> jagged attention, one autograd node
# ------------------------------------------------------------------------------------------------------------------
class _HSTUPreprocessAndAttentionFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, norm_weight, norm_bias, norm_eps, num_heads, attn_dim, hidden_dim, uvqk_weight, uvqk_bias,
                max_seq_len, seq_offsets, attn_alpha, num_targets, max_attn_len, contextual_seq_len, recompute_uvqk,
                recompute_normed_x, impl):
        x = _row_major(x)
        normed_x, mean, rstd = cuda_layer_norm_fwd(x, norm_weight, norm_bias, norm_eps, False)
        uvqk = torch.addmm(uvqk_bias, normed_x, uvqk_weight)
        H, dqk, dv = num_heads, attn_dim, hidden_dim
        u_pre, v, q, k = torch.split(uvqk, [dv * H, dv * H, dqk * H, dqk * H], dim=1)
        u = cuda_silu_fwd(u_pre)
        out = cuda_hstu_attention_fwd(max_seq_len, attn_alpha, q.view(-1, H, dqk), k.view(-1, H, dqk), v.view(-1, H, dv),
                                      seq_offsets, num_targets, max_attn_len, contextual_seq_len, 0, impl)
        ctx.save_for_backward(x, norm_weight, norm_bias, uvqk_weight, uvqk_bias, mean, rstd, seq_offsets, num_targets,
                              None if recompute_normed_x else normed_x,
                              None if recompute_uvqk else uvqk)
        ctx.cfg = (norm_eps, H, dqk, dv, max_seq_len, attn_alpha, max_attn_len, contextual_seq_len, impl)
        return u, out.view(-1, H * dv)

    @staticmethod
    def backward(ctx, du, dattn):
        (x, norm_weight, norm_bias, uvqk_weight, uvqk_bias, mean, rstd, seq_offsets, num_targets, normed_x,
         uvqk) = ctx.saved_tensors
        norm_eps, H, dqk, dv, max_seq_len, alpha, max_attn_len, contextual_seq_len, impl = ctx.cfg
        if normed_x is None:
            normed_x, _, _ = cuda_layer_norm_fwd(x, norm_weight, norm_bias, norm_eps, False, save_stats=False)
        if uvqk is None:
            uvqk = torch.addmm(uvqk_bias, normed_x, uvqk_weight)
        u_pre, v, q, k = torch.split(uvqk, [dv * H, dv * H, dqk * H, dqk * H], dim=1)
        duvqk = torch.empty_like(uvqk)
        d_u, d_v, d_q, d_k = torch.split(duvqk, [dv * H, dv * H, dqk * H, dqk * H], dim=1)
        dattn = _row_major(dattn)
        cuda_hstu_attention_bwd(max_seq_len, alpha, dattn.view(-1, H, dv), q.view(-1, H, dqk), k.view(-1, H, dqk),
                                v.view(-1, H, dv), d_q.view(-1, H, dqk), d_k.view(-1, H, dqk), d_v.view(-1, H, dv),
                                seq_offsets, num_targets, max_attn_len, contextual_seq_len, 0, impl)
        cuda_silu_bwd(du, u_pre, d_u)
        d_w = torch.mm(normed_x.t(), duvqk)
        d_b = duvqk.sum(dim=0)
        d_normed = torch.mm(duvqk, uvqk_weight.t())
        dx, dnw, dnb = cuda_layer_norm_bwd(d_normed, x, norm_weight, norm_bias, mean, rstd, False)
        return (dx, dnw.to(norm_weight.dtype), dnb.to(norm_bias.dtype), None, None, None, None, d_w, d_b, None, None, None,
                None, None, None, None, None, None)


def hstu_preprocess_and_attention(
    x: torch.Tensor, norm_weight: torch.Tensor, norm_bias: torch.Tensor, norm_eps: float, num_heads: int, attn_dim: int,
    hidden_dim: int, uvqk_weight: torch.Tensor, uvqk_bias: torch.Tensor, max_seq_len: int, seq_offsets: torch.Tensor,
    attn_alpha: float, causal: bool, num_targets: Optional[torch.Tensor], max_attn_len: int, contextual_seq_len: int,
    recompute_uvqk_in_backward: bool, recompute_normed_x_in_backward: bool, sort_by_length: bool, prefill: bool = False,
    kernel: HammerKernel = HammerKernel.CUDA, impl: int = _lib.IMPL_AUTO,
) -> Tuple[torch.Tensor, torch.Tensor, Optional[torch.Tensor], Optional[torch.Tensor]]:
    torch._assert(max_seq_len > 0, "max_seq_len must be larger than 0")
    torch._assert(x.dim() == 2, "x must be 2-D")
    torch._assert(x.shape[1] == uvqk_weight.shape[0], "x.shape[1] must equal uvqk_weight.shape[0]")
    torch._assert(uvqk_weight.shape[1] == 2 * num_heads * (hidden_dim + attn_dim),
                  "uvqk_weight.shape[1] must equal 2 * num_heads * (hidden_dim + attn_dim)")
    torch._assert(causal is True, "only causal attention is supported.")
    require_cuda_kernel(kernel, "hstu_preprocess_and_attention")
    if not prefill:
        u, attn_output = _HSTUPreprocessAndAttentionFunction.apply(
            x, norm_weight, norm_bias, norm_eps, num_heads, attn_dim, hidden_dim, uvqk_weight, uvqk_bias, max_seq_len,
            seq_offsets, attn_alpha, num_targets, max_attn_len, contextual_seq_len, recompute_uvqk_in_backward,
            recompute_normed_x_in_backward, impl)
        return u, attn_output, None, None
    # prefill: the caller needs k and v for the KV cache (hstu_compute.py:230-259)
    u, q, k, v = hstu_compute_uqvk(x, norm_weight, norm_bias, norm_eps, num_heads, attn_dim, hidden_dim, uvqk_weight,
                                   uvqk_bias, kernel)
    attn_output = hstu_mha(max_seq_len=max_seq_len, alpha=attn_alpha, q=q, k=k, v=v, seq_offsets=seq_offsets, causal=causal,
                           dropout_pr=0.0, training=False, num_targets=num_targets, max_attn_len=max_attn_len,
                           contextual_seq_len=contextual_seq_len, sort_by_length=sort_by_length, kernel=kernel,
                           impl=impl).view(-1, hidden_dim * num_heads)
    return u, attn_output, k, v
