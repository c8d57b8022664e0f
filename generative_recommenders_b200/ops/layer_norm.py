"""LayerNorm / SwishLayerNorm / RMSNorm on H100 -- host side of hstu_layer_norm_* / hstu_rms_norm_*.

Same surface as generative_recommenders/ops/layer_norm.py:46-184 (functions + the three HammerModules).
Statistics and parameter gradients are fp32; outputs keep x.dtype (pt_layer_norm.py:24-61).
"""
from typing import List, Optional, Tuple

import torch

from .. import _lib
from ..common import HammerKernel, HammerModule, require_cuda_kernel


def _rows2d(x: torch.Tensor) -> torch.Tensor:
    x2 = x.reshape(-1, x.shape[-1])
    return x2 if x2.stride(-1) == 1 else x2.contiguous()


def _partial(D: int, device) -> torch.Tensor:
    return torch.empty(_lib.lib().hstu_norm_bwd_partial_rows() * 2 * D, dtype=torch.float32, device=device)


def cuda_layer_norm_fwd(x2: torch.Tensor, weight, bias, eps: float, swish: bool,
                        save_stats: bool = True) -> Tuple[torch.Tensor, Optional[torch.Tensor], Optional[torch.Tensor]]:
    dev = _lib.require_cuda(x2, weight, bias)
    n, D = x2.shape
    y = torch.empty((n, D), dtype=x2.dtype, device=dev)
    mean = torch.empty(n, dtype=torch.float32, device=dev) if save_stats else None
    rstd = torch.empty(n, dtype=torch.float32, device=dev) if save_stats else None
    w = None if weight is None else weight.to(x2.dtype).contiguous()
    b = None if bias is None else bias.to(x2.dtype).contiguous()
    with torch.cuda.device(dev), _lib.timed("ln_fwd", dev):
        _lib.check(
            _lib.lib().hstu_layer_norm_fwd(x2.data_ptr(), _lib.ptr(w), _lib.ptr(b), y.data_ptr(), _lib.ptr(mean),
                                           _lib.ptr(rstd), n, D, x2.stride(0), y.stride(0), eps, _lib.dtype_code(x2),
                                           int(swish), _lib.stream_ptr(dev)),
            "hstu_layer_norm_fwd")
        _lib.note_launch(1)
    return y, mean, rstd


def cuda_layer_norm_bwd(dy2, x2, weight, bias, mean, rstd, swish: bool, need_wgrad: bool = True):
    dev = x2.device
    n, D = x2.shape
    dy2 = dy2 if dy2.stride(-1) == 1 else dy2.contiguous()
    dx = torch.empty((n, D), dtype=x2.dtype, device=dev)
    dw = torch.empty(D, dtype=torch.float32, device=dev) if need_wgrad else None
    db = torch.empty(D, dtype=torch.float32, device=dev) if need_wgrad else None
    part = _partial(D, dev) if need_wgrad else None
    w = None if weight is None else weight.to(x2.dtype).contiguous()
    b = None if bias is None else bias.to(x2.dtype).contiguous()
    with torch.cuda.device(dev), _lib.timed("ln_bwd", dev):
        _lib.check(
            _lib.lib().hstu_layer_norm_bwd(dy2.data_ptr(), x2.data_ptr(), _lib.ptr(w), _lib.ptr(b), mean.data_ptr(),
                                           rstd.data_ptr(), dx.data_ptr(), _lib.ptr(dw), _lib.ptr(db), _lib.ptr(part), n,
                                           D, x2.stride(0), dy2.stride(0), dx.stride(0), _lib.dtype_code(x2), int(swish),
                                           _lib.stream_ptr(dev)),
            "hstu_layer_norm_bwd")
        _lib.note_launch(2)
    return dx, dw, db


class _LayerNormFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, eps, swish):
        x2 = _rows2d(x)
        y, mean, rstd = cuda_layer_norm_fwd(x2, weight, bias, eps, swish)
        ctx.save_for_backward(x2, weight, bias, mean, rstd)
        ctx.swish = swish
        ctx.shape = x.shape
        return y.view(x.shape)

    @staticmethod
    def backward(ctx, dy):
        x2, weight, bias, mean, rstd = ctx.saved_tensors
        dx, dw, db = cuda_layer_norm_bwd(dy.reshape(x2.shape), x2, weight, bias, mean, rstd, ctx.swish)
        return dx.view(ctx.shape), dw.to(weight.dtype), db.to(bias.dtype), None, None


def layer_norm(x: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor, eps: float = 1e-5,
               kernel: HammerKernel = HammerKernel.CUDA) -> torch.Tensor:
    require_cuda_kernel(kernel, "layer_norm")
    return _LayerNormFunction.apply(x, weight, bias, eps, False)


def swish_layer_norm(x: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor, eps: float = 1e-5,
                     kernel: HammerKernel = HammerKernel.CUDA) -> torch.Tensor:
    require_cuda_kernel(kernel, "swish_layer_norm")
    return _LayerNormFunction.apply(x, weight, bias, eps, True)


class _RMSNormFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, eps):
        x2 = _rows2d(x).contiguous()
        dev = _lib.require_cuda(x2, weight)
        n, D = x2.shape
        y = torch.empty_like(x2)
        rstd = torch.empty(n, dtype=torch.float32, device=dev)
        w = weight.to(x2.dtype).contiguous()
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().hstu_rms_norm_fwd(x2.data_ptr(), w.data_ptr(), y.data_ptr(), rstd.data_ptr(), n, D, eps,
                                                    _lib.dtype_code(x2), _lib.stream_ptr(dev)), "hstu_rms_norm_fwd")
            _lib.note_launch(1)
        ctx.save_for_backward(x2, weight, rstd)
        ctx.shape = x.shape
        return y.view(x.shape)

    @staticmethod
    def backward(ctx, dy):
        x2, weight, rstd = ctx.saved_tensors
        dev = x2.device
        n, D = x2.shape
        dy2 = dy.reshape(n, D).contiguous()
        dx = torch.empty_like(x2)
        dw = torch.empty(D, dtype=torch.float32, device=dev)
        part = _partial(D, dev)
        w = weight.to(x2.dtype).contiguous()
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().hstu_rms_norm_bwd(dy2.data_ptr(), x2.data_ptr(), w.data_ptr(), rstd.data_ptr(),
                                                    dx.data_ptr(), dw.data_ptr(), part.data_ptr(), n, D,
                                                    _lib.dtype_code(x2), _lib.stream_ptr(dev)), "hstu_rms_norm_bwd")
            _lib.note_launch(2)
        return dx.view(ctx.shape), dw.to(weight.dtype), None


def rms_norm(x: torch.Tensor, weight: torch.Tensor, eps: float = 1e-5) -> torch.Tensor:
    return _RMSNormFunction.apply(x, weight, eps)


class LayerNorm(HammerModule):
    def __init__(self, dim: int, eps: float = 1e-5, is_inference: bool = False) -> None:
        super().__init__(is_inference=is_inference)
        self._normalized_shape: List[int] = [dim]
        self._eps = eps
        self.weight = torch.nn.Parameter(torch.ones(self._normalized_shape))
        self.bias = torch.nn.Parameter(torch.zeros(self._normalized_shape))

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return layer_norm(x=x, weight=self.weight, bias=self.bias, eps=self._eps, kernel=self.hammer_kernel())


class RMSNorm(HammerModule):
    def __init__(self, dim: int, eps: float = 1e-5, is_inference: bool = False) -> None:
        super().__init__(is_inference=is_inference)
        self._eps = eps
        self.weight = torch.nn.Parameter(torch.ones(dim))

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        require_cuda_kernel(self.hammer_kernel(), "RMSNorm")
        return rms_norm(x, self.weight, self._eps)


class SwishLayerNorm(HammerModule):
    def __init__(self, dim: int, eps: float = 1e-5, is_inference: bool = False) -> None:
        super().__init__(is_inference=is_inference)
        self._normalized_shape: List[int] = [dim]
        self.weight = torch.nn.Parameter(torch.ones(self._normalized_shape))
        self.bias = torch.nn.Parameter(torch.zeros(self._normalized_shape))
        self._eps = eps

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return swish_layer_norm(x=x, weight=self.weight, bias=self.bias, eps=self._eps, kernel=self.hammer_kernel())
