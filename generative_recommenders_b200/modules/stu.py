"""HSTU block (STULayer / STUStack) on the H100 ops.

Parameter names, config fields and forward / cached_forward semantics follow the reference
generative_recommenders/modules/stu.py:64-466 so that checkpoints (`_uvqk_weight`, `_uvqk_beta`,
`_input_norm_{weight,bias}`, `_output_weight`, `_output_norm_{weight,bias}`) load unchanged.
"""
import abc
from dataclasses import dataclass
from typing import List, Optional, Tuple

import torch
from torch.autograd.profiler import record_function

from ..common import HammerModule
from ..ops.hstu_attention import delta_hstu_mha
from ..ops.hstu_compute import hstu_compute_output, hstu_compute_uqvk, hstu_preprocess_and_attention
from ..ops.jagged_tensors import concat_2D_jagged, split_2D_jagged


@dataclass
class STULayerConfig:
    embedding_dim: int
    num_heads: int
    hidden_dim: int
    attention_dim: int
    output_dropout_ratio: float = 0.3
    causal: bool = True
    target_aware: bool = True
    max_attn_len: Optional[int] = None
    attn_alpha: Optional[float] = None
    use_group_norm: bool = False
    recompute_normed_x: bool = True
    recompute_uvqk: bool = True
    recompute_y: bool = True
    sort_by_length: bool = True
    contextual_seq_len: int = 0


class STU(HammerModule, abc.ABC):
    def cached_forward(self, delta_x, num_targets, max_kv_caching_len: int = 0, kv_caching_lengths=None):
        raise NotImplementedError

    @abc.abstractmethod
    def forward(self, x, x_lengths, x_offsets, max_seq_len, num_targets, max_kv_caching_len: int = 0,
                kv_caching_lengths=None):
        pass


def _complete_cumsum(lengths: torch.Tensor) -> torch.Tensor:
    out = torch.zeros(lengths.numel() + 1, dtype=lengths.dtype, device=lengths.device)
    out[1:] = torch.cumsum(lengths, dim=0)
    return out


class STULayer(STU):
    def __init__(self, config: STULayerConfig, is_inference: bool = False) -> None:
        super().__init__(is_inference=is_inference)
        self.reset_kv_cache()
        c = config
        self._num_heads, self._embedding_dim = c.num_heads, c.embedding_dim
        self._hidden_dim, self._attention_dim = c.hidden_dim, c.attention_dim
        self._output_dropout_ratio = c.output_dropout_ratio
        self._target_aware, self._causal = c.target_aware, c.causal
        self._max_attn_len = c.max_attn_len or 0
        self._attn_alpha = c.attn_alpha or 1.0 / (self._attention_dim**0.5)
        self._use_group_norm = c.use_group_norm
        self._recompute_normed_x, self._recompute_uvqk, self._recompute_y = c.recompute_normed_x, c.recompute_uvqk, c.recompute_y
        self._sort_by_length = c.sort_by_length
        self._contextual_seq_len = c.contextual_seq_len
        H, D, dv, dqk = c.num_heads, c.embedding_dim, c.hidden_dim, c.attention_dim
        self._uvqk_weight = torch.nn.Parameter(torch.empty((D, (dv * 2 + dqk * 2) * H)))
        torch.nn.init.xavier_uniform_(self._uvqk_weight)
        self._uvqk_beta = torch.nn.Parameter(torch.zeros((dv * 2 + dqk * 2) * H))
        self._input_norm_weight = torch.nn.Parameter(torch.ones((D,)))
        self._input_norm_bias = torch.nn.Parameter(torch.zeros((D,)))
        self._output_weight = torch.nn.Parameter(torch.empty((dv * H * 3, D)))
        torch.nn.init.xavier_uniform_(self._output_weight)
        nshape = H if c.use_group_norm else dv * H
        self._output_norm_weight = torch.nn.Parameter(torch.ones((nshape,)))
        self._output_norm_bias = torch.nn.Parameter(torch.zeros((nshape,)))

    # ---- KV cache (inference) ----
    def reset_kv_cache(self) -> None:
        self.k_cache: Optional[torch.Tensor] = None
        self.v_cache: Optional[torch.Tensor] = None
        self.kv_caching_offsets: Optional[torch.Tensor] = None
        self.max_kv_caching_len: int = 0

    def update_kv_cache(self, max_seq_len, seq_offsets, k, v, max_kv_caching_len, kv_caching_lengths) -> None:
        if kv_caching_lengths is None:
            return
        kv_off = _complete_cumsum(kv_caching_lengths)
        delta_off = seq_offsets - kv_off
        kern = self.hammer_kernel()
        self.k_cache, _ = split_2D_jagged(max_seq_len=max_seq_len, values=k.flatten(1, 2), max_len_left=None,
                                          max_len_right=None, offsets_left=kv_off, offsets_right=delta_off, kernel=kern)
        self.v_cache, _ = split_2D_jagged(max_seq_len=max_seq_len, values=v.flatten(1, 2), max_len_left=None,
                                          max_len_right=None, offsets_left=kv_off, offsets_right=delta_off, kernel=kern)
        self.max_kv_caching_len = max_kv_caching_len if max_kv_caching_len != 0 else int(kv_caching_lengths.max().item())
        self.kv_caching_offsets = kv_off

    def construct_full_kv(self, delta_k: torch.Tensor, delta_v: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, int, torch.Tensor]:
        L, _ = delta_k.shape
        B = self.kv_caching_offsets.shape[0] - 1
        delta = L // B
        kern = self.hammer_kernel()
        n = self.max_kv_caching_len + delta
        full_k = concat_2D_jagged(max_seq_len=n, values_left=self.k_cache, values_right=delta_k,
                                  max_len_left=self.max_kv_caching_len, max_len_right=delta,
                                  offsets_left=self.kv_caching_offsets, offsets_right=None, kernel=kern)
        full_v = concat_2D_jagged(max_seq_len=n, values_left=self.v_cache, values_right=delta_v,
                                  max_len_left=self.max_kv_caching_len, max_len_right=delta,
                                  offsets_left=self.kv_caching_offsets, offsets_right=None, kernel=kern)
        full_off = self.kv_caching_offsets + delta * torch.arange(B + 1, device=delta_k.device)
        return full_k, full_v, n, full_off

    def _output(self, attn, u, x):
        with record_function("## stu_compute_output ##"):
            return hstu_compute_output(
                attn=attn, u=u, x=x, norm_weight=self._output_norm_weight.to(x.dtype),
                norm_bias=self._output_norm_bias.to(x.dtype), norm_eps=1e-6, dropout_ratio=self._output_dropout_ratio,
                output_weight=self._output_weight.to(x.dtype), group_norm=self._use_group_norm, num_heads=self._num_heads,
                linear_dim=self._hidden_dim, concat_ux=True, training=self.training, kernel=self.hammer_kernel(),
                recompute_y_in_backward=self._recompute_y)

    def forward(self, x, x_lengths, x_offsets, max_seq_len, num_targets, max_kv_caching_len: int = 0,
                kv_caching_lengths: Optional[torch.Tensor] = None) -> torch.Tensor:
        with record_function("## stu_preprocess_and_attention ##"):
            u, attn_output, k, v = hstu_preprocess_and_attention(
                x=x, norm_weight=self._input_norm_weight.to(x.dtype), norm_bias=self._input_norm_bias.to(x.dtype),
                norm_eps=1e-6, num_heads=self._num_heads, attn_dim=self._attention_dim, hidden_dim=self._hidden_dim,
                uvqk_weight=self._uvqk_weight.to(x.dtype), uvqk_bias=self._uvqk_beta.to(x.dtype), max_seq_len=max_seq_len,
                seq_offsets=x_offsets, attn_alpha=self._attn_alpha, causal=self._causal,
                num_targets=num_targets if self._target_aware else None, max_attn_len=self._max_attn_len,
                contextual_seq_len=self._contextual_seq_len, recompute_uvqk_in_backward=self._recompute_uvqk,
                recompute_normed_x_in_backward=self._recompute_normed_x, sort_by_length=self._sort_by_length,
                prefill=kv_caching_lengths is not None, kernel=self.hammer_kernel())
        self.update_kv_cache(max_seq_len, x_offsets, k, v, max_kv_caching_len, kv_caching_lengths)
        return self._output(attn_output, u, x)

    def cached_forward(self, delta_x, num_targets, max_kv_caching_len: int = 0,
                       kv_caching_lengths: Optional[torch.Tensor] = None) -> torch.Tensor:
        if not self._causal:
            raise RuntimeError("STULayer.cached_forward: KV-cached (delta-q) attention is causal only; this layer has "
                               "causal=False")
        with record_function("## stu_compute_uqvk ##"):
            delta_u, delta_q, delta_k, delta_v = hstu_compute_uqvk(
                x=delta_x, norm_weight=self._input_norm_weight.to(delta_x.dtype),
                norm_bias=self._input_norm_bias.to(delta_x.dtype), norm_eps=1e-6, num_heads=self._num_heads,
                attn_dim=self._attention_dim, hidden_dim=self._hidden_dim, uvqk_weight=self._uvqk_weight.to(delta_x.dtype),
                uvqk_bias=self._uvqk_beta.to(delta_x.dtype), kernel=self.hammer_kernel())
        k, v, max_seq_len, seq_offsets = self.construct_full_kv(delta_k.flatten(1, 2), delta_v.flatten(1, 2))
        self.update_kv_cache(max_seq_len, seq_offsets, k.view(-1, self._num_heads, self._attention_dim),
                             v.view(-1, self._num_heads, self._hidden_dim), max_kv_caching_len, kv_caching_lengths)
        k = k.view(-1, self._num_heads, self._attention_dim)
        v = v.view(-1, self._num_heads, self._hidden_dim)
        with record_function("## delta_hstu_mha ##"):
            delta_attn = delta_hstu_mha(
                max_seq_len=max_seq_len, alpha=self._attn_alpha, delta_q=delta_q, k=k, v=v, seq_offsets=seq_offsets,
                num_targets=num_targets if self._target_aware else None, max_attn_len=self._max_attn_len,
                contextual_seq_len=self._contextual_seq_len, kernel=self.hammer_kernel(),
            ).view(-1, self._hidden_dim * self._num_heads)
        return self._output(delta_attn, delta_u, delta_x)


class STUStack(STU):
    def __init__(self, stu_list: List[STU], is_inference: bool = False) -> None:
        super().__init__(is_inference=is_inference)
        self._stu_layers = torch.nn.ModuleList(modules=stu_list)

    def forward(self, x, x_lengths, x_offsets, max_seq_len, num_targets, max_kv_caching_len: int = 0,
                kv_caching_lengths: Optional[torch.Tensor] = None) -> torch.Tensor:
        for layer in self._stu_layers:
            x = layer(x=x, x_lengths=x_lengths, x_offsets=x_offsets, max_seq_len=max_seq_len, num_targets=num_targets,
                      max_kv_caching_len=max_kv_caching_len, kv_caching_lengths=kv_caching_lengths)
        return x

    def cached_forward(self, delta_x, num_targets, max_kv_caching_len: int = 0,
                       kv_caching_lengths: Optional[torch.Tensor] = None) -> torch.Tensor:
        for layer in self._stu_layers:
            delta_x = layer.cached_forward(delta_x=delta_x, num_targets=num_targets,
                                           max_kv_caching_len=max_kv_caching_len, kv_caching_lengths=kv_caching_lengths)
        return delta_x
