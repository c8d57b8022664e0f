"""Research-path HSTU block on the H100 ops (SURVEY.md section 8 row a11).

Mirrors generative_recommenders/research/modeling/sequential/hstu.py:
  * `RelativeBucketedTimeAndPositionBasedBias` (:87-144) -- here only the parameter container (`_ts_w [num_buckets + 1]`,
    `_pos_w [2 n - 1]`); the bias itself is evaluated inside the attention kernel, never materialised as [B, n, n].
  * `SequentialTransductionUnitJagged` (:226-444), normalization "rel_bias" / "hstu_rel_bias", linear_config "uvqk",
    training / full-sequence forward:  LN (no affine) -> mm -> SiLU on all of uvqk -> split u|v|q|k ->
    silu(q k^T + rel_bias) / n under the causal mask -> u * LN(attn)  (or cat[u, a, u*a], a = LN(attn)) -> dropout ->
    Linear(+bias) + x.
Parameter names (`_uvqk`, `_o.weight`, `_o.bias`, `_rel_attn_bias._ts_w`, `_rel_attn_bias._pos_w`) are the reference's, so
its state dicts load unchanged.  Incremental decoding (`delta_x_offsets`, `cache`, `return_cache_states`, hstu.py:284-444) is
implemented with the reference's cache layout (v jagged, padded q / k [B, n, H dqk], outputs jagged): the delta rows are
projected, scattered into the cache, the attention is re-evaluated on the updated sequences by the same kernel and the delta rows
are taken from it -- the same work the reference does, without the [B, H, n, n] tensors.  The "softmax_rel_bias" ablation raises.
"""
from typing import Optional, Tuple

import torch

from ..common import HammerKernel, HammerModule
from ..ops.hstu_attention import hstu_rel_bias_attention
from ..ops.hstu_compute import _SiluFunction, hstu_compute_output
from ..ops.layer_norm import layer_norm


class RelativeBucketedTimeAndPositionBasedBias(torch.nn.Module):
    """Parameters of the bucketed time + position bias (research hstu.py:87-108).  `bucketization_fn` is fixed to the one the
    reference configures (`floor(log(max(|dt|, 1)) / 0.301)`, hstu.py:610-612): it is compiled into the attention kernel."""

    def __init__(self, max_seq_len: int, num_buckets: int = 128) -> None:
        super().__init__()
        self._max_seq_len = max_seq_len
        self._num_buckets = num_buckets
        self._ts_w = torch.nn.Parameter(torch.empty(num_buckets + 1).normal_(mean=0, std=0.02))
        self._pos_w = torch.nn.Parameter(torch.empty(2 * max_seq_len - 1).normal_(mean=0, std=0.02))


class SequentialTransductionUnitJagged(HammerModule):
    def __init__(
        self,
        embedding_dim: int,
        linear_hidden_dim: int,
        attention_dim: int,
        dropout_ratio: float,
        attn_dropout_ratio: float,
        num_heads: int,
        linear_activation: str,
        relative_attention_bias_module: Optional[RelativeBucketedTimeAndPositionBasedBias] = None,
        normalization: str = "rel_bias",
        linear_config: str = "uvqk",
        concat_ua: bool = False,
        epsilon: float = 1e-6,
        max_length: Optional[int] = None,
    ) -> None:
        super().__init__()
        if linear_config != "uvqk":
            raise ValueError(f"Unknown linear_config {linear_config}")
        if normalization not in ("rel_bias", "hstu_rel_bias"):
            raise NotImplementedError(f"normalization {normalization!r}: only the HSTU (silu) attention is built for H100")
        if linear_activation != "silu":
            raise NotImplementedError("linear_activation must be 'silu' (the setting of every reference config)")
        if relative_attention_bias_module is None:
            raise ValueError("relative_attention_bias_module is required for rel_bias normalization (hstu.py:342)")
        if attn_dropout_ratio != 0.0:
            raise NotImplementedError("attention dropout is not supported (unused by the reference's own path, hstu.py:150-223)")
        self._embedding_dim = embedding_dim
        self._linear_dim = linear_hidden_dim
        self._attention_dim = attention_dim
        self._dropout_ratio = dropout_ratio
        self._attn_dropout_ratio = attn_dropout_ratio
        self._num_heads = num_heads
        self._rel_attn_bias = relative_attention_bias_module
        self._normalization = normalization
        self._linear_config = linear_config
        self._linear_activation = linear_activation
        self._concat_ua = concat_ua
        self._eps = epsilon
        self._uvqk = torch.nn.Parameter(
            torch.empty((embedding_dim, linear_hidden_dim * 2 * num_heads + attention_dim * num_heads * 2)).normal_(mean=0, std=0.02))
        self._o = torch.nn.Linear(in_features=linear_hidden_dim * num_heads * (3 if concat_ua else 1), out_features=embedding_dim)
        torch.nn.init.xavier_uniform_(self._o.weight)
        # LayerNorm without affine parameters (hstu.py:276-282) = the affine kernel with constant ones / zeros
        self.register_buffer("_ones_in", torch.ones(embedding_dim), persistent=False)
        self.register_buffer("_zeros_in", torch.zeros(embedding_dim), persistent=False)
        self.register_buffer("_ones_attn", torch.ones(linear_hidden_dim * num_heads), persistent=False)
        self.register_buffer("_zeros_attn", torch.zeros(linear_hidden_dim * num_heads), persistent=False)

    def _check_mask(self, invalid_attn_mask: torch.Tensor, n: int) -> None:
        """The kernel applies the causal mask the reference builds (hstu.py:626-638,704: 1 - triu(ones(n, n), 1) = tril, 1 = may
        attend) and never reads this tensor; anything else would be silently ignored, so it is rejected.  Checked once per mask
        tensor (one device sync)."""
        key = (invalid_attn_mask.data_ptr(), invalid_attn_mask._version, tuple(invalid_attn_mask.shape))
        if getattr(self, "_mask_ok", None) == key:
            return
        if invalid_attn_mask.dim() < 2 or invalid_attn_mask.size(-2) != n:
            raise RuntimeError(f"invalid_attn_mask must be [..., n, n], got {tuple(invalid_attn_mask.shape)}")
        causal = torch.tril(torch.ones(n, n, device=invalid_attn_mask.device, dtype=torch.float32))
        if not bool((invalid_attn_mask.float() == causal).all()):
            raise NotImplementedError("only the causal invalid_attn_mask of the reference (tril(ones)) is supported by the CUDA attention")
        self._mask_ok = key

    def forward(
        self,
        x: torch.Tensor,
        x_offsets: torch.Tensor,
        all_timestamps: Optional[torch.Tensor],
        invalid_attn_mask: torch.Tensor,
        delta_x_offsets: Optional[Tuple[torch.Tensor, torch.Tensor]] = None,
        cache=None,
        return_cache_states: bool = False,
    ):
        """x [sum_i N_i, D]; x_offsets [B + 1]; all_timestamps [B, n] int64 or None; invalid_attn_mask [n, n] (or [B, n, n])
        -- only its size is used: the kernel applies the causal (lower-triangular) mask the reference builds (hstu.py:626-638).
        Returns (x', (v, padded_q, padded_k, x')) like the reference; padded q / k are only built when a cache is asked for
        (return_cache_states=True) or updated (delta_x_offsets)."""
        kern = self.hammer_kernel()
        if kern != HammerKernel.CUDA:
            raise RuntimeError(f"generative_recommenders_b200 only implements HammerKernel.CUDA (got {kern})")
        n = invalid_attn_mask.size(-1)
        self._check_mask(invalid_attn_mask, n)
        if n != self._rel_attn_bias._max_seq_len:
            raise RuntimeError(f"invalid_attn_mask is {n} x {n} but the relative bias module was built for max_seq_len "
                               f"{self._rel_attn_bias._max_seq_len}")
        H, dqk, dv = self._num_heads, self._attention_dim, self._linear_dim
        B = x_offsets.numel() - 1
        delta = delta_x_offsets is not None
        if delta:
            # hstu.py:309-315: everything below is restricted to the rows delta_x_offsets[0]; the cache holds the rest
            if cache is None:
                raise RuntimeError("delta_x_offsets needs the cache of a previous call (return_cache_states=True)")
            cached_v, cached_q, cached_k, cached_outputs = cache
            if cached_q is None or cached_k is None:
                raise RuntimeError("the cache was produced without return_cache_states=True: padded q / k are missing")
            x = x[delta_x_offsets[0], :]
        L_full = int(cached_v.shape[0]) if delta else x.shape[0]
        normed_x = layer_norm(x, self._ones_in, self._zeros_in, self._eps, kernel=kern)
        mm = _SiluFunction.apply(torch.mm(normed_x, self._uvqk.to(x.dtype)))
        u, v, q, k = torch.split(mm, [dv * H, dv * H, dqk * H, dqk * H], dim=1)
        padded_q = padded_k = None
        if delta or return_cache_states:
            # row (b, position) of every jagged row -> its slot b * n + position in the padded [B * n, .] cache layout
            lengths = x_offsets[1:] - x_offsets[:-1]
            seq_of_row = torch.repeat_interleave(torch.arange(B, device=x.device), lengths, output_size=L_full)
            slot_of_row = torch.arange(L_full, device=x.device) - x_offsets[:-1][seq_of_row] + seq_of_row * n
        if delta:
            v = cached_v.index_copy_(0, delta_x_offsets[0], v)                       # hstu.py:341-342
            flat = delta_x_offsets[1] + torch.arange(0, B * n, n, device=x.device, dtype=delta_x_offsets[1].dtype)
            padded_q = cached_q.view(B * n, -1).index_copy_(0, flat, q).view(B, n, -1)  # hstu.py:168-195
            padded_k = cached_k.view(B * n, -1).index_copy_(0, flat, k).view(B, n, -1)
            q = padded_q.view(B * n, -1)[slot_of_row]                                 # back to the jagged layout the kernel reads
            k = padded_k.view(B * n, -1)[slot_of_row]
        elif return_cache_states:
            padded_q = torch.zeros(B * n, H * dqk, dtype=q.dtype, device=x.device).index_copy_(0, slot_of_row, q.detach()).view(B, n, -1)
            padded_k = torch.zeros(B * n, H * dqk, dtype=k.dtype, device=x.device).index_copy_(0, slot_of_row, k.detach()).view(B, n, -1)
        rb = self._rel_attn_bias
        attn = hstu_rel_bias_attention(
            n, q.reshape(L_full, H, dqk).contiguous(), k.reshape(L_full, H, dqk).contiguous(), v.reshape(L_full, H, dv).contiguous(),
            x_offsets, rb._pos_w, rb._ts_w if all_timestamps is not None else None, all_timestamps,
        ).reshape(L_full, H * dv)
        if delta:
            attn = attn[delta_x_offsets[0], :]                                       # hstu.py:421-425
        residual = x + self._o.bias.to(x.dtype)
        # u * LN(attn) [or cat(u, a, u * a), a = LN(attn): concat mode 2 of the fused kernel] -> dropout -> x + y W_o: the fused
        # output stage of the STU block (one kernel forward, one backward; nothing materialised in between)
        out = hstu_compute_output(
            attn=attn, u=u.contiguous(), x=residual, norm_weight=self._ones_attn, norm_bias=self._zeros_attn, norm_eps=self._eps,
            output_weight=self._o.weight.t(), num_heads=H, linear_dim=dv, dropout_ratio=self._dropout_ratio,
            training=self.training, concat_ux=2 if self._concat_ua else False, group_norm=False, recompute_y_in_backward=False,
            kernel=kern,
        )
        if delta:
            out = cached_outputs.index_copy_(0, delta_x_offsets[0], out)              # hstu.py:439-442
        return out, (v.contiguous() if return_cache_states else v, padded_q, padded_k, out)
