"""TEST INFRASTRUCTURE ONLY -- pure-torch stand-ins for the three `torch.ops.fbgemm.*`
jagged ops the reference's PyTorch-eager path calls (plus `jagged_dense_elementwise_add_jagged_output` for ops/position.py).

The reference (generative_recommenders @ 2e81fab) depends on `fbgemm_gpu>=1.1.0`
(requirements.txt:2 of the reference), which is a third-party dependency that is NOT
vendored in the reference repository.
Its published semantics for the three ops on the hot path are restated here so that the
*unmodified* reference eager code can be imported and run on CPU to generate the golden
vectors in tests/golden/ (see tests/golden/make_golden.py).

Call sites in the reference that pin the semantics:
  * jagged_to_padded_dense : ops/pytorch/pt_hstu_attention.py:97-123,
                             ops/pytorch/pt_jagged_tensors.py:42-53,126-131
  * dense_to_jagged        : ops/pytorch/pt_hstu_attention.py:167-171
  * asynchronous_complete_cumsum : modules/stu.py:97

Nothing in the product package (generative_recommenders_b200/) imports this file.
"""
from typing import List, Optional, Tuple

import torch

_LIB = None


def _jagged_to_padded_dense(
    values: torch.Tensor,
    offsets: List[torch.Tensor],
    max_lengths: List[int],
    padding_value: float = 0.0,
) -> torch.Tensor:
    # values [L, D], offsets [[B+1]] -> [B, max_len, D]; rows >= max_len are truncated.
    assert len(offsets) == 1 and len(max_lengths) == 1
    off = offsets[0].to(torch.int64)
    max_len = int(max_lengths[0])
    B = off.numel() - 1
    squeeze = values.dim() == 1
    v2 = values.unsqueeze(-1) if squeeze else values
    D = v2.shape[1]
    lengths = off[1:] - off[:-1]
    pos = torch.arange(max_len, device=values.device).view(1, max_len)
    valid = pos < lengths.view(B, 1)  # [B, max_len]
    src = (off[:-1].view(B, 1) + pos).clamp_(max=max(v2.shape[0] - 1, 0))
    if v2.shape[0] == 0:
        out = torch.full((B, max_len, D), padding_value, dtype=values.dtype, device=values.device)
    else:
        gathered = v2[src.reshape(-1)].view(B, max_len, D)
        pad = torch.full_like(gathered, padding_value)
        out = torch.where(valid.unsqueeze(-1), gathered, pad)
    return out.squeeze(-1) if squeeze else out


def _dense_to_jagged(
    dense: torch.Tensor,
    x_offsets: List[torch.Tensor],
    total_L: Optional[int] = None,
) -> Tuple[torch.Tensor, List[torch.Tensor]]:
    # dense [B, N, D] -> values [L, D] taking the first len_b rows of each batch entry.  A jagged row past the dense length
    # (len_b > N) gets the padding value 0, as fbgemm writes it, so that there are always offsets[-1] rows.
    assert len(x_offsets) == 1
    off = x_offsets[0].to(torch.int64)
    B, N = dense.shape[0], dense.shape[1]
    lengths = off[1:] - off[:-1]
    longest = int(lengths.max()) if B > 0 else 0
    if longest > N:
        dense = torch.cat([dense, dense.new_zeros((B, longest - N) + tuple(dense.shape[2:]))], dim=1)
        N = longest
    pos = torch.arange(N, device=dense.device).view(1, N)
    valid = pos < lengths.view(B, 1)
    values = dense.reshape(B * N, -1)[valid.reshape(-1)]
    return values, [x_offsets[0]]


def _jagged_dense_elementwise_add_jagged_output(
    x_values: torch.Tensor, x_offsets: List[torch.Tensor], y: torch.Tensor
) -> Tuple[torch.Tensor, List[torch.Tensor]]:
    # x_values [L, D] jagged by x_offsets; y dense [B, N, D]: out[row of (b, n)] = x_values[row] + y[b, n]
    # (call site: ops/pytorch/pt_position.py:130-134)
    assert len(x_offsets) == 1
    picked, _ = _dense_to_jagged(y, x_offsets)
    return x_values + picked, [x_offsets[0]]


def _asynchronous_complete_cumsum(t_in: torch.Tensor) -> torch.Tensor:
    out = torch.zeros(t_in.numel() + 1, dtype=t_in.dtype, device=t_in.device)
    out[1:] = torch.cumsum(t_in, dim=0)
    return out


def install() -> None:
    """Register the shim under namespace `fbgemm` unless a real fbgemm_gpu is present."""
    global _LIB
    if _LIB is not None:
        return
    try:
        import fbgemm_gpu  # noqa: F401

        return
    except Exception:
        pass
    lib = torch.library.Library("fbgemm", "DEF")
    lib.define(
        "jagged_to_padded_dense(Tensor values, Tensor[] offsets, SymInt[] max_lengths, "
        "float padding_value=0.0) -> Tensor"
    )
    lib.define(
        "dense_to_jagged(Tensor dense, Tensor[] x_offsets, SymInt? total_L=None) "
        "-> (Tensor, Tensor[])"
    )
    lib.define("asynchronous_complete_cumsum(Tensor t_in) -> Tensor")
    lib.define(
        "jagged_dense_elementwise_add_jagged_output(Tensor x_values, Tensor[] x_offsets, Tensor y) -> (Tensor, Tensor[])"
    )
    lib.impl("jagged_dense_elementwise_add_jagged_output", _jagged_dense_elementwise_add_jagged_output,
             "CompositeImplicitAutograd")
    lib.impl("jagged_to_padded_dense", _jagged_to_padded_dense, "CompositeImplicitAutograd")
    lib.impl("dense_to_jagged", _dense_to_jagged, "CompositeImplicitAutograd")
    lib.impl("asynchronous_complete_cumsum", _asynchronous_complete_cumsum, "CompositeImplicitAutograd")
    _LIB = lib
