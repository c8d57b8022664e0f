"""TEST INFRASTRUCTURE ONLY -- the non-causal (causal=False) attention of the reference eager path, restated on the CPU.

The mask is ops/pytorch/pt_hstu_attention.py:33-84 (_get_valid_attn_mask) with causal=False, restricted to the real
positions of one sequence, as oracle/hstu_oracle.py::attn_valid_mask restates it for causal=True: the same ids (the
contextual prefix shares id 0, targets are clamped to max_ids), dist = |id_i - id_j| (:64-65), valid = (i == j) |
(dist > 0), then max_attn_len / min_full_attn_seq_len on dist and the contextual rule.  The forward and backward are those
of oracle/hstu_oracle.py (hstu_mha_fwd / hstu_mha_bwd) under this mask; the causal oracle itself is unchanged.
Pinned against tests/golden/bidir_attn_*.pt (tests/golden/make_golden_bidir.py).
"""
from typing import Optional, Tuple

import numpy as np
import torch


def attn_valid_mask_bidir(length: int, num_targets: Optional[int] = None, max_attn_len: int = 0, contextual_seq_len: int = 0,
                          min_full_attn_seq_len: int = 0, rows: Optional[np.ndarray] = None) -> np.ndarray:
    """Boolean [len(rows), length] validity of (query position i, key position j) under causal=False."""
    pos = np.arange(length, dtype=np.int64)
    ids = pos.copy()
    max_ids = length
    if contextual_seq_len > 0:
        ids = np.maximum(ids - contextual_seq_len + 1, 0)
        max_ids = max_ids - contextual_seq_len + 1
    if num_targets is not None:
        max_ids = max_ids - int(num_targets)
        ids = np.minimum(ids, max_ids)
    if rows is None:
        rows = pos
    row_ids = ids[rows].reshape(-1, 1)
    col_ids = ids.reshape(1, -1)
    dist = np.abs(row_ids - col_ids)  # :64-65, causal=False
    valid = (rows.reshape(-1, 1) == pos.reshape(1, -1)) | (dist > 0)
    if max_attn_len > 0:
        if min_full_attn_seq_len > 0:
            valid &= (dist <= max_attn_len) | (row_ids >= max_ids - min_full_attn_seq_len)
        else:
            valid &= dist <= max_attn_len
    if contextual_seq_len > 0:
        valid |= (row_ids == 0) & (col_ids < max_ids)
    return valid


def _per_sequence(seq_offsets, max_seq_len, num_targets, max_attn_len, contextual_seq_len, min_full_attn_seq_len):
    off = seq_offsets.detach().cpu().numpy().astype(np.int64)
    nt = None if num_targets is None else num_targets.detach().cpu().numpy()
    for b in range(len(off) - 1):
        s, e = int(off[b]), int(off[b + 1])
        n = min(e - s, max_seq_len)  # jagged_to_padded_dense truncates rows >= N; they stay zero
        if n <= 0:
            continue
        m = attn_valid_mask_bidir(n, None if nt is None else int(nt[b]), max_attn_len, contextual_seq_len,
                                  min_full_attn_seq_len)
        yield s, n, torch.from_numpy(m)


def hstu_mha_fwd_bidir(max_seq_len: int, alpha: float, q, k, v, seq_offsets, num_targets=None, max_attn_len: int = 0,
                       contextual_seq_len: int = 0, min_full_attn_seq_len: int = 0,
                       dtype: torch.dtype = torch.float64) -> torch.Tensor:
    """O = (silu(alpha Q K^T) / N * mask) V per (sequence, head) in `dtype`: pt_hstu_attention.py:130-171 with causal=False."""
    L, H, _ = q.shape
    out = torch.zeros(L, H, v.shape[2], dtype=dtype)
    for s, n, m in _per_sequence(seq_offsets, max_seq_len, num_targets, max_attn_len, contextual_seq_len,
                                 min_full_attn_seq_len):
        qb, kb, vb = (t[s:s + n].to(dtype).transpose(0, 1) for t in (q, k, v))
        p = torch.nn.functional.silu(torch.matmul(qb, kb.transpose(1, 2)) * alpha) / max_seq_len * m.to(dtype)
        out[s:s + n] = torch.matmul(p, vb).transpose(0, 1)
    return out


def hstu_mha_bwd_bidir(max_seq_len: int, alpha: float, dout, q, k, v, seq_offsets, num_targets=None, max_attn_len: int = 0,
                       contextual_seq_len: int = 0, min_full_attn_seq_len: int = 0,
                       dtype: torch.dtype = torch.float64) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """The explicit gradient of hstu_mha_fwd_bidir (the formulas of oracle/hstu_oracle.py::hstu_mha_bwd)."""
    dq, dk, dv = (torch.zeros(t.shape, dtype=dtype) for t in (q, k, v))
    c = 1.0 / max_seq_len
    for s, n, m in _per_sequence(seq_offsets, max_seq_len, num_targets, max_attn_len, contextual_seq_len,
                                 min_full_attn_seq_len):
        m = m.to(dtype)
        qb, kb, vb, dob = (t[s:s + n].to(dtype).transpose(0, 1) for t in (q, k, v, dout))
        S = torch.matmul(qb, kb.transpose(1, 2)) * alpha
        sig = torch.sigmoid(S)
        P = c * S * sig * m
        dv[s:s + n] = torch.matmul(P.transpose(1, 2), dob).transpose(0, 1)
        dS = c * torch.matmul(dob, vb.transpose(1, 2)) * sig * (1.0 + S * (1.0 - sig)) * m
        dq[s:s + n] = (alpha * torch.matmul(dS, kb)).transpose(0, 1)
        dk[s:s + n] = (alpha * torch.matmul(dS.transpose(1, 2), qb)).transpose(0, 1)
    return dq, dk, dv
