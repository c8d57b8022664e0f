"""TEST INFRASTRUCTURE ONLY -- CPU restatement of the reference's HSTU hot path.

This file is the *oracle* for the CUDA kernels: an independent, per-sequence, fp32/fp64
restatement (torch CPU tensors + numpy integer routing; explicit backward formulas for the
attention) of the reference's PyTorch-eager path.  It is imported only by `tests/`,
`__graft_entry__.smoke()` and the `cpu_baseline` / `--impl reference` legs of `bench.py`.
The product package never imports it.

Parity pin: the reference ships no golden vectors for this path (SURVEY.md section 8c), so the
oracle is pinned against outputs of the *unmodified* reference eager code run in the build
container (through oracle/fbgemm_shim.py) -- see tests/golden/make_golden.py and
tests/test_oracle_vs_golden.py.  The third-party fbgemm_gpu jagged ops (>=1.1.0, not vendored)
are restated in the shim; that boundary itself is "parity unpinned" by the reference repo.

Every function cites the reference file:line it follows (paths relative to
generative_recommenders/ of the reference).
"""
from __future__ import annotations

import math
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch

# --------------------------------------------------------------------------------------
# mask
# --------------------------------------------------------------------------------------


def attn_valid_mask(
    length: int,
    num_targets: Optional[int] = None,
    max_attn_len: int = 0,
    contextual_seq_len: int = 0,
    min_full_attn_seq_len: int = 0,
    rows: Optional[np.ndarray] = None,
) -> np.ndarray:
    """Boolean [len(rows), length] validity of (query position i, key position j).

    Follows ops/pytorch/pt_hstu_attention.py:33-84 (_get_valid_attn_mask) restricted to the
    real positions 0..length-1 of one sequence (padded positions never reach the output:
    padded keys are zero rows -> silu(0)=0, padded queries are dropped by dense_to_jagged).
    """
    pos = np.arange(length, dtype=np.int64)
    ids = pos.copy()
    max_ids = length
    if contextual_seq_len > 0:  # :46-49
        ids = np.maximum(ids - contextual_seq_len + 1, 0)
        max_ids = max_ids - contextual_seq_len + 1
    if num_targets is not None:  # :50-55
        max_ids = max_ids - int(num_targets)
        ids = np.minimum(ids, max_ids)
    if rows is None:
        rows = pos
    row_ids = ids[rows].reshape(-1, 1)
    col_ids = ids.reshape(1, -1)
    dist = row_ids - col_ids  # :63
    valid = (rows.reshape(-1, 1) == pos.reshape(1, -1)) | (dist > 0)  # :64-67 (causal)
    if max_attn_len > 0:  # :68-81
        if min_full_attn_seq_len > 0:
            valid &= (dist <= max_attn_len) | (row_ids >= max_ids - min_full_attn_seq_len)
        else:
            valid &= dist <= max_attn_len
    if contextual_seq_len > 0:  # :82-85
        valid |= (row_ids == 0) & (col_ids < max_ids)
    return valid


# --------------------------------------------------------------------------------------
# attention (ops path): forward / backward / delta-q
# --------------------------------------------------------------------------------------


def _lens(seq_offsets: torch.Tensor) -> np.ndarray:
    return seq_offsets.detach().cpu().numpy().astype(np.int64)


def hstu_mha_fwd(
    max_seq_len: int,
    alpha: float,
    q: torch.Tensor,
    k: torch.Tensor,
    v: torch.Tensor,
    seq_offsets: torch.Tensor,
    num_targets: Optional[torch.Tensor] = None,
    max_attn_len: int = 0,
    contextual_seq_len: int = 0,
    min_full_attn_seq_len: int = 0,
    dtype: torch.dtype = torch.float32,
) -> torch.Tensor:
    """O = (silu(alpha*Q K^T)/N * mask) V per (sequence, head); N = max_seq_len.

    ops/pytorch/pt_hstu_attention.py:130-171 (pytorch_hstu_mha), evaluated one sequence at a
    time (exact: sequences are independent) in `dtype` on the given input values.
    Returns [L, H, dv] in `dtype`.
    """
    off = _lens(seq_offsets)
    L, H, _ = q.shape
    dv = v.shape[2]
    out = torch.zeros(L, H, dv, dtype=dtype)
    nt = None if num_targets is None else num_targets.detach().cpu().numpy()
    for b in range(len(off) - 1):
        s, e = int(off[b]), int(off[b + 1])
        n = min(e - s, max_seq_len)  # jagged_to_padded_dense truncates rows >= N
        if n <= 0:
            continue
        m = torch.from_numpy(
            attn_valid_mask(
                n, None if nt is None else int(nt[b]), max_attn_len, contextual_seq_len, min_full_attn_seq_len
            )
        )
        hc = max(1, min(H, (1 << 26) // max(1, n * n)))  # heads per chunk: bounds the [hc, n, n] temporaries
        for h0 in range(0, H, hc):
            qb = q[s : s + n, h0 : h0 + hc].to(dtype).transpose(0, 1)  # [hc, n, d]
            kb = k[s : s + n, h0 : h0 + hc].to(dtype).transpose(0, 1)
            vb = v[s : s + n, h0 : h0 + hc].to(dtype).transpose(0, 1)
            sc = torch.matmul(qb, kb.transpose(1, 2)) * alpha  # :150
            p = torch.nn.functional.silu(sc) / max_seq_len  # :151
            p = p * m.to(dtype)  # :163
            out[s : s + n, h0 : h0 + hc] = torch.matmul(p, vb).transpose(0, 1)  # :166
    return out


def hstu_mha_bwd(
    max_seq_len: int,
    alpha: float,
    dout: torch.Tensor,
    q: torch.Tensor,
    k: torch.Tensor,
    v: torch.Tensor,
    seq_offsets: torch.Tensor,
    num_targets: Optional[torch.Tensor] = None,
    max_attn_len: int = 0,
    contextual_seq_len: int = 0,
    min_full_attn_seq_len: int = 0,
    dtype: torch.dtype = torch.float32,
) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """Explicit gradient of hstu_mha_fwd (what autograd derives from pt_hstu_attention.py:150-166;
    the same math the reference's own kernels implement, ops/triton/triton_hstu_attention.py:995-1006,1222):

        S = alpha Q K^T, sig = sigmoid(S), c = 1/N
        dV = P^T dO,  dP = dO V^T,  dS = c dP sig (1 + S (1 - sig)) mask
        dQ = alpha dS K,  dK = alpha dS^T Q
    """
    off = _lens(seq_offsets)
    dq = torch.zeros(q.shape, dtype=dtype)
    dk = torch.zeros(k.shape, dtype=dtype)
    dv_ = torch.zeros(v.shape, dtype=dtype)
    nt = None if num_targets is None else num_targets.detach().cpu().numpy()
    c = 1.0 / max_seq_len
    for b in range(len(off) - 1):
        s, e = int(off[b]), int(off[b + 1])
        n = min(e - s, max_seq_len)
        if n <= 0:
            continue
        m = torch.from_numpy(
            attn_valid_mask(
                n, None if nt is None else int(nt[b]), max_attn_len, contextual_seq_len, min_full_attn_seq_len
            )
        ).to(dtype)
        H = q.shape[1]
        hc = max(1, min(H, (1 << 26) // max(1, n * n)))
        for h0 in range(0, H, hc):
            qb = q[s : s + n, h0 : h0 + hc].to(dtype).transpose(0, 1)
            kb = k[s : s + n, h0 : h0 + hc].to(dtype).transpose(0, 1)
            vb = v[s : s + n, h0 : h0 + hc].to(dtype).transpose(0, 1)
            dob = dout[s : s + n, h0 : h0 + hc].to(dtype).transpose(0, 1)
            S = torch.matmul(qb, kb.transpose(1, 2)) * alpha
            sig = torch.sigmoid(S)
            P = c * S * sig * m
            dv_[s : s + n, h0 : h0 + hc] = torch.matmul(P.transpose(1, 2), dob).transpose(0, 1)
            dP = torch.matmul(dob, vb.transpose(1, 2))
            dS = c * dP * sig * (1.0 + S * (1.0 - sig)) * m
            dq[s : s + n, h0 : h0 + hc] = (alpha * torch.matmul(dS, kb)).transpose(0, 1)
            dk[s : s + n, h0 : h0 + hc] = (alpha * torch.matmul(dS.transpose(1, 2), qb)).transpose(0, 1)
    return dq, dk, dv_


def delta_hstu_mha_fwd(
    max_seq_len: int,
    alpha: float,
    delta_q: torch.Tensor,
    k: torch.Tensor,
    v: torch.Tensor,
    seq_offsets: torch.Tensor,
    num_targets: Optional[torch.Tensor] = None,
    max_attn_len: int = 0,
    contextual_seq_len: int = 0,
    dtype: torch.dtype = torch.float32,
) -> torch.Tensor:
    """Cached / delta-q attention: the last `delta_size` query rows of every sequence against
    the full K/V.  ops/pytorch/pt_hstu_attention.py:175-235 (pytorch_cached_hstu_mha)."""
    off = _lens(seq_offsets)
    B = len(off) - 1
    Lq, H, _ = delta_q.shape
    delta = Lq // B
    dv = v.shape[2]
    out = torch.zeros(Lq, H, dv, dtype=dtype)
    nt = None if num_targets is None else num_targets.detach().cpu().numpy()
    for b in range(B):
        s, e = int(off[b]), int(off[b + 1])
        n = e - s
        rows = np.arange(n - delta, n, dtype=np.int64)  # :218-222
        m = torch.from_numpy(
            attn_valid_mask(n, None if nt is None else int(nt[b]), max_attn_len, contextual_seq_len, 0, rows=rows)
        ).to(dtype)
        qb = delta_q[b * delta : (b + 1) * delta].to(dtype).transpose(0, 1)
        kb = k[s:e].to(dtype).transpose(0, 1)
        vb = v[s:e].to(dtype).transpose(0, 1)
        sc = torch.matmul(qb, kb.transpose(1, 2)) * alpha
        p = torch.nn.functional.silu(sc) / max_seq_len * m
        out[b * delta : (b + 1) * delta] = torch.matmul(p, vb).transpose(0, 1)
    return out


# --------------------------------------------------------------------------------------
# attention (research path): relative position + time-bucket bias, plain causal mask
# --------------------------------------------------------------------------------------


def rel_bias(
    n: int, pos_w: torch.Tensor, ts_w: Optional[torch.Tensor], timestamps: Optional[torch.Tensor]
) -> torch.Tensor:
    """[n, n] (no timestamps) or [B, n, n] bias.

    research/modeling/sequential/hstu.py:66-144: rel_pos_bias[i,j] = pos_w[n-1+j-i];
    rel_ts_bias[i,j] = ts_w[clamp(floor(log(max(|ts[i+1]-ts[j]|,1))/0.301),0,num_buckets)]
    with ts[n] := ts[n-1]  (`ext_timestamps`, :129-133).
    """
    i = torch.arange(n).view(n, 1)
    j = torch.arange(n).view(1, n)
    bias = pos_w[(n - 1 + j - i)]
    if ts_w is None or timestamps is None:
        return bias
    ts = timestamps.to(torch.int64)
    ext = torch.cat([ts, ts[:, n - 1 : n]], dim=1)  # [B, n+1]
    d = ext[:, 1:].unsqueeze(2) - ext[:, :-1].unsqueeze(1)  # [B, n(i), n(j)] = ts[i+1]-ts[j]
    nb = ts_w.numel() - 1
    bucket = torch.clamp(
        (torch.log(torch.abs(d).clamp(min=1).to(torch.float32)) / 0.301).long(), min=0, max=nb
    )
    return bias.unsqueeze(0) + ts_w[bucket]


def hstu_rel_bias_attention_fwd(
    n: int,
    q: torch.Tensor,
    k: torch.Tensor,
    v: torch.Tensor,
    seq_offsets: torch.Tensor,
    pos_w: torch.Tensor,
    ts_w: Optional[torch.Tensor] = None,
    timestamps: Optional[torch.Tensor] = None,
    dtype: torch.dtype = torch.float32,
) -> torch.Tensor:
    """O = (silu(Q K^T + bias)/n * tril) V.  research/modeling/sequential/hstu.py:150-223
    (_hstu_attention_maybe_from_cache, no cache): q,k [L,H,dqk], v [L,H,dv]."""
    off = _lens(seq_offsets)
    L, H, _ = q.shape
    out = torch.zeros(L, H, v.shape[2], dtype=dtype)
    bias = rel_bias(n, pos_w.to(dtype), None if ts_w is None else ts_w.to(dtype), timestamps)
    for b in range(len(off) - 1):
        s, e = int(off[b]), int(off[b + 1])
        m = min(e - s, n)
        if m <= 0:
            continue
        bb = bias if bias.dim() == 2 else bias[b]
        qb = q[s : s + m].to(dtype).transpose(0, 1)
        kb = k[s : s + m].to(dtype).transpose(0, 1)
        vb = v[s : s + m].to(dtype).transpose(0, 1)
        sc = torch.matmul(qb, kb.transpose(1, 2)) + bb[:m, :m].unsqueeze(0)  # :204-210
        p = torch.nn.functional.silu(sc) / n  # :211
        p = p * torch.tril(torch.ones(m, m, dtype=dtype))  # :212 (invalid_attn_mask = tril)
        out[s : s + m] = torch.matmul(p, vb).transpose(0, 1)
    return out


# --------------------------------------------------------------------------------------
# layer norms (ops/pytorch/pt_layer_norm.py) and the output stage (pt_hstu_linear.py)
# --------------------------------------------------------------------------------------


def layer_norm_fwd(x, weight, bias, eps, dtype=torch.float32):
    """pt_layer_norm.py:24-38: LN over the last dim computed in fp32."""
    xf = x.to(dtype)
    mean = xf.mean(-1, keepdim=True)
    var = ((xf - mean) ** 2).mean(-1, keepdim=True)
    rstd = torch.rsqrt(var + eps)
    y = (xf - mean) * rstd
    if weight is not None:
        y = y * weight.to(dtype)
    if bias is not None:
        y = y + bias.to(dtype)
    return y, mean.squeeze(-1), rstd.squeeze(-1)


def layer_norm_bwd(dy, x, weight, mean, rstd, dtype=torch.float32):
    """Gradient of layer_norm_fwd: dx, dw, db (what autograd derives from pt_layer_norm.py:31-38;
    same math as ops/triton/triton_layer_norm.py:129-309)."""
    xf, dyf = x.to(dtype), dy.to(dtype)
    xhat = (xf - mean.unsqueeze(-1)) * rstd.unsqueeze(-1)
    wdy = dyf * (weight.to(dtype) if weight is not None else 1.0)
    D = x.shape[-1]
    c1 = (xhat * wdy).sum(-1, keepdim=True) / D
    c2 = wdy.sum(-1, keepdim=True) / D
    dx = (wdy - (xhat * c1 + c2)) * rstd.unsqueeze(-1)
    dw = (dyf * xhat).sum(0)
    db = dyf.sum(0)
    return dx, dw, db


def swish_layer_norm_fwd(x, weight, bias, eps, dtype=torch.float32):
    """pt_layer_norm.py:41-61: x * sigmoid(LN(x))."""
    y, _, _ = layer_norm_fwd(x, weight, bias, eps, dtype)
    return x.to(dtype) * torch.sigmoid(y)


def rms_norm_fwd(x, weight, eps, dtype=torch.float32):
    """ops/layer_norm.py:150-158 (RMSNorm eager branch)."""
    xf = x.to(dtype)
    return xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps) * weight.to(dtype)


def norm_mul_dropout_fwd(
    x, u, weight, bias, eps, silu_u=False, concat_ux=False, group_norm=False, num_heads=1, linear_dim=-1,
    dtype=torch.float32,
):
    """pt_hstu_linear.py:23-66 with dropout_ratio = 0 (the only setting the reference tests compare)."""
    uf = u.to(dtype)
    if silu_u:
        uf = torch.nn.functional.silu(uf)
    xf = x.to(dtype)
    if group_norm:  # :42-49 per-head normalisation with scalar affine per head
        xh = xf.view(-1, num_heads, linear_dim)
        mean = xh.mean(-1, keepdim=True)
        var = ((xh - mean) ** 2).mean(-1, keepdim=True)
        nh = (xh - mean) * torch.rsqrt(var + eps)
        nh = nh * weight.to(dtype).view(1, num_heads, 1) + bias.to(dtype).view(1, num_heads, 1)
        y = uf * nh.reshape(-1, num_heads * linear_dim)
    else:
        y = uf * layer_norm_fwd(xf, weight, bias, eps, dtype)[0]
    if concat_ux:  # :57-58
        y = torch.cat([uf, xf, y], dim=1)
    return y


def hstu_compute_output_fwd(
    attn, u, x, norm_weight, norm_bias, output_weight, eps, silu_u=False, concat_ux=False, group_norm=False,
    num_heads=1, linear_dim=-1, dtype=torch.float32,
):
    """pt_hstu_linear.py:68-99: out = x + y W_o."""
    y = norm_mul_dropout_fwd(attn, u, norm_weight, norm_bias, eps, silu_u, concat_ux, group_norm, num_heads,
                             linear_dim, dtype)
    return x.to(dtype) + y @ output_weight.to(dtype)


def hstu_compute_uqvk_fwd(x, norm_weight, norm_bias, norm_eps, num_heads, attn_dim, hidden_dim, uvqk_weight,
                          uvqk_bias, dtype=torch.float32):
    """ops/hstu_compute.py:50-89: LN -> addmm -> split [u|v|q|k] -> silu(u)."""
    nx = layer_norm_fwd(x, norm_weight, norm_bias, norm_eps, dtype)[0]
    uvqk = uvqk_bias.to(dtype) + nx @ uvqk_weight.to(dtype)
    u, v, q, k = torch.split(
        uvqk, [hidden_dim * num_heads, hidden_dim * num_heads, attn_dim * num_heads, attn_dim * num_heads], dim=1
    )
    u = torch.nn.functional.silu(u)
    return (u, q.reshape(-1, num_heads, attn_dim), k.reshape(-1, num_heads, attn_dim),
            v.reshape(-1, num_heads, hidden_dim))


def stu_layer_fwd(
    x, x_offsets, max_seq_len, num_targets, params: dict, num_heads, attn_dim, hidden_dim, max_attn_len=0,
    contextual_seq_len=0, attn_alpha=None, use_group_norm=False, target_aware=True, dtype=torch.float32,
):
    """modules/stu.py:291-352 (STULayer.forward, training path without KV cache), dropout 0.
    `params` uses the reference parameter names (stu.py:206-245)."""
    alpha = attn_alpha if attn_alpha is not None else 1.0 / math.sqrt(attn_dim)
    u, q, k, v = hstu_compute_uqvk_fwd(
        x, params["_input_norm_weight"], params["_input_norm_bias"], 1e-6, num_heads, attn_dim, hidden_dim,
        params["_uvqk_weight"], params["_uvqk_beta"], dtype,
    )
    attn = hstu_mha_fwd(max_seq_len, alpha, q, k, v, x_offsets, num_targets if target_aware else None,
                        max_attn_len, contextual_seq_len, 0, dtype).reshape(-1, num_heads * hidden_dim)
    return hstu_compute_output_fwd(
        attn, u, x, params["_output_norm_weight"], params["_output_norm_bias"], params["_output_weight"], 1e-6,
        False, True, use_group_norm, num_heads, hidden_dim, dtype,
    )


# --------------------------------------------------------------------------------------
# timestamp + position embedding add  -- ops/position.py:43-96, ops/pytorch/pt_position.py:39-134
# --------------------------------------------------------------------------------------


def position_indices(seq_offsets, seq_lengths, timestamps, num_targets, max_contextual_seq_len, max_pos_ind,
                     num_time_buckets, interleave_targets, time_bucket_fn):
    """Integer part of the op, per jagged row: (pos_ind [L] int64, ts_bucket [L] int64).

    pos_ind: pt_position.py:39-72 (_get_col_indices) for the real positions of each sequence.
    ts_bucket: pt_position.py:97-123 -- query time = timestamp of row len-1 (index clamped to >= 0 of the zero-padded row),
    dt -> float32 (torch promotes the int64 clamp(min=1e-6) to float32), /60, log|sqrt, clamp(min=0).int(), clamp to
    [0, num_time_buckets]."""
    off = _lens(seq_offsets)
    lens = seq_lengths.detach().cpu().numpy().astype(np.int64)
    ts = timestamps.detach().cpu().numpy().astype(np.int64)
    nt = None if num_targets is None else num_targets.detach().cpu().numpy().astype(np.int64)
    L = int(off[-1])
    pos = np.zeros(L, dtype=np.int64)
    bkt = np.zeros(L, dtype=np.int64)
    for b in range(len(off) - 1):
        s, e = int(off[b]), int(off[b + 1])
        if e <= s:
            continue
        n = np.arange(e - s, dtype=np.int64)
        ln = int(lens[b])
        if nt is not None:
            high = ln - int(nt[b]) * (2 if interleave_targets else 1)
            c = high - np.minimum(n, high)
        else:
            c = ln - n
        c = np.minimum(c + max_contextual_seq_len, max_pos_ind - 1)
        c = np.where(n < max_contextual_seq_len, n, c)
        pos[s:e] = c
        qi = max(ln - 1, 0)
        qt = ts[s + qi] if s + qi < e else 0
        dt = (qt - ts[s:e]).astype(np.float32)
        x = np.maximum(dt, np.float32(1e-6)) / np.float32(60.0)
        x = np.log(x) if time_bucket_fn == "log" else np.sqrt(x)
        x = np.maximum(x.astype(np.float32), np.float32(0.0))
        bkt[s:e] = np.clip(x.astype(np.int32), 0, num_time_buckets)
    return torch.from_numpy(pos), torch.from_numpy(bkt)


def add_timestamp_positional_embeddings(alpha, max_contextual_seq_len, pos_w, ts_w, seq_offsets, seq_lengths, seq_embeddings,
                                        timestamps, num_targets, interleave_targets, time_bucket_fn, dout=None):
    """out = (seq * alpha) + (pos_w[pos] + ts_w[bucket]).to(dtype) with the reference's roundings (position.py:58,
    pt_position.py:124-133); with `dout`: also (d_seq, d_pos_w, d_ts_w) = (dout * alpha, scatter-adds of dout in fp32)."""
    dt = seq_embeddings.dtype
    pos, bkt = position_indices(seq_offsets, seq_lengths, timestamps, num_targets, max_contextual_seq_len, pos_w.shape[0],
                                ts_w.shape[1] - 1, interleave_targets, time_bucket_fn)
    emb = (ts_w.float()[bkt] + pos_w.float()[pos]).to(dt)
    out = (seq_embeddings * alpha) + emb
    if dout is None:
        return out
    g = dout.float()
    dpos = torch.zeros(pos_w.shape, dtype=torch.float32).index_add_(0, pos, g)
    dts = torch.zeros(ts_w.shape, dtype=torch.float32).index_add_(0, bkt, g)
    return out, (dout * alpha), dpos, dts


# --------------------------------------------------------------------------------------
# jagged x dense bmm + broadcast bias -- ops/jagged_tensors.py:210-253, ops/pytorch/pt_jagged.py:77-98
# --------------------------------------------------------------------------------------


def jagged_dense_bmm_broadcast_add(max_seq_len, seq_offsets, jagged, dense, bias):
    """out[rows of b] = jagged[rows of b] @ dense[b] + bias[b], operands promoted to fp32 and the result cast back to the dtype
    of `jagged` (pt_jagged.py:84-97); one sequence at a time (exact: sequences are independent).  Differentiable (autograd)."""
    off = _lens(seq_offsets)
    outs = []
    for b in range(len(off) - 1):
        s, e = int(off[b]), int(off[b + 1])
        rows = jagged[s:e].to(torch.float32)
        outs.append(rows @ dense[b].to(torch.float32) + bias[b].to(torch.float32).unsqueeze(0))
    out = torch.cat(outs, dim=0) if outs else jagged.new_zeros((0, dense.shape[2]), dtype=torch.float32)
    return out.to(jagged.dtype)


# --------------------------------------------------------------------------------------
# sampled-softmax loss -- research/modeling/sequential/losses/sampled_softmax.py:43-89 (dot-product similarity,
# LocalNegativesSampler: autoregressive_losses.py:29-121)
# --------------------------------------------------------------------------------------


def sampled_softmax_loss(q, pos_ids, pos_emb, weights, neg_ids, table, temperature, l2_norm, l2_eps, dtype=torch.float32):
    """Differentiable (torch autograd) restatement in `dtype`: returns the scalar loss."""
    def norm(x):  # autoregressive_losses.py:39-45
        if l2_norm:
            x = x / torch.clamp(torch.linalg.norm(x, ord=2, dim=-1, keepdim=True), min=l2_eps)
        return x

    qf = q.to(dtype)
    pe = norm(pos_emb.to(dtype))
    ne = norm(table.to(dtype)[neg_ids])                                  # [N, R, D]
    pos_logits = (qf * pe).sum(-1, keepdim=True) / temperature           # dot_product_similarity_fn.py:62-67 with X = 1
    neg_logits = torch.bmm(ne, qf.unsqueeze(2)).squeeze(2) / temperature
    neg_logits = torch.where(pos_ids.unsqueeze(1) == neg_ids, torch.full_like(neg_logits, -5e4), neg_logits)  # :80-84
    rows = -torch.nn.functional.log_softmax(torch.cat([pos_logits, neg_logits], dim=1), dim=1)[:, 0]
    w = weights.to(dtype)
    return (rows * w).sum() / w.sum()


# --------------------------------------------------------------------------------------
# jagged row routing (integer-exact)  -- ops/pytorch/pt_jagged_tensors.py
# --------------------------------------------------------------------------------------


def _dense_offsets(n_batches: int, max_len: int) -> np.ndarray:
    return max_len * np.arange(n_batches + 1, dtype=np.int64)


def concat_2D_jagged_index(
    offsets_left: Optional[Sequence[int]], offsets_right: Optional[Sequence[int]], total_left: int,
    total_right: int, max_len_left: Optional[int], max_len_right: Optional[int], n_prefix_from_right: int = 0,
) -> np.ndarray:
    """Row routing of concat_2D_jagged: returns src[int64, L_out] where src >= 0 indexes values_left
    and src < 0 encodes row (-src-1) of values_right.  pt_jagged_tensors.py:31-122; with
    n_prefix_from_right = contextual_seq_len it is hstu_concat_l2_embeddings (:201-246):
    out_b = [right_b[:n_prefix] | left_b | right_b[n_prefix:]].  A `None` offsets means the side is dense
    with `max_len` rows per batch entry (:86-101)."""
    if offsets_left is None:
        B = total_left // max_len_left
        ol = _dense_offsets(B, max_len_left)
    else:
        ol = np.asarray(offsets_left, dtype=np.int64)
    if offsets_right is None:
        B = total_right // max_len_right
        orr = _dense_offsets(B, max_len_right)
    else:
        orr = np.asarray(offsets_right, dtype=np.int64)
    out: List[int] = []
    for b in range(len(ol) - 1):
        l0, l1, r0, r1 = int(ol[b]), int(ol[b + 1]), int(orr[b]), int(orr[b + 1])
        npre = min(n_prefix_from_right, r1 - r0)
        out += [-(r + 1) for r in range(r0, r0 + npre)]
        out += list(range(l0, l1))
        out += [-(r + 1) for r in range(r0 + npre, r1)]
    return np.asarray(out, dtype=np.int64)


def concat_2D_jagged(values_left, values_right, max_len_left=None, max_len_right=None, offsets_left=None,
                     offsets_right=None, n_prefix_from_right: int = 0) -> torch.Tensor:
    src = concat_2D_jagged_index(
        None if offsets_left is None else offsets_left.tolist(),
        None if offsets_right is None else offsets_right.tolist(),
        values_left.shape[0], values_right.shape[0], max_len_left, max_len_right, n_prefix_from_right,
    )
    out = torch.empty(len(src), values_left.shape[1], dtype=values_left.dtype)
    isl = torch.from_numpy(src >= 0)
    out[isl] = values_left[torch.from_numpy(src[src >= 0])]
    out[~isl] = values_right[torch.from_numpy(-src[src < 0] - 1)]
    return out


def split_2D_jagged(values, max_len_left=None, max_len_right=None, offsets_left=None, offsets_right=None,
                    n_prefix_to_right: int = 0) -> Tuple[torch.Tensor, torch.Tensor]:
    """Inverse of concat_2D_jagged.  pt_jagged_tensors.py:125-198 (n_prefix_to_right = 0) and
    pytorch_hstu_split_l2_embeddings (:169-198, n_prefix_to_right = contextual_seq_len)."""
    if offsets_left is None:
        nb = len(offsets_right) - 1
        ol = _dense_offsets(nb, max_len_left)
    else:
        ol = offsets_left.numpy().astype(np.int64)
    if offsets_right is None:
        nb = len(ol) - 1
        orr = _dense_offsets(nb, max_len_right)
    else:
        orr = offsets_right.numpy().astype(np.int64)
    src = concat_2D_jagged_index(ol, orr, int(ol[-1]), int(orr[-1]), None, None, n_prefix_to_right)
    left = torch.empty(int(ol[-1]), values.shape[1], dtype=values.dtype)
    right = torch.empty(int(orr[-1]), values.shape[1], dtype=values.dtype)
    isl = torch.from_numpy(src >= 0)
    left[torch.from_numpy(src[src >= 0])] = values[isl]
    right[torch.from_numpy(-src[src < 0] - 1)] = values[~isl]
    return left, right


# --------------------------------------------------------------------------------------
# autograd wrapper over the explicit forward / backward (used by the CPU-baseline timing: bounded memory)
# --------------------------------------------------------------------------------------


class OracleAttention(torch.autograd.Function):
    """hstu_mha_fwd / hstu_mha_bwd under autograd, so that a whole layer can be differentiated on CPU without
    autograd retaining the [H, n, n] temporaries of every op."""

    @staticmethod
    def forward(ctx, max_seq_len, alpha, q, k, v, seq_offsets, num_targets, max_attn_len, contextual_seq_len):
        ctx.save_for_backward(q, k, v, seq_offsets, num_targets)
        ctx.cfg = (max_seq_len, alpha, max_attn_len, contextual_seq_len)
        return hstu_mha_fwd(max_seq_len, alpha, q, k, v, seq_offsets, num_targets, max_attn_len, contextual_seq_len)

    @staticmethod
    def backward(ctx, dout):
        q, k, v, seq_offsets, num_targets = ctx.saved_tensors
        n, alpha, mal, ctxlen = ctx.cfg
        dq, dk, dv = hstu_mha_bwd(n, alpha, dout, q, k, v, seq_offsets, num_targets, mal, ctxlen)
        return None, None, dq, dk, dv, None, None, None, None


def stu_layer_fwd_bwd_timed(x, x_offsets, max_seq_len, num_targets, params, num_heads, attn_dim, hidden_dim):
    """One STU layer forward + backward on CPU (fp32), attention through OracleAttention.  Returns (y, dx)."""
    x = x.detach().float().requires_grad_()
    ps = {k: v.detach().float().requires_grad_() for k, v in params.items()}
    alpha = 1.0 / math.sqrt(attn_dim)
    u, q, k, v = hstu_compute_uqvk_fwd(x, ps["_input_norm_weight"], ps["_input_norm_bias"], 1e-6, num_heads, attn_dim,
                                       hidden_dim, ps["_uvqk_weight"], ps["_uvqk_beta"])
    attn = OracleAttention.apply(max_seq_len, alpha, q, k, v, x_offsets, num_targets, 0, 0)
    y = hstu_compute_output_fwd(attn.reshape(-1, num_heads * hidden_dim), u, x, ps["_output_norm_weight"],
                                ps["_output_norm_bias"], ps["_output_weight"], 1e-6, False, True, False, num_heads,
                                hidden_dim)
    y.backward(torch.ones_like(y))
    return y.detach(), x.grad


def stu_stack_fwd_bwd(x, x_offsets, max_seq_len, num_targets, layer_params, num_heads, attn_dim, hidden_dim, dout):
    """A whole STU stack (modules/stu.py:421-466: layers applied in sequence; each layer = stu.py:291-352, dropout 0,
    LayerNorm output norm, concat_ux) forward + backward in fp32 on CPU with the attention through OracleAttention.
    `layer_params`: one dict of reference parameter names per layer.  Returns (y, dx, [dict of parameter grads per layer])."""
    h = x.detach().float().requires_grad_()
    x_leaf = h
    alpha = 1.0 / math.sqrt(attn_dim)
    leaves = []
    for params in layer_params:
        ps = {k: v.detach().float().requires_grad_() for k, v in params.items()}
        leaves.append(ps)
        u, q, k, v = hstu_compute_uqvk_fwd(h, ps["_input_norm_weight"], ps["_input_norm_bias"], 1e-6, num_heads, attn_dim,
                                           hidden_dim, ps["_uvqk_weight"], ps["_uvqk_beta"])
        attn = OracleAttention.apply(max_seq_len, alpha, q, k, v, x_offsets, num_targets, 0, 0)
        h = hstu_compute_output_fwd(attn.reshape(-1, num_heads * hidden_dim), u, h, ps["_output_norm_weight"],
                                    ps["_output_norm_bias"], ps["_output_weight"], 1e-6, False, True, False, num_heads,
                                    hidden_dim)
    h.backward(dout.float())
    return h.detach(), x_leaf.grad, [{k: v.grad for k, v in ps.items()} for ps in leaves]


# --------------------------------------------------------------------------------------
# error metric shared by the parity tests
# --------------------------------------------------------------------------------------


def rel_l2(a: torch.Tensor, ref: torch.Tensor) -> float:
    a64, r64 = a.detach().double().cpu(), ref.detach().double().cpu()
    den = float(r64.norm())
    return float((a64 - r64).norm()) / (den if den > 0 else 1.0)


def storage_quantisation(ref: torch.Tensor, dtype: torch.dtype) -> float:
    """rel-L2 error of merely storing `ref` in `dtype` (0 for fp32)."""
    if dtype == torch.float32:
        return 0.0
    return rel_l2(ref.to(dtype).to(torch.float32), ref)


def research_block_fwd(
    x: torch.Tensor,
    seq_offsets: torch.Tensor,
    timestamps: Optional[torch.Tensor],
    uvqk: torch.Tensor,
    o_weight: torch.Tensor,
    o_bias: torch.Tensor,
    pos_w: torch.Tensor,
    ts_w: Optional[torch.Tensor],
    n: int,
    num_heads: int,
    attention_dim: int,
    linear_dim: int,
    concat_ua: bool = False,
    eps: float = 1e-6,
) -> torch.Tensor:
    """SequentialTransductionUnitJagged.forward, "rel_bias" normalisation, silu activation, no cache, dropout 0
    (research/modeling/sequential/hstu.py:318-436): LN without affine (:276-277) -> mm (no bias) -> SiLU on ALL of uvqk
    (:322-323) -> split u|v|q|k (:326-335) -> rel-bias attention (:343-357) -> u * LN(attn) or cat[u, a, u*a] with
    a = LN(attn) (:418-422) -> Linear(+bias) + x (:424-433).  Differentiable (torch ops only)."""
    H, dqk, dv = num_heads, attention_dim, linear_dim
    dt = x.dtype
    normed = torch.nn.functional.layer_norm(x, [x.shape[1]], eps=eps)
    mm = torch.nn.functional.silu(torch.mm(normed, uvqk))
    u, v, q, k = torch.split(mm, [dv * H, dv * H, dqk * H, dqk * H], dim=1)
    L = x.shape[0]
    attn = hstu_rel_bias_attention_fwd(n, q.reshape(L, H, dqk), k.reshape(L, H, dqk), v.reshape(L, H, dv), seq_offsets,
                                       pos_w, ts_w, timestamps, dtype=dt).reshape(L, H * dv)
    a = torch.nn.functional.layer_norm(attn, [H * dv], eps=eps)
    o_in = torch.cat([u, a, u * a], dim=-1) if concat_ua else u * a
    return torch.nn.functional.linear(o_in, o_weight, o_bias) + x
