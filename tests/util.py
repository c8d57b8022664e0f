"""Shared helpers of the parity tests."""
import math

import torch

from oracle import hstu_oracle as O

# north-star tolerance: activations / grads within 1e-3 relative (L2) of the reference evaluated in fp32 on the same
# input values.  Outputs stored in bf16/fp16 additionally carry the unavoidable storage rounding of that dtype
# (measured on the reference tensor itself, ~1.7e-3 for bf16); the two are combined in quadrature and NOTHING else is
# granted: the tensor-core kernels keep their P / dS operands in fp16 (11-bit significand) precisely so that no operand
# rounding term is needed here.  fp32: 1e-3 flat would be far too loose for an fp32 kernel, so fp32 paths are held to 2e-5.
TOL = {torch.float32: 2e-5, torch.bfloat16: 1e-3, torch.float16: 1e-3}


def assert_rel(actual: torch.Tensor, ref32: torch.Tensor, what: str, tol: float = None) -> float:
    """rel-L2(actual, ref32) <= sqrt(tol^2 + q^2), q = storage rounding of actual.dtype measured on ref32."""
    dt = actual.dtype
    t = TOL[dt] if tol is None else tol
    q = O.storage_quantisation(ref32.float().cpu(), dt)
    err = O.rel_l2(actual.float().cpu(), ref32.float().cpu())
    lim = math.sqrt(t * t + q * q)
    assert err <= lim, f"{what}: rel-L2 error {err:.3e} > {lim:.3e} (tol {t:.1e}, storage rounding {q:.2e})"
    return err


SEG_ROWS = 64        # rows of one segment: the query / key tile of the wgmma kernels
SEG_MIN_ELEMS = 2048  # smaller segments are merged: below this, bf16 output rounding alone breaks a 6e-4 kernel error's bound


def assert_rel_segments(actual: torch.Tensor, ref: torch.Tensor, seq_offsets, max_seq_len: int, what: str,
                        tol: float = None) -> float:
    """The bound of assert_rel on every segment of a jagged [L, H, d] tensor instead of on the whole of it, so that an error
    confined to one tile of one sequence cannot hide in the rest.  A segment is one (sequence, head, 64-row block); a block
    of fewer than SEG_MIN_ELEMS elements joins the previous block of its (sequence, head), and the (sequence, head) slices
    still below that are pooled per head (a pool that stays below it is left to the whole-tensor bound).  Each segment meets
    sqrt(tol^2 + q^2), q the storage rounding measured on that segment; nothing else is granted.  Rows at positions
    >= max_seq_len must be exactly zero.  The failure names the worst segment.  Returns the largest per-segment rel-L2."""
    dt = actual.dtype
    t = TOL[dt] if tol is None else tol
    off = [int(x) for x in torch.as_tensor(seq_offsets).cpu().tolist()]
    L, H = actual.shape[0], actual.shape[1]
    a = actual.detach().float().cpu().reshape(L, H, -1).double()
    r = ref.detach().float().cpu().reshape(L, H, -1).double()
    d = a.shape[2]
    # per (row, head) sums of squares: error, reference, storage rounding of the reference
    e2 = (a - r).square().sum(-1)
    r2 = r.square().sum(-1)
    q2 = (r.float().to(dt).double() - r).square().sum(-1)

    segs = []  # (err, lim, label)

    def check(rows, h, label):
        den = float(r2[rows, h].sum())
        den = den if den > 0 else 1.0
        err = math.sqrt(float(e2[rows, h].sum()) / den)
        q = math.sqrt(float(q2[rows, h].sum()) / den)
        segs.append((err, math.sqrt(t * t + q * q), q, label))

    pooled = {h: [] for h in range(H)}  # head -> [(sequence, rows)] of the short (sequence, head) slices
    for b in range(len(off) - 1):
        s, e = off[b], off[b + 1]
        n = min(e - s, max_seq_len)
        if e - s > n:
            bad = (a[s + n:e] != 0).reshape(e - s - n, -1).any(-1).nonzero()
            assert bad.numel() == 0, f"{what}: sequence {b} row {n + int(bad[0])} (>= max_seq_len {max_seq_len}) is not zero"
        if n <= 0:
            continue
        if n * d < SEG_MIN_ELEMS:
            for h in range(H):
                pooled[h].append((b, torch.arange(s, s + n)))
            continue
        bounds = [0]
        for p in range(SEG_ROWS, n, SEG_ROWS):
            if (p - bounds[-1]) * d >= SEG_MIN_ELEMS:
                bounds.append(p)
        if (n - bounds[-1]) * d < SEG_MIN_ELEMS:
            bounds.pop()  # the short last block joins the previous one
        bounds.append(n)
        for h in range(H):
            for p0, p1 in zip(bounds[:-1], bounds[1:]):
                check(slice(s + p0, s + p1), h, f"sequence {b} head {h} rows [{p0}, {p1})")
    for h, parts in pooled.items():
        rows = torch.cat([p[1] for p in parts]) if parts else torch.zeros(0, dtype=torch.int64)
        if rows.numel() * d >= SEG_MIN_ELEMS:
            check(rows, h, f"sequences {[p[0] for p in parts]} head {h} (short sequences pooled)")
    over = [x for x in segs if not x[0] <= x[1]]  # NaN counts as over
    if over:
        err, lim, q, label = max(over, key=lambda x: x[0] / x[1] if x[0] == x[0] else math.inf)
        raise AssertionError(f"{what}: {label}: rel-L2 error {err:.3e} > {lim:.3e} (tol {t:.1e}, storage rounding "
                             f"{q:.2e}); {len(over)} of {len(segs)} segments over their bound")
    return max((x[0] for x in segs), default=0.0)


def assert_finite_rows(t: torch.Tensor, seq_offsets, skip, what: str) -> None:
    """Every row of every sequence not in `skip` is finite; the message names the first sequence and row that is not."""
    off = [int(x) for x in torch.as_tensor(seq_offsets).cpu().tolist()]
    x = t.detach().float().cpu().reshape(t.shape[0], -1)
    for b in range(len(off) - 1):
        if b in skip:
            continue
        bad = (~torch.isfinite(x[off[b]:off[b + 1]])).any(-1).nonzero()
        assert bad.numel() == 0, f"{what}: sequence {b} row {int(bad[0])} is not finite"


def offsets_from(lengths, device="cpu", dtype=torch.int64):
    off = torch.zeros(len(lengths) + 1, dtype=dtype, device=device)
    off[1:] = torch.cumsum(torch.as_tensor(lengths, dtype=dtype, device=device), 0)
    return off


def normal_case(lengths, targets, H, d, sigma, dtype, seed, i32=False):
    """q, k ~ N(0, sigma^2) and v, dout ~ N(0, 1) of a jagged batch, rounded to `dtype`.  With alpha = 1/sqrt(d) the logits
    alpha S have an rms of sigma^2, whatever d is.  Returns (q, k, v, dout, seq_offsets, num_targets)."""
    g = torch.Generator().manual_seed(seed)
    idt = torch.int32 if i32 else torch.int64
    off = offsets_from(lengths, dtype=idt)
    L = int(off[-1])
    q, k = ((sigma * torch.randn(L, H, d, generator=g)).to(dtype) for _ in range(2))
    v, dout = (torch.randn(L, H, d, generator=g).to(dtype) for _ in range(2))
    return q, k, v, dout, off, None if targets is None else torch.tensor(targets, dtype=idt)
