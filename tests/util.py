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


BLOCK_ROWS = 4224  # rows of one pass of the length-256 output-stage backward: 528 CTAs x 8 warps, one row per warp each


def rel_row_sums(actual: torch.Tensor, ref: torch.Tensor) -> torch.Tensor:
    """[n, 4] fp64 per-row sums of two [n, W] tensors: squared error, squared reference, squared storage rounding of the
    reference in actual.dtype, and the element count.  Sums of row chunks concatenate, so a check of a tensor too large for
    host memory can be assembled chunk by chunk."""
    a = actual.detach().cpu().double().reshape(actual.shape[0], -1)
    r = ref.detach().cpu().double().reshape(ref.shape[0], -1)
    q = torch.zeros_like(r) if actual.dtype == torch.float32 else r.to(actual.dtype).double() - r
    cnt = torch.full((r.shape[0],), float(r.shape[1]), dtype=torch.float64)
    return torch.stack([(a - r).square().sum(1), r.square().sum(1), q.square().sum(1), cnt], 1)


def assert_rel_row_sums(sums: torch.Tensor, dtype: torch.dtype, what: str, block: int = BLOCK_ROWS,
                        tol: float = None) -> float:
    """The bound of assert_rel, sqrt(tol^2 + q^2) with q the storage rounding of `dtype` measured on the reference, on the
    whole tensor and on every block of `block` rows, from the per-row sums of rel_row_sums.  So an error confined to one pass
    of a persistent kernel's grid cannot hide in the rest.  A last block of fewer than SEG_MIN_ELEMS elements joins the one
    before it.  The failure names the worst block.  Returns the largest rel-L2 of a block."""
    t = TOL[dtype] if tol is None else tol
    n = sums.shape[0]
    bounds = list(range(0, n, block)) + [n]
    if len(bounds) > 2 and float(sums[bounds[-2]:, 3].sum()) < SEG_MIN_ELEMS:
        bounds.pop(-2)
    segs = []
    for r0, r1 in [(0, n)] + list(zip(bounds[:-1], bounds[1:])):
        e2, r2, q2, _ = (float(x) for x in sums[r0:r1].sum(0))
        den = r2 if r2 > 0 else 1.0
        err, q = math.sqrt(e2 / den), math.sqrt(q2 / den)
        segs.append((err, math.sqrt(t * t + q * q), q, "all rows" if (r0, r1) == (0, n) else f"rows [{r0}, {r1})"))
    over = [x for x in segs if not x[0] <= x[1]]  # NaN counts as over
    if over:
        err, lim, q, label = max(over, key=lambda x: x[0] / x[1] if x[0] == x[0] else math.inf)
        raise AssertionError(f"{what}: {label}: rel-L2 error {err:.3e} > {lim:.3e} (tol {t:.1e}, storage rounding "
                             f"{q:.2e}); {len(over)} of {len(segs)} checks over their bound")
    return max(x[0] for x in segs[1:])


def assert_rel_blocks(actual: torch.Tensor, ref: torch.Tensor, what: str, block: int = BLOCK_ROWS, tol: float = None) -> float:
    """assert_rel on the whole of an [n, W] tensor and on every block of `block` rows (assert_rel_row_sums)."""
    return assert_rel_row_sums(rel_row_sums(actual, ref), actual.dtype, what, block, tol)


def assert_finite_rows(t: torch.Tensor, seq_offsets, skip, what: str) -> None:
    """Every row of every sequence not in `skip` is finite; the message names the first sequence and row that is not."""
    off = [int(x) for x in torch.as_tensor(seq_offsets).cpu().tolist()]
    x = t.detach().float().cpu().reshape(t.shape[0], -1)
    for b in range(len(off) - 1):
        if b in skip:
            continue
        bad = (~torch.isfinite(x[off[b]:off[b + 1]])).any(-1).nonzero()
        assert bad.numel() == 0, f"{what}: sequence {b} row {int(bad[0])} is not finite"


U32 = 2.0 ** -24  # unit roundoff of fp32

_BITS = {torch.float32: (23, -126), torch.bfloat16: (7, -126), torch.float16: (10, -14)}  # fraction bits, min normal exponent


def _ulp(r, dtype):
    """Spacing of `dtype` at the (fp64) values r, which are representable in dtype."""
    p, emin = _BITS[dtype]
    e = torch.floor(torch.log2(r.abs().clamp_min(2.0 ** emin))).clamp_min(emin)
    return torch.exp2(e - p)


def _assert_ulp(got, ref64, mag, dtype, what):
    """got within 1 ulp of dtype of the fp64 value rounded to dtype, plus the error of the fp32 evaluation itself: the kernel
    uses __expf (at most 2 + 1.173 |x| ulp) and __fdividef (2 ulp) and a few more roundings, so (10 + 1.2 |x|) fp32 ulp of the
    magnitude `mag` of the unrounded terms.  That second part is far below one bf16 / fp16 ulp except where the result
    cancels to nearly zero; in fp32 it is the whole bound."""
    r = ref64.to(dtype).double()
    x_abs = mag[1]
    lim = _ulp(r, dtype) + (10 + 1.2 * x_abs) * 2.0 ** -23 * mag[0]
    err = (got.double().cpu() - r).abs()
    bad = ~(err <= lim)
    assert not bad.any(), (f"{what}: {int(bad.sum())} elements beyond 1 ulp; first at {tuple(int(i) for i in bad.nonzero()[0])}: "
                           f"got {float(got.double().cpu()[bad][0]):.8e}, ref {float(ref64[bad][0]):.8e}")


def assert_zero_from(table: torch.Tensor, start: int, what: str) -> None:
    """table[start:] is exactly zero (e.g. the j > i diagonals of a causal position-bias gradient)."""
    bad = (table.detach().float().cpu()[start:] != 0).nonzero()
    assert bad.numel() == 0, f"{what}: entry {start + int(bad[0])} is {float(table[start + int(bad[0])]):.3e}, must be exactly 0"


def assert_table_entries(got: torch.Tensor, ref: torch.Tensor, lim: torch.Tensor, what: str) -> None:
    """Per entry of a gradient table that is a sum of many terms: |got - ref| <= lim, lim = c * sum|terms| of that entry
    (from the fp64 reference).  An entry no term feeds has lim = 0 and must be exactly zero.  The failure names the worst
    entry."""
    g, r, b = (t.detach().double().cpu().reshape(-1) for t in (got, ref, lim))
    err = (g - r).abs()
    over = ~(err <= b)  # NaN counts as over
    if over.any():
        ratio = torch.where(over, torch.where(b > 0, err / b.clamp_min(1e-300), torch.full_like(err, math.inf)), torch.zeros_like(err))
        k = int(torch.argmax(torch.nan_to_num(ratio, nan=math.inf)))
        raise AssertionError(f"{what}: entry {k}: |got - ref| = {float(err[k]):.3e} > {float(b[k]):.3e} (got {float(g[k]):.6e}, "
                             f"ref {float(r[k]):.6e}); {int(over.sum())} of {g.numel()} entries over their bound")


def rel_bias_reference(n, q, k, v, dout, seq_offsets, pos_w, ts_w=None, timestamps=None) -> dict:
    """The research-path relative-bias attention in fp64 on the given (already rounded) values: out and the gradients of q,
    k, v, pos_w, ts_w by torch autograd through O.hstu_rel_bias_attention_fwd, plus, per entry of each bias table, the sum of
    |dS| over the scores that feed it and the number of those scores (dS from the oracle's score formula; its per-entry sums
    are checked against the autograd table gradients)."""
    q64, k64, v64, pw = (t.detach().double().requires_grad_() for t in (q, k, v, pos_w))
    tw = None if ts_w is None else ts_w.detach().double().requires_grad_()
    out = O.hstu_rel_bias_attention_fwd(n, q64, k64, v64, seq_offsets, pw, tw, timestamps, dtype=torch.float64)
    out.backward(dout.double())
    res = dict(out=out.detach(), dq=q64.grad, dk=k64.grad, dv=v64.grad, dpos=pw.grad, dts=None if tw is None else tw.grad)
    bias = O.rel_bias(n, pw.detach(), None if tw is None else tw.detach(), timestamps)
    nb = 0 if tw is None else tw.numel() - 1
    # the oracle's own bucket of every (b, i, j): its time bias with ts_w = [0, 1, ..., nb] and no position bias
    bkt = None if tw is None else O.rel_bias(n, torch.zeros(2 * n - 1, dtype=torch.float64),
                                             torch.arange(nb + 1, dtype=torch.float64), timestamps).long()
    mass_pos = torch.zeros(2 * n - 1, dtype=torch.float64)
    cnt_pos = torch.zeros(2 * n - 1, dtype=torch.float64)
    sum_pos = torch.zeros(2 * n - 1, dtype=torch.float64)
    mass_ts, cnt_ts = torch.zeros(nb + 1, dtype=torch.float64), torch.zeros(nb + 1, dtype=torch.float64)
    off = [int(x) for x in torch.as_tensor(seq_offsets).tolist()]
    for b in range(len(off) - 1):
        s, m = off[b], min(off[b + 1] - off[b], n)
        if m <= 0:
            continue
        qb, kb, vb, db = (t[s:s + m].double().transpose(0, 1) for t in (q, k, v, dout))
        S = qb @ kb.transpose(1, 2) + (bias if bias.dim() == 2 else bias[b])[:m, :m]
        sg = torch.sigmoid(S)
        dS = (db @ vb.transpose(1, 2)) * sg * (1 + S * (1 - sg)) / n * torch.tril(torch.ones(m, m, dtype=torch.float64))
        i = torch.arange(m).view(m, 1)
        j = torch.arange(m).view(1, m)
        diag = (n - 1 + j - i).expand(m, m).reshape(-1)
        a = dS.abs().sum(0).reshape(-1)
        c = (dS != 0).sum(0).double().reshape(-1)
        mass_pos.index_add_(0, diag, a)
        cnt_pos.index_add_(0, diag, c)
        sum_pos.index_add_(0, diag, dS.sum(0).reshape(-1))
        if bkt is not None:
            bb = bkt[b][:m, :m].reshape(-1)
            mass_ts.index_add_(0, bb, a)
            cnt_ts.index_add_(0, bb, c)
    scale = float(res["dpos"].abs().max()) or 1.0
    assert float((sum_pos - res["dpos"]).abs().max()) <= 1e-9 * scale, "explicit dS disagrees with the autograd dpos_w"
    res.update(mass_pos=mass_pos, cnt_pos=cnt_pos, mass_ts=mass_ts if tw is not None else None, cnt_ts=cnt_ts)
    return res


def table_bound(mass: torch.Tensor, count: torch.Tensor, d: int) -> torch.Tensor:
    """Allowed |got - ref| of a bias-table entry accumulated in fp32 from `count` score gradients dS of total magnitude `mass`.
    Each dS is formed in fp32 from length-d dot products (q.k and dO.v) and a few elementwise ops: a relative error of about
    d u of the magnitudes involved.  The terms are then summed in fp32 in whatever order the shared- and global-memory atomics
    happen to take; with random signs that rounding error grows like sqrt(count) u (the probabilistic bound of Higham and Mary,
    SIAM J. Sci. Comput. 2019), not like the worst-case count u.  So lim = 4 u (d + sqrt(count)) * sum|dS|, a factor 4 of
    headroom on that model.  A mass moved by one diagonal or one bucket changes an entry by about sum|dS| / sqrt(count), far
    above this for every count below 10^12."""
    return 4 * U32 * (d + count.sqrt()) * mass


# the research benchmark's configurations (profiles/h100_bench_research.json) with B = 6
RESEARCH_CONFIGS = {
    "ml20m": dict(D=256, H=8, dqk=32, dv=32, n=211, lengths=[211, 210, 65, 64, 1, 137]),
    "amzn_books": dict(D=64, H=8, dqk=8, dv=8, n=61, lengths=[61, 60, 33, 1, 17, 45]),
}
RESEARCH_PARAMS = ("_uvqk", "_o.weight", "_o.bias", "_rel_attn_bias._ts_w", "_rel_attn_bias._pos_w")


def research_case(config: str, concat_ua: bool, seed: int = 0) -> dict:
    """bf16 inputs, parameters (the module's state-dict names) and output gradient of one research block at a benchmarked
    shape; timestamps are cumulative gaps of up to one day as in the benchmark's data."""
    c = dict(RESEARCH_CONFIGS[config], concat_ua=concat_ua)
    g = torch.Generator().manual_seed(seed)
    D, H, dqk, dv, n = c["D"], c["H"], c["dqk"], c["dv"], c["n"]
    off = offsets_from(c["lengths"])
    L, B = int(off[-1]), len(c["lengths"])
    bf = torch.bfloat16
    w_in = dv * H * (3 if concat_ua else 1)
    c["params"] = {
        "_uvqk": (torch.randn(D, 2 * H * (dv + dqk), generator=g) / math.sqrt(D)).to(bf),  # x W has an rms of 1
        "_o.weight": (torch.randn(D, w_in, generator=g) / math.sqrt(w_in)).to(bf),
        "_o.bias": (0.1 * torch.randn(D, generator=g)).to(bf),
        "_rel_attn_bias._ts_w": (0.3 * torch.randn(129, generator=g)).to(bf),
        "_rel_attn_bias._pos_w": (0.3 * torch.randn(2 * n - 1, generator=g)).to(bf),
    }
    c["x"] = torch.randn(L, D, generator=g).to(bf)
    c["dy"] = torch.randn(L, D, generator=g).to(bf)
    c["seq_offsets"] = off
    c["timestamps"] = torch.randint(0, 86400, (B, n), generator=g).cumsum(1)
    return c


def _research_eval(c: dict, store) -> dict:
    leaves = {k: c["params"][k].double().requires_grad_() for k in RESEARCH_PARAMS}
    x = c["x"].double().requires_grad_()
    y = O.research_block_fwd(x, c["seq_offsets"], c["timestamps"], leaves["_uvqk"], leaves["_o.weight"], leaves["_o.bias"],
                             leaves["_rel_attn_bias._pos_w"], leaves["_rel_attn_bias._ts_w"], c["n"], c["H"], c["dqk"], c["dv"],
                             c["concat_ua"], 1e-6, store=store)
    y.backward(c["dy"].double())
    return dict(y=y.detach(), x=x.grad, **{k: t.grad for k, t in leaves.items()})


def research_reference(c: dict):
    """(staged, exact, dist): the research block in fp64 with bf16 rounding at every boundary where the module stores an
    activation, the same in plain fp64, and per gradient the rel-L2 distance of the staged one from the exact one -- how far
    bf16 storage of the forward activations alone moves each gradient."""
    staged, exact = _research_eval(c, torch.bfloat16), _research_eval(c, None)
    dist = {k: O.rel_l2(staged[k], exact[k]) for k in exact if k != "y"}
    return staged, exact, dist


def assert_pos_bands(got: torch.Tensor, ref: torch.Tensor, n: int, tol: float, what: str, band: int = SEG_ROWS) -> None:
    """rel-L2 <= tol on every band of `band` diagonals of a [2n - 1] position-bias gradient (entry n - 1 - delta belongs to the
    diagonal i - j = delta), so that the cross-tile diagonals (delta >= 64) are judged apart from the near-diagonal mass."""
    g, r = got.detach().double().cpu(), ref.detach().double().cpu()
    for d0 in range(0, n, band):
        d1 = min(n, d0 + band)
        sl = slice(n - d1, n - d0)  # entries of the diagonals delta in [d0, d1)
        err = O.rel_l2(g[sl], r[sl])
        assert err <= tol, f"{what}: diagonals i - j in [{d0}, {d1}): rel-L2 {err:.3e} > {tol:.1e}"


def assert_same_zeros(a: torch.Tensor, b: torch.Tensor, what: str) -> None:
    """The zero patterns of a and b are identical; the failure names the first element where they differ."""
    za, zb = (a == 0).cpu(), (b == 0).cpu()
    diff = (za != zb).nonzero()
    assert diff.numel() == 0, (f"{what}: zero patterns differ at {tuple(int(x) for x in diff[0])} "
                               f"({int(diff.shape[0])} elements)")


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
