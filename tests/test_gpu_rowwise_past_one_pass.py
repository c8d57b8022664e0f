"""The length-256 16-bit row-wise kernels of csrc/norm_fast.cu past their first grid pass, at the benchmark's row count and
dropout rate, against an fp64 oracle.

These kernels are persistent: the grid is capped and each warp loops over rows.  One pass of the output-stage backward covers
528 CTAs x 8 warps = 4,224 rows, one row per warp per step, and each lane sums its share of dw / db in registers over all the
rows of its warp.  One pass of the output-stage forward covers 1,056 x 8 x 2 = 16,896 rows.  A benchmark step has about 125k
rows (16 sequences of 0.9 - 1.0 x 8192), so each backward warp takes about 30 rows.  Here:

- the output stage u' * LN(attn) [concat], forward and backward, at 38,023 rows (two forward passes and a tail, nine backward
  passes and a tail) in both 16-bit dtypes, the three concat modes, silu(u) on and off and p in {0, 0.2, 0.5}; at the first row
  of each kernel's second pass; and at 124,519 rows in the configuration the benchmark trains.  out, dattn and du meet the
  assert_rel bound on the whole tensor and on every 4,224-row block, dw / db / mean / rstd the fp32 bound;
- dropout by value: the mask is a function of (seed, p, flat output index) only, so it is read off a forward of the same shape
  on inputs whose every output is bounded away from zero.  The oracle applies it, with the 1 / (1 - p) scale, to its forward
  output and to the incoming gradient, so a backward whose mask differs from the forward's fails on the values;
- the statistics of that mask at 124,519 rows and p = 0.2: the keep rate, overall and per block, and the agreement of rows one
  backward pass and one forward pass apart, and of the three concat parts of a row, at the rate of independent draws;
- SiLU on the u columns of a [124,519, 1024] uvqk buffer, and LayerNorm forward / backward at 124,519 rows;
- one STU layer at the benchmark's size: with y recomputed in the backward, the recomputed y is the saved one bit for bit,
  mask included, and every gradient equals that of the layer that keeps y.

Inputs are rounded to the kernel's dtype first; the oracle runs in fp64 on those values, 8,192 rows at a time.
"""
import math

import pytest
import torch

from oracle import hstu_oracle as O
from test_gpu_rowwise_general import _silu_refs
from util import (BLOCK_ROWS, TOL, _assert_ulp, assert_rel, assert_rel_row_sums, offsets_from, rel_row_sums)

pytestmark = pytest.mark.gpu
DEV = "cuda"
IDS = {torch.float32: "fp32", torch.bfloat16: "bf16", torch.float16: "fp16"}
F32 = TOL[torch.float32]  # statistics and parameter gradients are fp32 outputs: the fp32 bound
EPS = 1e-6
H, DV = 8, 32
W = H * DV                 # the normalised length of the fast kernels
BWD_PASS = BLOCK_ROWS      # rows of one pass of the output-stage backward (528 CTAs x 8 warps)
FWD_PASS = 1056 * 8 * 2    # rows of one pass of the output-stage forward (1,056 CTAs x 8 warps x 2 rows)
N_GRID = 38023             # 2 x 16,896 + 4,231 and 9 x 4,224 + 7
N_BENCH = 124519           # the order of one benchmark step's rows
CHUNK = 8192               # rows per oracle evaluation


def _ops():
    from generative_recommenders_b200.ops import hstu_compute as hc
    from generative_recommenders_b200.ops import layer_norm as ln
    return hc, ln


# ------------------------------------------------------------------------------------------------------------------
# oracle and checks (also used by test_rowwise_past_one_pass_cpu.py)
# ------------------------------------------------------------------------------------------------------------------
def nmd_oracle(attn, u, w, b, dout, keep, p, silu_u, concat):
    """The output stage in fp64 on a chunk of rows: out = dropout(u' * LN(attn)) or dropout([u' | attn or LN(attn) | y]),
    u' = silu(u) or u, and its backward from `dout`.  `keep` (bool, the shape of out, or None for no dropout) is the mask:
    kept elements are scaled by 1 / (1 - p) in out and in the incoming gradient.  Returns out, dattn, du, and this chunk's
    share of dw and db, and its mean and rstd."""
    a, uu, w64, b64, g = (t.detach().cpu().double() for t in (attn, u, w, b, dout))
    mean = a.mean(1, keepdim=True)
    xc = a - mean
    rstd = torch.rsqrt(xc.square().mean(1, keepdim=True) + EPS)
    xhat = xc * rstd
    nrm = xhat * w64 + b64
    if silu_u:
        sg = torch.sigmoid(uu)
        uf, dsil = uu * sg, sg * (1 + uu * (1 - sg))
    else:
        uf = uu
    y = uf * nrm
    out = y if concat == 0 else torch.cat([uf, a if concat == 1 else nrm, y], 1)
    if keep is not None:
        scale = keep.cpu().double() / (1.0 - p)
        out, g = out * scale, g * scale
    if concat:
        gu, ga, gy = g.split(W, 1)
    else:
        gu = ga = torch.zeros_like(g)
        gy = g
    duf = gy * nrm + gu
    dn = gy * uf + (ga if concat == 2 else 0.0)  # d / d LN(attn)
    dxh = dn * w64
    dattn = (dxh - dxh.mean(1, keepdim=True) - xhat * (dxh * xhat).mean(1, keepdim=True)) * rstd
    if concat == 1:
        dattn = dattn + ga  # concat_ux: the middle part is attn itself
    du = duf * dsil if silu_u else duf
    return out, dattn, du, (dn * xhat).sum(0), dn.sum(0), mean.squeeze(1), rstd.squeeze(1)


def _within(count_hit, count, expect, label, what):
    """count_hit of count Bernoulli(expect) trials: within 5 binomial standard deviations of expect."""
    rate = count_hit / count
    lim = 5 * math.sqrt(expect * (1 - expect) / count)
    assert abs(rate - expect) <= lim, (f"{what}: {label}: rate {rate:.5f} over {count} elements, expected {expect:.5f} "
                                       f"+- {lim:.1e} (5 binomial sd)")


def _per_block(row_counts, per_row, expect, label, what):
    """The rate of `row_counts` [n] (hits per row, `per_row` trials each) overall and per BWD_PASS-row block."""
    n = row_counts.shape[0]
    _within(int(row_counts.sum()), n * per_row, expect, label, what)
    for r0 in range(0, n, BWD_PASS):
        r1 = min(n, r0 + BWD_PASS)
        _within(int(row_counts[r0:r1].sum()), (r1 - r0) * per_row, expect, f"{label}, rows [{r0}, {r1})", what)


def check_mask_stats(keep, p, what):
    """keep [n, K] (bool, K = W or 3 W): the keep rate is 1 - p overall and per block; rows r and r + BWD_PASS, and rows r
    and r + FWD_PASS, agree at the rate of independent draws p^2 + (1 - p)^2 (overall and per block of r), as do the three
    concat parts of a row.  Each bound is 5 binomial standard deviations.  A mask indexed by the row's position within its
    pass of the grid instead of its absolute row agrees at rate 1 across a pass."""
    n, K = keep.shape
    _per_block(keep.sum(1), K, 1 - p, "keep rate", what)
    agree = p * p + (1 - p) ** 2
    for shift in (BWD_PASS, FWD_PASS):
        _per_block((keep[shift:] == keep[:-shift]).sum(1), K, agree, f"rows r and r + {shift} agree", what)
    if K == 3 * W:
        parts = keep.view(n, 3, W)
        for i, j in ((0, 1), (1, 2), (0, 2)):
            _within(int((parts[:, i] == parts[:, j]).sum()), n * W, agree, f"concat parts {i} and {j} agree", what)


# ------------------------------------------------------------------------------------------------------------------
# output stage
# ------------------------------------------------------------------------------------------------------------------
def _inputs(n, concat, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    attn = (torch.randn(n, W, generator=g) * 0.8 + 0.1).to(dtype)
    u = torch.randn(n, W, generator=g).to(dtype)
    w = (1 + 0.5 * torch.randn(W, generator=g)).to(dtype)  # far from ones: a backward that drops w cannot pass
    b = (0.2 * torch.randn(W, generator=g)).to(dtype)
    dout = torch.randn(n, W * (3 if concat else 1), generator=g).to(dtype)
    return attn, u, w, b, dout


def dropout_keep(n, concat, p, seed, dtype):
    """The kernel's keep mask for (seed, p) over an [n, W] output stage: the non-zeros of a forward on attn ~ U[2, 4],
    u ~ U[0.5, 1.5], w = 1, b = 4, whose outputs u, attn and u * (LN(attn) + 4) are all at least 0.5 before the 1 / (1 - p)
    scale (LN of a uniform row lies within +-1.8), so an output is zero exactly where it was dropped."""
    hc, _ = _ops()
    g = torch.Generator(device=DEV).manual_seed(seed % 2**31)
    attn = (2 + 2 * torch.rand(n, W, generator=g, device=DEV)).to(dtype)
    u = (0.5 + torch.rand(n, W, generator=g, device=DEV)).to(dtype)
    w = torch.ones(W, device=DEV, dtype=dtype)
    b = torch.full((W,), 4.0, device=DEV, dtype=dtype)
    out, _, _ = hc.cuda_norm_mul_dropout_fwd(attn, u, w, b, EPS, p, seed, False, concat, False, H, DV)
    kept = out != 0
    assert bool((out[kept] >= 0.5).all()), "mask probe: an output that is not dropped is below 0.5"
    return kept


def _output_stage_case(n, dtype, concat, silu_u, p, seed):
    hc, _ = _ops()
    attn, u, w, b, dout = _inputs(n, concat, dtype, seed)
    dseed = 0x2545F4914F6CDD1D + 7919 * seed  # the dropout seed of this case
    ad, ud, wd, bd = (t.to(DEV) for t in (attn, u, w, b))
    out, mean, rstd = hc.cuda_norm_mul_dropout_fwd(ad, ud, wd, bd, EPS, p, dseed, silu_u, concat, False, H, DV)
    dattn, du, dw, db = hc.cuda_norm_mul_dropout_bwd(dout.to(DEV), ad, ud, wd, bd, mean, rstd, p, dseed, silu_u, concat,
                                                     False, H, DV)
    keep = dropout_keep(n, concat, p, dseed, dtype) if p > 0 else None
    names = ("out", "dattn", "du")
    sums = {k: [] for k in names}
    dw_r = db_r = 0.0
    mean_r, rstd_r = [], []
    for r0 in range(0, n, CHUNK):
        r1 = min(n, r0 + CHUNK)
        ref = nmd_oracle(attn[r0:r1], u[r0:r1], w, b, dout[r0:r1], None if keep is None else keep[r0:r1], p, silu_u, concat)
        for k, got, r in zip(names, (out, dattn, du), ref[:3]):
            sums[k].append(rel_row_sums(got[r0:r1], r))
        dw_r, db_r = dw_r + ref[3], db_r + ref[4]
        mean_r.append(ref[5])
        rstd_r.append(ref[6])
    case = f"n {n} {IDS[dtype]} concat {concat} silu {silu_u} p {p}"
    for k in names:
        assert_rel_row_sums(torch.cat(sums[k]), dtype, f"{k} ({case})")
    assert_rel(dw, dw_r, f"dw ({case})", tol=F32)
    assert_rel(db, db_r, f"db ({case})", tol=F32)
    assert_rel(mean, torch.cat(mean_r), f"mean ({case})", tol=F32)
    assert_rel(rstd, torch.cat(rstd_r), f"rstd ({case})", tol=F32)


@pytest.mark.parametrize("p", [0.0, 0.2, 0.5])
@pytest.mark.parametrize("silu_u", [False, True])
@pytest.mark.parametrize("concat", [0, 1, 2])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=IDS.get)
def test_output_stage_past_one_pass(dtype, concat, silu_u, p):
    _output_stage_case(N_GRID, dtype, concat, silu_u, p, seed=100 * concat + 10 * int(silu_u) + int(10 * p)
                       + (1000 if dtype == torch.float16 else 0))


@pytest.mark.parametrize("silu_u", [False, True])
@pytest.mark.parametrize("n", [BWD_PASS + 1, FWD_PASS + 1])  # the first row of the backward's / the forward's second pass
def test_output_stage_first_row_of_the_second_pass(n, silu_u):
    _output_stage_case(n, torch.bfloat16, 1, silu_u, 0.2, seed=n + int(silu_u))


def test_output_stage_at_the_benchmark_rows():
    """bf16, concat_ux, no silu on u, p = 0.2: the output stage of every benchmarked STU layer."""
    _output_stage_case(N_BENCH, torch.bfloat16, 1, False, 0.2, seed=8192)


@pytest.mark.parametrize("concat", [0, 1])
def test_dropout_mask_statistics_at_the_benchmark_rows(concat):
    check_mask_stats(dropout_keep(N_BENCH, concat, 0.2, 0x5DEECE66D + concat, torch.bfloat16), 0.2, f"concat {concat}")


# ------------------------------------------------------------------------------------------------------------------
# SiLU and LayerNorm at the benchmark's row count
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16], ids=IDS.get)
def test_silu_on_the_uvqk_u_columns_at_the_benchmark_rows(dtype):
    """The u columns of uvqk at the benchmark's layout (H = 8, dv = dqk = 32: row stride 2 H (dv + dqk) = 1024).  The
    backward writes d_u in place into a NaN-poisoned duvqk: every other column must stay bit-identical."""
    hc, _ = _ops()
    n, c, stride = N_BENCH, W, 2 * H * (DV + DV)
    g = torch.Generator().manual_seed(31 + c)
    buf = (3 * torch.randn(n, stride, generator=g)).to(dtype)
    dy = torch.randn(n, c, generator=g).to(dtype)
    bufd = buf.to(DEV)
    x = bufd[:, :c]
    y = hc.cuda_silu_fwd(x)
    poison = torch.full((n, stride), float("nan"), dtype=dtype, device=DEV)
    before = poison.clone()
    hc.cuda_silu_bwd(dy.to(DEV), x, poison[:, :c])
    for r0 in range(0, n, 4 * CHUNK):
        r1 = min(n, r0 + 4 * CHUNK)
        fwd, bwd, mag_f, mag_b = _silu_refs(buf[r0:r1, :c], dy[r0:r1])
        _assert_ulp(y[r0:r1], fwd, mag_f, dtype, f"silu forward, rows from {r0}")
        _assert_ulp(poison[r0:r1, :c], bwd, mag_b, dtype, f"silu backward, rows from {r0}")
    ibits = {torch.float32: torch.int32, torch.bfloat16: torch.int16, torch.float16: torch.int16}[dtype]
    assert torch.equal(poison[:, c:].view(ibits), before[:, c:].view(ibits)), "silu backward wrote outside d_u"
    assert torch.equal(bufd.view(ibits), buf.to(DEV).view(ibits)), "silu forward modified its input"


def test_layer_norm_256_at_the_benchmark_rows():
    _, ln = _ops()
    n, dtype = N_BENCH, torch.bfloat16
    g = torch.Generator().manual_seed(256)
    x = (torch.randn(n, W, generator=g) * 1.7 + 0.3).to(dtype)
    w = (1 + 0.5 * torch.randn(W, generator=g)).to(dtype)
    b = (0.2 * torch.randn(W, generator=g)).to(dtype)
    dy = torch.randn(n, W, generator=g).to(dtype)
    xd, wd, bd = x.to(DEV), w.to(DEV), b.to(DEV)
    y, mean, rstd = ln.cuda_layer_norm_fwd(xd, wd, bd, EPS, False)
    dx, dw, db = ln.cuda_layer_norm_bwd(dy.to(DEV), xd, wd, bd, mean, rstd, False)
    sums = {"y": [], "dx": []}
    dw_r = db_r = 0.0
    mean_r, rstd_r = [], []
    for r0 in range(0, n, CHUNK):
        r1 = min(n, r0 + CHUNK)
        yr, mr, rr = O.layer_norm_fwd(x[r0:r1], w, b, EPS, dtype=torch.float64)
        dxr, dwr, dbr = O.layer_norm_bwd(dy[r0:r1], x[r0:r1], w, mr, rr, dtype=torch.float64)
        sums["y"].append(rel_row_sums(y[r0:r1], yr))
        sums["dx"].append(rel_row_sums(dx[r0:r1], dxr))
        dw_r, db_r = dw_r + dwr, db_r + dbr
        mean_r.append(mr)
        rstd_r.append(rr)
    for k, s in sums.items():
        assert_rel_row_sums(torch.cat(s), dtype, f"layer norm {k}")
    assert_rel(dw, dw_r, "layer norm dw", tol=F32)
    assert_rel(db, db_r, "layer norm db", tol=F32)
    assert_rel(mean, torch.cat(mean_r), "layer norm mean", tol=F32)
    assert_rel(rstd, torch.cat(rstd_r), "layer norm rstd", tol=F32)


# ------------------------------------------------------------------------------------------------------------------
# the STU layer at the benchmark's size: y recomputed in the backward against y kept from the forward
# ------------------------------------------------------------------------------------------------------------------
def test_stu_layer_recomputed_y_is_the_saved_y_at_the_benchmark_size(monkeypatch):
    """One bf16 STU layer in the benchmarked configuration (D = 256, H = 8, dqk = dv = 32, output dropout 0.2) on 16
    sequences of [0.9, 1.0) x 8192 rows with 1 - 20 targets, run with recompute_y on and off after the same
    torch.cuda.manual_seed.  The output stage's forward is recorded at every call: the y recomputed in the backward must be
    the forward's y bit for bit (its dropout mask included), and x.grad and every parameter gradient must be bitwise equal
    between the two modes."""
    from generative_recommenders_b200.modules.stu import STULayer, STULayerConfig
    hc, _ = _ops()
    g = torch.Generator().manual_seed(1001)
    lengths = (8192 * (0.9 + 0.1 * torch.rand(16, generator=g, dtype=torch.float64))).long()
    nt = torch.minimum(torch.randint(1, 21, (16,), generator=g), lengths)
    off = offsets_from(lengths)
    L, D = int(off[-1]), 256
    torch.manual_seed(7)
    layer = STULayer(STULayerConfig(embedding_dim=D, num_heads=H, hidden_dim=DV, attention_dim=DV, output_dropout_ratio=0.2,
                                    target_aware=True, recompute_normed_x=True, recompute_uvqk=True, recompute_y=True,
                                    sort_by_length=True)).to(DEV).to(torch.bfloat16)
    x0 = torch.randn(L, D, generator=g).to(torch.bfloat16).to(DEV)
    dy = torch.randn(L, D, generator=g).to(torch.bfloat16).to(DEV)
    ys = []
    real_fwd = hc.cuda_norm_mul_dropout_fwd

    def recording_fwd(*args):
        res = real_fwd(*args)
        ys.append(res[0])
        return res

    monkeypatch.setattr(hc, "cuda_norm_mul_dropout_fwd", recording_fwd)
    runs = {}
    for recompute in (True, False):
        layer._recompute_y = recompute
        layer.zero_grad(set_to_none=True)
        ys.clear()
        torch.cuda.manual_seed(4321)
        x = x0.clone().requires_grad_()
        out = layer(x=x, x_lengths=lengths.to(DEV), x_offsets=off.to(DEV), max_seq_len=8192, num_targets=nt.to(DEV))
        out.backward(dy)
        runs[recompute] = dict(ys=list(ys), grads={"x": x.grad, **{n: p.grad for n, p in layer.named_parameters()}})
    assert [len(runs[True]["ys"]), len(runs[False]["ys"])] == [2, 1], "output-stage forwards per step: recompute / keep y"
    y_fwd, y_re = runs[True]["ys"]
    assert y_fwd.shape == (L, 3 * W)
    i16 = torch.int16
    assert torch.equal(y_fwd.view(i16), y_re.view(i16)), "the y recomputed in the backward differs from the forward's y"
    assert torch.equal(y_fwd.view(i16), runs[False]["ys"][0].view(i16)), "y differs between recompute_y on and off"
    dropped = (y_fwd == 0).sum().item() / y_fwd.numel()
    assert abs(dropped - 0.2) < 0.005, f"share of zeros in y: {dropped:.4f}, expected about 0.2"
    for k, a in runs[True]["grads"].items():
        r = runs[False]["grads"][k]
        assert a is not None and r is not None and a.dtype == r.dtype == torch.bfloat16, k
        assert torch.equal(a.view(i16), r.view(i16)), f"{k}.grad differs between recompute_y on and off"
