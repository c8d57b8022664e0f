"""The kernels on the model's input path at the edges where they branch, through the C ABI with NaN-poisoned outputs so that
a row no thread writes cannot pass:

* jagged x dense bmm (csrc/jagged_bmm.cu): forward, d_jagged (the same kernel reading dense transposed) and the wgrad kernel,
  at K / N tails and several N tiles, sequences shorter than, equal to and longer than max_seq_len (past the last 64-row
  tile of the grid too), fp32 / bf16 / fp16, int32 / int64 offsets.  Rows at positions >= max_seq_len must be exact zeros.
* timestamp + position embeddings (csrc/position.cu): forward bit for bit against the oracle on its 16-bit vector and scalar
  paths and in fp32; the backward's 1, 2 and 4 columns per thread, one and many rows per CTA; position and time-bucket index
  edges.
* jagged concat / split (csrc/jagged.cu): bitwise, at each copy width (16, 4, 2, 1 bytes) and on unaligned base pointers.

Each element is judged on its own: |got - ref| against a bound from the fp32 accumulation of that element's terms, so a
misrouted row, column or tile fails even when the rest of the tensor is right."""
import math

import numpy as np
import pytest
import torch

from oracle import hstu_oracle as O
from util import U32, assert_table_entries, offsets_from

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")

U = {torch.float32: 0.0, torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}  # unit roundoff of the stored result
TINY = {torch.float32: 0.0, torch.bfloat16: 0.0, torch.float16: 2.0 ** -25}    # absolute rounding in fp16's subnormal range


def _lib():
    from generative_recommenders_b200 import _lib

    return _lib


def _stream():
    return _lib().stream_ptr(DEV)


def _nan(shape, dtype):
    return torch.full(shape, float("nan"), dtype=dtype, device=DEV)


def _assert_elements(got, ref, mag, count, dtype, what):
    """|got - ref| <= u |ref| + (1 + u) (count + 1) 2^-24 mag per element: the fp32 sum of `count` products whose absolute
    values sum to `mag` (plus the bias, counted in mag), then one rounding to the stored dtype (u = 0 in fp32).  An element
    without terms (mag = 0) must be exactly zero; NaN fails."""
    u = U[dtype]
    mag = mag.double()
    lim = u * ref.abs() + (1 + u) * (count + 1) * U32 * mag + TINY[dtype] * (mag > 0)
    assert_table_entries(got, ref, lim, what)


def _assert_zero_rows(t, off, max_seq_len, what):
    """Rows at positions >= max_seq_len of each sequence are exact zeros (NaN, i.e. never written, fails)."""
    x = t.detach().float().cpu()
    for b in range(len(off) - 1):
        s, e = off[b], off[b + 1]
        if e - s <= max_seq_len:
            continue
        bad = (x[s + max_seq_len:e] != 0).any(-1).nonzero()
        assert bad.numel() == 0, (f"{what}: sequence {b} (length {e - s}) row {max_seq_len + int(bad[0])} (>= max_seq_len "
                                  f"{max_seq_len}) is not zero: {x[s + max_seq_len + int(bad[0])][:4].tolist()}")


# ----------------------------------------------------------------------------------------------------------------------------
# jagged x dense bmm + broadcast bias
# ----------------------------------------------------------------------------------------------------------------------------

BMM_KN = [(1, 1), (15, 17), (16, 64), (100, 130), (512, 65)]  # K tails, N tails; N = 130 and d_jagged's N = 512: several N tiles


def _bmm_lengths(m):
    # empty first and last; one 64-row tile, its tail and the next; max_seq_len and just past it; past the grid's last
    # 64-row tile (64 * ceil(m / 64)) by up to two tiles
    return [0, 1, 63, 64, 65, 127, 128, 129, m, m + 1, m + 64, 3 * m, 0]


def _bmm_inputs(lengths, K, N, dtype, idt, seed):
    g = torch.Generator().manual_seed(seed)
    off = offsets_from(lengths, dtype=idt)
    L, B = int(off[-1]), len(lengths)
    jag = torch.empty(L, K).uniform_(-1, 1, generator=g).to(dtype)
    dense = torch.empty(B, K, N).uniform_(-1, 1, generator=g).to(dtype)
    bias = torch.empty(B, N).uniform_(-1, 1, generator=g).to(dtype)
    dout = torch.randn(L, N, generator=g).to(dtype)
    return off, jag, dense, bias, dout


def _bmm_reference(m, off, jag, dense, bias, dout):
    """fp64 oracle on the rounded inputs: (out, d_jagged, d_dense, d_bias), and the same on their absolute values (the sums
    of |terms| per element that bound the fp32 accumulation)."""
    def run(j, d, b, g):
        j, d, b = (t.double().requires_grad_() for t in (j, d, b))
        out = O.jagged_dense_bmm_broadcast_add(m, off, j, d, b)
        out.backward(g.double())
        return out.detach(), j.grad, d.grad, b.grad

    return run(jag, dense, bias, dout), run(jag.abs(), dense.abs(), bias.abs(), dout.abs())


def _bmm_check(m, off, K, N, dtype, got, ref, mag, what):
    out, dj, dd, db = got
    offl = [int(x) for x in off.tolist()]
    _assert_zero_rows(out, offl, m, f"{what} out")
    _assert_zero_rows(dj, offl, m, f"{what} d_jagged")
    _assert_elements(out, ref[0], mag[0], K, dtype, f"{what} out")
    _assert_elements(dj, ref[1], mag[1], N, dtype, f"{what} d_jagged")
    rows = (off[1:] - off[:-1]).clamp(max=m).double()  # rows summed into each batch entry's d_dense / d_bias
    _assert_elements(dd, ref[2], mag[2], rows.view(-1, 1, 1), dtype, f"{what} d_dense")
    _assert_elements(db, ref[3], mag[3], rows.view(-1, 1), dtype, f"{what} d_bias")


def _bmm_abi(m, off, jag, dense, bias, dout):
    """Forward, d_jagged and wgrad through the C ABI into NaN-filled outputs."""
    lib = _lib()
    L, K = jag.shape
    B, _, N = dense.shape
    dt = jag.dtype
    j, d, b, g, o = (t.to(DEV).contiguous() for t in (jag, dense, bias, dout, off))
    i64 = int(o.dtype == torch.int64)
    code = lib.dtype_code(j)
    out, dj, dd, db = _nan((L, N), dt), _nan((L, K), dt), _nan((B, K, N), dt), _nan((B, N), dt)
    lib.check(lib.lib().hstu_jagged_dense_bmm_broadcast_add(j.data_ptr(), d.data_ptr(), b.data_ptr(), out.data_ptr(),
                                                            o.data_ptr(), i64, B, K, N, m, 0, code, _stream()), "bmm")
    # d_jagged = dout @ dense^T: inner dimension N, K outputs per row
    lib.check(lib.lib().hstu_jagged_dense_bmm_broadcast_add(g.data_ptr(), d.data_ptr(), None, dj.data_ptr(), o.data_ptr(),
                                                            i64, B, N, K, m, 1, code, _stream()), "bmm d_jagged")
    lib.check(lib.lib().hstu_jagged_dense_bmm_wgrad(j.data_ptr(), g.data_ptr(), dd.data_ptr(), db.data_ptr(), o.data_ptr(), i64,
                                                    B, K, N, m, code, _stream()), "bmm wgrad")
    torch.cuda.synchronize()
    return tuple(t.cpu() for t in (out, dj, dd, db))


@pytest.mark.parametrize("idt", [torch.int32, torch.int64], ids=["off32", "off64"])
@pytest.mark.parametrize("m", [1, 100, 128])
@pytest.mark.parametrize("K,N", BMM_KN, ids=[f"K{k}N{n}" for k, n in BMM_KN])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16], ids=["f32", "bf16", "f16"])
def test_jagged_bmm_edges(dtype, K, N, m, idt):
    """Row tiles at and past max_seq_len (m = 1, 100: not a multiple of 64, 128: one), K / N tails; every element per its
    bound, rows past max_seq_len exact zeros in out and d_jagged and absent from d_dense / d_bias."""
    off, jag, dense, bias, dout = _bmm_inputs(_bmm_lengths(m), K, N, dtype, idt, seed=K * 1000 + N + m)
    got = _bmm_abi(m, off, jag, dense, bias, dout)
    ref, mag = _bmm_reference(m, off, jag, dense, bias, dout)
    _bmm_check(m, off, K, N, dtype, got, ref, mag, f"{dtype} K={K} N={N} max_seq_len={m}")


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
def test_jagged_bmm_all_empty(dtype):
    """Every sequence empty: no row to write, and d_dense / d_bias are exact zeros (the wgrad kernel's zero-row loop)."""
    off, jag, dense, bias, dout = _bmm_inputs([0, 0, 0], 15, 17, dtype, torch.int64, seed=3)
    out, dj, dd, db = _bmm_abi(100, off, jag, dense, bias, dout)
    assert out.shape == (0, 17) and dj.shape == (0, 15)
    assert torch.equal(dd, torch.zeros_like(dd)) and torch.equal(db, torch.zeros_like(db))


def test_jagged_bmm_autograd_facade():
    """The autograd facade on one of the cases above (bf16, K = 100, N = 130, max_seq_len = 100, int32 offsets)."""
    from generative_recommenders_b200.common import HammerKernel
    from generative_recommenders_b200.ops.jagged_tensors import jagged_dense_bmm_broadcast_add

    m, K, N, dtype = 100, 100, 130, torch.bfloat16
    off, jag, dense, bias, dout = _bmm_inputs(_bmm_lengths(m), K, N, dtype, torch.int32, seed=K * 1000 + N + m)
    j, d, b = (t.to(DEV).requires_grad_() for t in (jag, dense, bias))
    out = jagged_dense_bmm_broadcast_add(max_seq_len=m, seq_offsets=off.to(DEV), jagged=j, dense=d, bias=b,
                                         kernel=HammerKernel.CUDA)
    out.backward(dout.to(DEV))
    got = tuple(t.detach().cpu() for t in (out, j.grad, d.grad, b.grad))
    ref, mag = _bmm_reference(m, off, jag, dense, bias, dout)
    _bmm_check(m, off, K, N, dtype, got, ref, mag, "facade")


# ----------------------------------------------------------------------------------------------------------------------------
# timestamp + position embeddings
# ----------------------------------------------------------------------------------------------------------------------------

BASE_TS = 10 ** 12


def _sqrt_edge_dts():
    # exact bucket boundaries under sqrt: dt = 60 k^2 gives x = k^2 exactly, so bucket k; 60 k^2 - 1 is bucket k - 1.
    # dt = 0 and negative dt (clamped to 1e-6: bucket 0); dt above 2^24 (the int64 -> fp32 conversion rounds) and far past
    # the last bucket (clamped to num_time_buckets)
    edges = [v for k in range(1, 6) for v in (60 * k * k, 60 * k * k - 1, 60 * k * k + 1)]
    return edges + [0, -1, -86400, 2 ** 24 + 1, 2 ** 24 + 3, 2 ** 25 + 1, 123456789013, 60 * 30 * 30]


def _log_dts(g, n):
    """Random dt for the log buckets, away from values whose fp32 log lies within 1e-4 of an integer: CUDA's logf and the
    host's fp32 log may differ by an ulp there and so round to different buckets.  Includes dt = 0, negative dt and dt past
    2^24 (all kept off the integer boundaries by the same test)."""
    cand = torch.cat([torch.tensor([0, -7, 2 ** 24 + 5, 3 * 10 ** 9 + 1]),
                      torch.randint(1, 10 ** 7, (4 * n,), generator=g)]).numpy()
    x = np.maximum(cand.astype(np.float32), np.float32(1e-6)) / np.float32(60.0)
    y = np.log(x.astype(np.float64))
    keep = cand[(np.abs(y - np.round(y)) > 1e-4) | (y < 0)]
    return keep[:n].tolist()


def _pos_case(dtype, D, lengths, *, targets=None, interleave=False, ctx=0, pos_rows=None, ts_rows=200, fn="sqrt",
              same_ts=(), seed=0):
    """Inputs of one position-embedding case.  targets: None, or a list of num_targets (int32 tensor); `same_ts`: sequences
    whose rows all share one timestamp (dt = 0: one time bucket for the whole sequence)."""
    g = torch.Generator().manual_seed(seed)
    B = len(lengths)
    max_len = max(lengths + [1])
    off = offsets_from(lengths)
    L = int(off[-1])
    dts = _sqrt_edge_dts() if fn == "sqrt" else _log_dts(g, 64)
    ts = []
    for b, n in enumerate(lengths):
        if b in same_ts:
            ts += [BASE_TS] * n
            continue
        # row r gets dt = pool[(r + b) % len(pool)] against the last row, whose dt is 0 (the query time)
        ts += [BASE_TS - dts[(r + b) % len(dts)] for r in range(n - 1)] + ([BASE_TS] if n else [])
    return dict(
        alpha=0.5 if seed % 2 else 1.7, ctx=ctx, interleave=interleave, fn=fn, seq_offsets=off,
        seq_lengths=torch.tensor(lengths, dtype=torch.int64), timestamps=torch.tensor(ts, dtype=torch.int64).view(L),
        num_targets=None if targets is None else torch.tensor(targets, dtype=torch.int32),
        pos_w=torch.empty(pos_rows or max_len + ctx, D).uniform_(-1, 1, generator=g),
        ts_w=torch.empty(ts_rows, D).uniform_(-1, 1, generator=g),
        x=torch.empty(L, D).uniform_(-1, 1, generator=g).to(dtype),
        dout=torch.randn(L, D, generator=g).to(dtype))


def _pos_abi(c, misalign=False):
    """Forward and backward through the C ABI: out and d_seq NaN-filled, the index buffers -1-filled.  misalign: activation
    and output one element past a 16-byte boundary, so the 16-bit kernel takes its scalar path whatever D is."""
    lib = _lib()
    x = c["x"]
    L, D = x.shape
    dt = x.dtype
    pw, tw = c["pos_w"].to(DEV), c["ts_w"].to(DEV)
    nb = min(tw.shape[1] - 1, tw.shape[0] - 1)
    sh = 1 if misalign else 0
    xbuf = torch.empty(L * D + sh, dtype=dt, device=DEV)
    xbuf[sh:] = x.reshape(-1).to(DEV)
    obuf = _nan((L * D + sh,), dt)
    xd, out = xbuf[sh:].view(L, D), obuf[sh:].view(L, D)
    off, lens, ts = c["seq_offsets"].to(DEV), c["seq_lengths"].to(DEV), c["timestamps"].to(DEV)
    nt = None if c["num_targets"] is None else c["num_targets"].to(DEV)
    pi = torch.full((L,), -1, dtype=torch.int32, device=DEV)
    ti = torch.full((L,), -1, dtype=torch.int32, device=DEV)
    lib.check(lib.lib().hstu_position_embeddings_fwd(
        xd.data_ptr(), out.data_ptr(), pw.data_ptr(), tw.data_ptr(), off.data_ptr(), lens.data_ptr(), lib.ptr(nt), ts.data_ptr(),
        pi.data_ptr(), ti.data_ptr(), L, len(c["seq_lengths"]), D, pw.shape[0], nb, c["ctx"], c["alpha"], int(c["interleave"]),
        int(c["fn"] == "log"), 1, 1, 0, lib.dtype_code(xd), _stream()), "position fwd")
    g = c["dout"].to(DEV)
    dseq = _nan((L, D), dt)
    dpos, dts = torch.zeros_like(pw), torch.zeros_like(tw)
    lib.check(lib.lib().hstu_position_embeddings_bwd(g.data_ptr(), dseq.data_ptr(), dpos.data_ptr(), dts.data_ptr(), pi.data_ptr(),
                                                     ti.data_ptr(), L, D, c["alpha"], lib.dtype_code(g), _stream()), "position bwd")
    torch.cuda.synchronize()
    if misalign:
        assert math.isnan(float(obuf[0])), "the element in front of the output was written"
    return out.cpu(), pi.cpu().long(), ti.cpu().long(), dseq.cpu(), dpos.cpu(), dts.cpu(), nb


def _pos_check(c, misalign=False):
    out, pi, ti, dseq, dpos, dts, nb = _pos_abi(c, misalign)
    args = (c["seq_offsets"], c["seq_lengths"], c["timestamps"], c["num_targets"], c["ctx"])
    pos, bkt = O.position_indices(*args, c["pos_w"].shape[0], nb, c["interleave"], c["fn"])
    assert torch.equal(pi, pos), f"position indices differ at row {int((pi != pos).nonzero()[0])}"
    assert torch.equal(ti, bkt), f"time buckets differ at row {int((ti != bkt).nonzero()[0])}"
    rout, rdseq, _, _ = O.add_timestamp_positional_embeddings(
        c["alpha"], c["ctx"], c["pos_w"], c["ts_w"], c["seq_offsets"], c["seq_lengths"], c["x"], c["timestamps"],
        c["num_targets"], c["interleave"], c["fn"], c["dout"], num_time_buckets=nb)
    # the three roundings of the eager path, bit for bit (NaN rows, never written, differ too)
    bad = (out.view(-1, out.shape[1]) != rout).any(-1).nonzero()
    assert bad.numel() == 0, f"out differs from the oracle first at row {int(bad[0])}"
    assert torch.equal(dseq, rdseq), "d_seq must be dout * alpha rounded once"
    # table gradients: fp64 scatter-adds, each entry within (count) 2^-24 sum|dout| of its rows (fp32 atomics in any order)
    g = c["dout"].double()
    for got, idx, what in ((dpos, pos, "d_pos_w"), (dts, bkt, "d_ts_w")):
        ref = torch.zeros(got.shape, dtype=torch.float64).index_add_(0, idx, g)
        mass = torch.zeros(got.shape, dtype=torch.float64).index_add_(0, idx, g.abs())
        cnt = torch.bincount(idx, minlength=got.shape[0]).double().view(-1, 1)
        assert_table_entries(got, ref, cnt * U32 * mass, what)
    return pos, bkt, nb


# [empty first, middle, last] ... one-row sequences, sequences shorter than the contextual prefix
_EDGE_LENGTHS = [0, 1, 2, 17, 0, 40, 5, 1, 33, 0]


def test_position_vec16_targets_ctx():
    """bf16 D = 64, aligned: the 16-bit vector path (8 columns per lane).  int32 num_targets, one of them equal to its
    sequence's length (no history left); a contextual prefix (ctx = 3) longer than the one- and two-row sequences; sqrt
    buckets at their exact boundaries."""
    lengths = _EDGE_LENGTHS
    nt = [0, 1, 0, 4, 0, 40, 2, 0, 7, 0]
    c = _pos_case(torch.bfloat16, 64, lengths, targets=nt, ctx=3, seed=1)
    pos, bkt, nb = _pos_check(c)
    assert {1, 2, 3, 4, 5, nb} <= set(bkt.tolist()) and 0 in bkt.tolist()  # boundaries reached, clamp at the top reached


def test_position_vec16_interleave_clamped_pos():
    """fp16 D = 136 (17 vectors per row: a partial second step of the lanes): interleaved targets; a pos_w of 12 rows, fewer
    than max_seq_len + ctx, so the index clamp to max_pos_ind - 1 fires; log buckets."""
    nt = [0, 0, 1, 3, 0, 10, 1, 0, 16, 0]
    c = _pos_case(torch.float16, 136, _EDGE_LENGTHS, targets=nt, interleave=True, ctx=2, pos_rows=12, fn="log", seed=2)
    pos, _, _ = _pos_check(c)
    assert int(pos.max()) == 11


def test_position_scalar16_d36():
    """bf16 D = 36 (D % 8 != 0): the 16-bit scalar path.  No num_targets; a ts_w of 20 rows, fewer than its 36 columns, so
    the bucket clamp is min(ts_w rows, columns) - 1 = 19."""
    c = _pos_case(torch.bfloat16, 36, _EDGE_LENGTHS, ctx=8, ts_rows=20, seed=3)
    _, bkt, nb = _pos_check(c)
    assert nb == 19 and int(bkt.max()) == 19


def test_position_scalar16_misaligned_d64():
    """fp16 D = 64 on a one-element storage offset: vec_ok is false, so the scalar path runs where D alone would pick the
    vector one."""
    c = _pos_case(torch.float16, 64, _EDGE_LENGTHS, targets=[0, 1, 0, 2, 0, 5, 5, 1, 0, 0], ctx=1, seed=4)
    _pos_check(c, misalign=True)


@pytest.mark.parametrize("D", [36, 136])
def test_position_f32(D):
    """fp32 activations (always the scalar path) with log and sqrt buckets."""
    c = _pos_case(torch.float32, D, _EDGE_LENGTHS, targets=[0, 0, 2, 1, 0, 3, 0, 1, 9, 0], ctx=2,
                  fn="log" if D == 36 else "sqrt", seed=5 + D)
    _pos_check(c)


@pytest.mark.parametrize("D", [256, 257, 512, 513, 1000, 1024])
def test_position_bwd_columns(D):
    """The backward's columns per thread: 1 (D <= 256), 2 (D <= 512), 4 (D <= 1024); fewer than 32 rows per CTA (L < 32 at
    one CTA)."""
    c = _pos_case(torch.bfloat16, D, [0, 3, 1, 0, 20, 0], targets=[0, 1, 0, 0, 2, 0], ctx=2, seed=D)
    assert c["x"].shape[0] < 32
    _pos_check(c)


def test_position_bwd_many_rows_per_cta():
    """L > 132 * 8 * 32, so a CTA walks more than 32 rows (here 38).  One sequence of 6000 rows shares a single timestamp:
    its bucket-0 run crosses many CTA boundaries and is flushed by each CTA separately."""
    lengths = [0, 6000, 1, 20000, 0, 9000, 5000, 0]
    L = sum(lengths)
    assert L > 132 * 8 * 32 and (L + 132 * 8 - 1) // (132 * 8) > 32
    c = _pos_case(torch.bfloat16, 256, lengths, targets=[0, 3, 0, 10, 0, 0, 7, 0], ctx=4, pos_rows=4000, same_ts=(1,),
                  seed=6)
    _, bkt, _ = _pos_check(c)
    assert bool((bkt[:6000] == 0).all())


def test_position_bwd_d1025_refused():
    """D = 1025 has no backward kernel: the host refuses it with an error, nothing is launched."""
    lib = _lib()
    L, D = 4, 1025
    g, dseq = torch.zeros(L, D, dtype=torch.bfloat16, device=DEV), torch.zeros(L, D, dtype=torch.bfloat16, device=DEV)
    dpos, dts = torch.zeros(8, D, device=DEV), torch.zeros(8, D, device=DEV)
    idx = torch.zeros(L, dtype=torch.int32, device=DEV)
    rc = lib.lib().hstu_position_embeddings_bwd(g.data_ptr(), dseq.data_ptr(), dpos.data_ptr(), dts.data_ptr(), idx.data_ptr(),
                                                idx.data_ptr(), L, D, 1.0, lib.BF16, _stream())
    with pytest.raises(RuntimeError, match="not supported"):
        lib.check(rc, "position bwd")


# ----------------------------------------------------------------------------------------------------------------------------
# jagged concat / split
# ----------------------------------------------------------------------------------------------------------------------------

# (dtype, D): row bytes divisible by 16 -> 16-byte copies, by 4 -> 4-byte, by 2 -> 2-byte, odd -> 1-byte
COPY_WIDTHS = [(torch.bfloat16, 8, 16), (torch.bfloat16, 6, 4), (torch.float16, 5, 2), (torch.uint8, 7, 1)]
LEN_L = [0, 3, 0, 7, 1, 0, 4]  # empty left sides first, in the middle and last
LEN_R = [2, 0, 0, 5, 9, 1, 0]  # empty right sides; the third entry is empty on both
DENSE_LEN = 4
CTX = 2                        # the l2 wrappers' contextual prefix: right sides of 0 and 1 rows are shorter than it


def _bits(n, D, dtype, g):
    """Random bit patterns (NaN payloads and infinities included for the 16-bit types) as an integer tensor and as `dtype`."""
    if dtype == torch.uint8:
        b = torch.randint(0, 256, (n, D), generator=g, dtype=torch.uint8)
        return b, b
    b = torch.randint(-32768, 32768, (n, D), generator=g, dtype=torch.int16)
    return b, b.view(dtype)


def _dev(t, misalign):
    """t on the GPU, its base pointer one element past an aligned address when misalign."""
    sh = int(misalign)
    buf = torch.empty(t.numel() + sh, dtype=t.dtype, device=DEV)
    buf[sh:] = t.reshape(-1).to(DEV)
    return buf[sh:].view(t.shape)


def _poisoned(shape, dtype, misalign):
    sh = int(misalign)
    if dtype == torch.uint8:
        buf = torch.full((math.prod(shape) + sh,), 0xA5, dtype=dtype, device=DEV)
    else:
        buf = _nan((math.prod(shape) + sh,), dtype)
    return buf[sh:].view(shape)


def _intbits(t):
    return t.cpu() if t.dtype == torch.uint8 else t.cpu().view(torch.int16)


@pytest.mark.parametrize("misalign", [False, True], ids=["aligned", "offset1"])
@pytest.mark.parametrize("mode", ["jagged_jagged", "jagged_dense", "dense_jagged", "l2"])
@pytest.mark.parametrize("dtype,D,width", COPY_WIDTHS, ids=[f"{w}B" for _, _, w in COPY_WIDTHS])
def test_concat_split_bitwise(dtype, D, width, mode, misalign):
    """concat then split through the C ABI into poisoned outputs, compared bit for bit with the oracle's row routing.  The
    copy width is 16 / 4 / 2 / 1 bytes by the row size; a base pointer one element off an aligned address lowers it (16-bit
    types to 2 bytes).  int32 offsets on aligned pointers, int64 on the offset ones.  l2: n_prefix = CTX rows of each right side go in front of the left side (hstu_concat_l2_embeddings)."""
    lib = _lib()
    g = torch.Generator().manual_seed(width * 10 + len(mode) + int(misalign))
    B = len(LEN_L)
    idt = torch.int64 if misalign else torch.int32
    ol = None if mode == "dense_jagged" else offsets_from(LEN_L, dtype=idt)
    orr = None if mode == "jagged_dense" else offsets_from(LEN_R, dtype=idt)
    nl = B * DENSE_LEN if ol is None else int(ol[-1])
    nr = B * DENSE_LEN if orr is None else int(orr[-1])
    npre = CTX if mode == "l2" else 0
    max_seq_len = max((DENSE_LEN if ol is None else a) + (DENSE_LEN if orr is None else b) for a, b in zip(LEN_L, LEN_R))
    lb, lv = _bits(nl, D, dtype, g)
    rb, rv = _bits(nr, D, dtype, g)
    ref = O.concat_2D_jagged(lb, rb, DENSE_LEN, DENSE_LEN, ol, orr, npre)
    left, right = _dev(lv, misalign), _dev(rv, misalign)
    out = _poisoned((nl + nr, D), dtype, misalign)
    pl = None if ol is None else ol.to(DEV)
    pr = None if orr is None else orr.to(DEV)
    esz = torch.empty(0, dtype=dtype).element_size()
    i64 = int(idt == torch.int64)
    lib.check(lib.lib().hstu_jagged_concat(left.data_ptr(), right.data_ptr(), out.data_ptr(), lib.ptr(pl), lib.ptr(pr), i64, B,
                                           DENSE_LEN, DENSE_LEN, npre, D, esz, max_seq_len, _stream()), "concat")
    sl, sr = _poisoned((nl, D), dtype, misalign), _poisoned((nr, D), dtype, misalign)
    lib.check(lib.lib().hstu_jagged_split(out.data_ptr(), sl.data_ptr(), sr.data_ptr(), lib.ptr(pl), lib.ptr(pr), i64, B,
                                          DENSE_LEN, DENSE_LEN, npre, D, esz, max_seq_len, _stream()), "split")
    torch.cuda.synchronize()
    got = _intbits(out)
    bad = (got != ref).any(-1).nonzero()
    assert bad.numel() == 0, f"concat row {int(bad[0]) if bad.numel() else -1} differs from the oracle"
    for name, a, r in (("split left", _intbits(sl), lb), ("split right", _intbits(sr), rb)):
        bad = (a != r).any(-1).nonzero()
        assert bad.numel() == 0, f"{name} row {int(bad[0])} differs from the input"


def test_concat_split_autograd_mixed_offsets():
    """The facades with int32 left and int64 right offsets: concat_2D_jagged, its backward (split), split_2D_jagged and its
    backward (concat), and the l2 wrappers with a contextual prefix, all bit for bit against the oracle."""
    from generative_recommenders_b200.common import HammerKernel
    from generative_recommenders_b200.ops import jagged_tensors as J

    g = torch.Generator().manual_seed(11)
    D = 6
    ol, orr = offsets_from(LEN_L, dtype=torch.int32), offsets_from(LEN_R, dtype=torch.int64)
    nl, nr = int(ol[-1]), int(orr[-1])
    max_l, max_r = max(LEN_L), max(LEN_R)
    lb, lv = _bits(nl, D, torch.bfloat16, g)
    rb, rv = _bits(nr, D, torch.bfloat16, g)
    db, dv = _bits(nl + nr, D, torch.bfloat16, g)
    K = HammerKernel.CUDA
    for npre in (0, CTX):
        ref = O.concat_2D_jagged(lb, rb, None, None, ol, orr, npre)
        ref_dl, ref_dr = O.split_2D_jagged(db, None, None, ol, orr, npre)
        xl, xr = lv.to(DEV).requires_grad_(), rv.to(DEV).requires_grad_()
        if npre:
            out = J.hstu_concat_l2_embeddings(max_l, xl, ol.to(DEV), max_r, xr, orr.to(DEV), npre, kernel=K)
        else:
            out = J.concat_2D_jagged(max_l + max_r, xl, xr, max_l, max_r, ol.to(DEV), orr.to(DEV), kernel=K)
        out.backward(dv.to(DEV))
        assert torch.equal(_intbits(out.detach()), ref), f"concat (n_prefix {npre})"
        assert torch.equal(_intbits(xl.grad), ref_dl) and torch.equal(_intbits(xr.grad), ref_dr), f"concat backward ({npre})"
        x = dv.to(DEV).requires_grad_()
        if npre:
            sl, sr = J.hstu_split_l2_embeddings(max_l + max_r, x, ol.to(DEV), orr.to(DEV), npre, kernel=K)
        else:
            sl, sr = J.split_2D_jagged(max_l + max_r, x, None, None, max_l, max_r, ol.to(DEV), orr.to(DEV), kernel=K)
        assert torch.equal(_intbits(sl.detach()), ref_dl) and torch.equal(_intbits(sr.detach()), ref_dr), f"split ({npre})"
        torch.autograd.backward([sl, sr], [lv.to(DEV), rv.to(DEV)])
        assert torch.equal(_intbits(x.grad), ref), f"split backward (n_prefix {npre})"
