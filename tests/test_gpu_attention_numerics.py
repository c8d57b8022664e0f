"""GPU parity of the wgmma attention kernels where the other parity tests do not look:

1. Logits of the size a trained model produces.  With q, k drawn from +-0.5 the logits alpha S stay below ~0.1, where
   silu(2x) = x (1 + tanh x) is x + x^2 to 2e-5: such tests cannot see the tanh.approx error, nor the cancellation of the
   backward's 1 + g2 = 1 + t + h (1 - t^2) near |t| = 1.  Here q, k ~ N(0, sigma^2), so rms(alpha S) = sigma^2 up to 4.
   The generic kernels (exp / divide sigmoid) run at the largest scale as a control.
2. A long d = 32 sequence whose contextual prefix alone wraps the 4-stage query-tile ring of the dK / dV kernel before its
   causal range starts, with a window, a full-attention tail and targets; int32 and int64 offsets.
3. Sequence isolation.  The TMA box of a tile that crosses a sequence end loads rows of the next sequence (or rows past
   max_seq_len of the same one); P and dS are zero there, but the rows still enter an MMA as its other factor
   (O += P V, dQ += dS K, dV += P^T dO, dK += dS^T Q), and 0 * NaN = NaN.  Non-finite rows must reach no other sequence.

Every comparison is made on the whole tensor (assert_rel) and per 64-row segment (assert_rel_segments) against the oracle
evaluated in fp64.  The sweep's inputs are shared with tests/test_attention_numerics_cpu.py, which shows that the sweep
fails a kernel without the nonlinearity of tanh.
"""
import ctypes as C

import pytest
import torch

from oracle import hstu_oracle as O
from util import assert_finite_rows, assert_rel, assert_rel_segments, normal_case, offsets_from

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda")

# q, k ~ N(0, sigma^2) with alpha = 1/sqrt(d): rms(alpha S) = sigma^2 = 0.09, 1, 2.25, 4
SIGMAS = [0.3, 1.0, 1.5, 2.0]
SWEEP = dict(lengths=[1500, 731, 260, 1], targets=[7, 3, 0, 1], H=2)
SWEEP_N = 1536


def _mods():
    from generative_recommenders_b200 import _lib
    from generative_recommenders_b200.common import HammerKernel
    from generative_recommenders_b200.ops.hstu_attention import _fill_common, hstu_mha

    return _lib, HammerKernel, hstu_mha, _fill_common


def _assert_auto_selects_wgmma(N, alpha, q, k, v, off, nt, win=0, ctx=0, min_full=0):
    """AUTO dispatches this problem to the wgmma kernels, so forcing them tests what a user runs."""
    _lib, _, _, fill = _mods()
    qd, kd, vd, offd = q.to(DEV), k.to(DEV), v.to(DEV), off.to(DEV)
    ntd = None if nt is None else nt.to(DEV)
    p = _lib.AttnParams()
    fill(p, N, alpha, qd, kd, vd, offd, ntd, win, ctx, min_full, _lib.IMPL_AUTO)
    out = torch.empty_like(vd)
    p.out, p.o_row_stride, p.o_head_stride = out.data_ptr(), out.stride(0), out.stride(1)
    assert _lib.lib().hstu_attn_select_impl(C.byref(p), 0) == _lib.IMPL_UMMA


def _run(impl, N, alpha, q, k, v, dout, off, nt, win=0, ctx=0, min_full=0, bwd=True):
    _lib, HK, hstu_mha, _ = _mods()
    qd, kd, vd = (t.to(DEV).requires_grad_(bwd) for t in (q, k, v))
    out = hstu_mha(N, alpha, qd, kd, vd, off.to(DEV), num_targets=None if nt is None else nt.to(DEV), max_attn_len=win,
                   contextual_seq_len=ctx, min_full_attn_seq_len=min_full, kernel=HK.CUDA, impl=impl)
    if not bwd:
        return out.detach(), None, None, None
    out.backward(dout.to(DEV))
    torch.cuda.synchronize()
    return out.detach(), qd.grad, kd.grad, vd.grad


def _oracle(N, alpha, q, k, v, dout, off, nt, win=0, ctx=0, min_full=0, bwd=True):
    kw = dict(num_targets=nt, max_attn_len=win, contextual_seq_len=ctx, min_full_attn_seq_len=min_full, dtype=torch.float64)
    out = O.hstu_mha_fwd(N, alpha, q, k, v, off, **kw)
    return (out,) + (O.hstu_mha_bwd(N, alpha, dout, q, k, v, off, **kw) if bwd else (None, None, None))


def _compare(got, ref, off, N, tag):
    for name, a, r in zip(("out", "dq", "dk", "dv"), got, ref):
        if a is None:
            continue
        assert_rel(a, r, f"{tag} {name}")
        assert_rel_segments(a, r, off, N, f"{tag} {name}")


def _sweep_case(sigma, d, dtype):
    return normal_case(SWEEP["lengths"], SWEEP["targets"], SWEEP["H"], d, sigma, dtype, 2024 + d)


@pytest.mark.parametrize("sigma", SIGMAS)
@pytest.mark.parametrize("d", [32, 64, 128, 256])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_wgmma_vs_oracle_across_score_scales(sigma, d, dtype):
    """Forward at d = 32..256, backward at d = 32 (dK / dV + dQ kernels) and d = 64 / 128 (fused kernel)."""
    _lib = _mods()[0]
    q, k, v, dout, off, nt = _sweep_case(sigma, d, dtype)
    alpha, bwd = d**-0.5, d <= 128
    _assert_auto_selects_wgmma(SWEEP_N, alpha, q, k, v, off, nt)
    got = _run(_lib.IMPL_UMMA, SWEEP_N, alpha, q, k, v, dout, off, nt, bwd=bwd)
    ref = _oracle(SWEEP_N, alpha, q, k, v, dout, off, nt, bwd=bwd)
    _compare(got, ref, off, SWEEP_N, f"wgmma d={d} {dtype} rms(alpha S)={sigma**2:g}")


@pytest.mark.parametrize("d", [32, 64, 128])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_wgmma_vs_oracle_large_scores_window_and_context(d, dtype):
    """The largest scale with a window, a contextual prefix and targets (the per-element mask on most tiles)."""
    _lib = _mods()[0]
    N, win, ctx = 1280, 150, 37
    q, k, v, dout, off, nt = normal_case([1280, 517, 300, 70], [9, 0, 4, 2], 2, d, SIGMAS[-1], dtype, 77 + d)
    alpha = d**-0.5
    _assert_auto_selects_wgmma(N, alpha, q, k, v, off, nt, win, ctx)
    got = _run(_lib.IMPL_UMMA, N, alpha, q, k, v, dout, off, nt, win, ctx)
    ref = _oracle(N, alpha, q, k, v, dout, off, nt, win, ctx)
    _compare(got, ref, off, N, f"wgmma d={d} {dtype} window + context")


@pytest.mark.parametrize("d", [32, 64, 128, 256])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_generic_vs_oracle_at_the_largest_score_scale(d, dtype):
    """Control: the generic kernels form the sigmoid from exp and a divide.  If they meet the bound on the same inputs where a
    wgmma kernel does not, the fault is the kernel's, not the oracle's or the tolerance's."""
    _lib = _mods()[0]
    q, k, v, dout, off, nt = _sweep_case(SIGMAS[-1], d, dtype)
    alpha = d**-0.5
    got = _run(_lib.IMPL_GENERIC, SWEEP_N, alpha, q, k, v, dout, off, nt)
    ref = _oracle(SWEEP_N, alpha, q, k, v, dout, off, nt)
    _compare(got, ref, off, SWEEP_N, f"generic d={d} {dtype} rms(alpha S)={SIGMAS[-1]**2:g}")


@pytest.mark.parametrize("dtype,i32", [(torch.bfloat16, True), (torch.float16, False)])
def test_wgmma_d32_long_sequence_with_context_window_and_targets(dtype, i32):
    """d = 32 at 4096 rows: a contextual prefix of 300 rows makes the dK / dV kernel walk A = 5 prefix query tiles, more than
    its 4 ring stages, before the causal range of every key tile from 384 on; window 500 with a 256-row full-attention
    tail; targets."""
    _lib = _mods()[0]
    d, N, win, ctx, min_full = 32, 4096, 500, 300, 256
    q, k, v, dout, off, nt = normal_case([4096, 1000, 333, 650], [20, 5, 0, 1], 2, d, 1.0, dtype, 4096, i32=i32)
    alpha = d**-0.5
    _assert_auto_selects_wgmma(N, alpha, q, k, v, off, nt, win, ctx, min_full)
    got = _run(_lib.IMPL_UMMA, N, alpha, q, k, v, dout, off, nt, win, ctx, min_full)
    ref = _oracle(N, alpha, q, k, v, dout, off, nt, win, ctx, min_full)
    _compare(got, ref, off, N, f"wgmma d=32 long {dtype} int{32 if i32 else 64}")


ISO_LENGTHS, ISO_N, ISO_TARGETS = [300, 77, 190, 513], 400, [5, 2, 0, 9]
ISO_POISONED = 2  # sequence whose rows hold NaN / Inf; rows >= ISO_N of sequence 3 as well


def _poison(t, value, seed):
    """Copy of t with the rows of sequence ISO_POISONED and the rows past ISO_N of the last sequence set to `value`
    ("inf": +-Inf with random signs)."""
    off = offsets_from(ISO_LENGTHS)
    t = t.clone()
    rows = torch.cat([torch.arange(int(off[ISO_POISONED]), int(off[ISO_POISONED + 1])),
                      torch.arange(int(off[3]) + ISO_N, int(off[4]))])
    if value == "inf":
        sign = torch.randn(len(rows), *t.shape[1:], generator=torch.Generator().manual_seed(seed)).sign()
        t[rows] = (sign * float("inf")).to(t.dtype)
    else:
        t[rows] = float(value)
    return t


def _drop_poisoned(t):
    off = offsets_from(ISO_LENGTHS)
    keep = torch.cat([torch.arange(int(off[b]), int(off[b + 1])) for b in range(len(ISO_LENGTHS)) if b != ISO_POISONED])
    return t.detach().cpu()[keep]


@pytest.mark.parametrize("d", [32, 64, 128, 256])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("value", ["nan", "inf"])
@pytest.mark.parametrize("impl", ["wgmma", "generic"])
def test_non_finite_rows_stay_in_their_sequence(d, dtype, value, impl):
    """q, k, v and dO of one sequence (and the rows past max_seq_len of another) hold NaN or +-Inf.  Every other sequence's
    out, dq, dk and dv are finite, match the oracle, and are bitwise those of a run whose poisoned rows hold zeros (the
    fused d = 64 / 128 backward accumulates dQ with atomics, so its dq is held to the oracle bound only).  The truncated
    sequence's rows past max_seq_len are zero.  d = 256: forward only (its backward runs on the generic kernels)."""
    _lib = _mods()[0]
    q, k, v, dout, off, nt = normal_case(ISO_LENGTHS, ISO_TARGETS, 2, d, 0.7, dtype, 300 + d)
    alpha, bwd = d**-0.5, d <= 128 or impl == "generic"
    code = _lib.IMPL_UMMA if impl == "wgmma" else _lib.IMPL_GENERIC
    if impl == "wgmma":
        _assert_auto_selects_wgmma(ISO_N, alpha, q, k, v, off, nt)
    clean = [_poison(t, 0.0, 0) for t in (q, k, v, dout)]
    dirty = [_poison(t, value, i) for i, t in enumerate((q, k, v, dout))]
    got = _run(code, ISO_N, alpha, *dirty, off, nt, bwd=bwd)
    base = _run(code, ISO_N, alpha, *clean, off, nt, bwd=bwd)
    ref = _oracle(ISO_N, alpha, *clean, off, nt, bwd=bwd)
    _check_isolated(got, base, ref, f"{impl} d={d} {dtype} {value}", dq_atomics=impl == "wgmma" and d in (64, 128))


def _check_isolated(got, base, ref, tag, dq_atomics=False):
    """The checks of test_non_finite_rows_stay_in_their_sequence on (out, dq, dk, dv) of the poisoned run `got`, the run with
    zeros in the poisoned rows `base` and the oracle `ref` (None entries are skipped)."""
    off = offsets_from(ISO_LENGTHS)
    kept_off = offsets_from([n for b, n in enumerate(ISO_LENGTHS) if b != ISO_POISONED])
    for name, a, a0, r in zip(("out", "dq", "dk", "dv"), got, base, ref):
        if a is None:
            continue
        assert_finite_rows(a, off, {ISO_POISONED}, f"{tag} {name}")
        a, a0, r = _drop_poisoned(a), _drop_poisoned(a0), _drop_poisoned(r)
        if not (dq_atomics and name == "dq"):
            assert torch.equal(a, a0), f"{tag} {name}: differs from the run whose poisoned rows hold zeros"
        assert_rel(a, r, f"{tag} {name}")
        assert_rel_segments(a, r, kept_off, ISO_N, f"{tag} {name}")
