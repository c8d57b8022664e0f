"""The attention parity checks have teeth (CPU, oracle only).  Each test feeds a check a result that is wrong in one way a
kernel could be wrong, and shows where the check catches it:

- a kernel without the nonlinearity of tanh (tanh x = x, so silu is its quadratic part) passes the whole-tensor bound at the
  input scale of the older parity tests, and fails it at every scale of the sweep in test_gpu_attention_numerics.py from
  rms(alpha S) = 1 on;
- a 1 % error in one 64-row tile of one sequence passes the whole-tensor bound and fails the per-segment one, which names
  the tile;
- NaN in the last rows of one sequence, as a tile that crosses a sequence end would leave them, trips the isolation check.
"""
import pytest
import torch

import test_gpu_attention_numerics as N
from oracle import hstu_oracle as O
from util import assert_rel, assert_rel_segments, normal_case, offsets_from

NAMES = ("out", "dq", "dk", "dv")


def _oracle(case, n, alpha, dtype=torch.float64):
    q, k, v, dout, off, nt = case
    out = O.hstu_mha_fwd(n, alpha, q, k, v, off, nt, dtype=dtype)
    return (out,) + O.hstu_mha_bwd(n, alpha, dout, q, k, v, off, nt, dtype=dtype)


def _oracle_tanh_linear(monkeypatch, case, n, alpha):
    """The oracle with tanh x replaced by x in sigmoid(2x) = (1 + tanh x) / 2: P and dS keep their exact form up to x^2."""
    with monkeypatch.context() as m:
        m.setattr(torch, "sigmoid", lambda s: 0.5 + 0.25 * s)
        m.setattr(torch.nn.functional, "silu", lambda s: s * (0.5 + 0.25 * s))
        return _oracle(case, n, alpha)


def _uniform_case(lengths, targets, H, d, scale, seed):
    """The input distribution of the older parity tests: q, k, v ~ U(-scale, scale) (test_gpu_parity_fullsize.py)."""
    g = torch.Generator().manual_seed(seed)
    off = offsets_from(lengths)
    L = int(off[-1])
    q, k, v = (torch.empty(L, H, d).uniform_(-scale, scale, generator=g).to(torch.bfloat16) for _ in range(3))
    dout = torch.randn(L, H, d, generator=g).to(torch.bfloat16)
    return q, k, v, dout, off, torch.tensor(targets)


def test_linear_tanh_passes_at_the_old_input_scale(monkeypatch):
    case = _uniform_case([512, 300], [3, 9], 2, 32, 0.5, 7)
    n, alpha = 512, 32**-0.5
    exact, lin = _oracle(case, n, alpha), _oracle_tanh_linear(monkeypatch, case, n, alpha)
    for name, a, r in zip(NAMES, lin, exact):
        assert_rel(a.to(torch.bfloat16), r, f"tanh x = x, U(-0.5, 0.5): {name}")


@pytest.mark.parametrize("sigma", [s for s in N.SIGMAS if s * s >= 1])
def test_linear_tanh_fails_the_sweep(monkeypatch, sigma):
    case = N._sweep_case(sigma, 32, torch.bfloat16)
    alpha = 32**-0.5
    exact, lin = _oracle(case, N.SWEEP_N, alpha), _oracle_tanh_linear(monkeypatch, case, N.SWEEP_N, alpha)
    for name, a, r in zip(NAMES, lin, exact):
        with pytest.raises(AssertionError, match="rel-L2 error"):
            assert_rel(a.to(torch.bfloat16), r, f"tanh x = x, rms(alpha S) = {sigma**2:g}: {name}")


def test_one_bad_tile_passes_globally_and_fails_its_segment():
    lengths, targets, n = [1024, 77, 0, 640, 1, 255, 256, 257], [3, 0, 0, 20, 1, 0, 9, 2], 1024  # the full-size d = 32 case
    case = _uniform_case(lengths, targets, 3, 32, 0.5, 4274)
    ref = _oracle(case, n, 32**-0.5, dtype=torch.float32)
    s = int(case[4][3])  # sequence 3, head 1, rows [320, 384)
    for name, r in zip(NAMES, ref):
        bad = r.clone()
        bad[s + 320:s + 384, 1] *= 1.01
        bad = bad.to(torch.bfloat16)
        assert_rel(bad, r, f"one bad tile: {name}")
        assert_rel_segments(r.to(torch.bfloat16), r, case[4], n, f"no bad tile: {name}")
        with pytest.raises(AssertionError, match=r"sequence 3 head 1 rows \[320, 384\)"):
            assert_rel_segments(bad, r, case[4], n, f"one bad tile: {name}")


def test_segments_check_rows_past_max_seq_len():
    case = normal_case([300, 77], None, 2, 32, 1.0, torch.bfloat16, 5)
    ref = _oracle(case, 256, 32**-0.5, dtype=torch.float32)[0]
    got = ref.to(torch.bfloat16)
    assert_rel_segments(got, ref, case[4], 256, "rows past max_seq_len zero")
    got[299, 1, 5] = 1e-3
    with pytest.raises(AssertionError, match="sequence 0 row 299"):
        assert_rel_segments(got, ref, case[4], 256, "rows past max_seq_len not zero")


@pytest.mark.parametrize("rows", [1, 13])
def test_isolation_check_trips_on_a_poisoned_sequence_end(rows):
    """NaN where the last rows of sequence 1 (77 rows: its second key / query tile crosses into the poisoned sequence 2)
    would get it from the dragged-in rows."""
    case = normal_case(N.ISO_LENGTHS, N.ISO_TARGETS, 2, 32, 0.7, torch.bfloat16, 332)
    ref = _oracle(case, N.ISO_N, 32**-0.5, dtype=torch.float32)
    got = tuple(r.to(torch.bfloat16) for r in ref)
    N._check_isolated(got, got, ref, "oracle")
    e = int(case[4][2])
    for i, name in enumerate(NAMES):
        bad = list(got)
        bad[i] = bad[i].clone()
        bad[i][e - rows:e] = float("nan")
        with pytest.raises(AssertionError, match=f"{name}: sequence 1 row {77 - rows} is not finite"):
            N._check_isolated(tuple(bad), got, ref, "oracle")
