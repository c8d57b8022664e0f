"""The checks of the research-path GPU tests (test_gpu_rel_bias_attention.py, test_gpu_rowwise_general.py) catch what they are
meant to catch: they are applied here to the fp64 oracle's own results with one deliberate defect each -- gradient mass moved
by one diagonal inside a cross-tile band, one time bucket shifted, one nonzero j > i diagonal, one flipped dropout decision --
and must fail, while the unmodified results pass.  Also pins the distance of the bf16-staged research-block oracle from fp64,
from which the bf16 block test derives its gradient bounds."""
import pytest
import torch

from oracle import hstu_oracle as O
from util import (TOL, assert_pos_bands, assert_same_zeros, assert_table_entries, assert_zero_from, offsets_from,
                  rel_bias_reference, research_case, research_reference, table_bound)

N = 211


@pytest.fixture(scope="module")
def ref():
    """The ml20m-shaped relative-bias attention (n = 211, d = 32) with position and time bias, in fp64 on bf16 values."""
    g = torch.Generator().manual_seed(0)
    lengths = [211, 0, 65, 1, 150]
    off = offsets_from(lengths)
    L, H, d = int(off[-1]), 2, 32
    q, k = ((d ** -0.25 * torch.randn(L, H, d, generator=g)).to(torch.bfloat16) for _ in range(2))
    v, dout = (torch.randn(L, H, d, generator=g).to(torch.bfloat16) for _ in range(2))
    pos_w = (0.5 * torch.randn(2 * N - 1, generator=g)).to(torch.bfloat16)
    ts_w = (0.5 * torch.randn(17, generator=g)).to(torch.bfloat16)
    ts = torch.randint(0, 3, (len(lengths), N), generator=g).cumsum(1)
    ts = ts + (torch.rand(len(lengths), N, generator=g) < 0.15) * torch.randint(-10**9, 10**9, (len(lengths), N), generator=g)
    r = rel_bias_reference(N, q, k, v, dout, off, pos_w, ts_w, ts)
    r["d"] = d
    return r


def _pos_checks(got, r):
    assert_zero_from(got, N, "dpos_w")
    assert_table_entries(got, r["dpos"], table_bound(r["mass_pos"], r["cnt_pos"], r["d"]), "dpos_w")
    assert_pos_bands(got, r["dpos"], N, TOL[torch.float32], "dpos_w")


def test_unmodified_reference_passes(ref):
    got = ref["dpos"].float()  # the fp64 result stored in fp32: within every bound
    _pos_checks(got, ref)
    assert_table_entries(ref["dts"].float(), ref["dts"], table_bound(ref["mass_ts"], ref["cnt_ts"], ref["d"]), "dts_w")
    assert ref["cnt_ts"][-1] > 0  # the clamped last bucket is fed


@pytest.mark.parametrize("delta", [70, 130, 200])  # cross-tile diagonals i - j = delta >= 64
def test_mass_moved_by_one_diagonal_fails(ref, delta):
    got = ref["dpos"].clone()
    e = N - 1 - delta
    got[e - 1] += got[e]  # the gradient of diagonal delta lands on diagonal delta + 1
    got[e] = 0
    with pytest.raises(AssertionError):
        assert_table_entries(got, ref["dpos"], table_bound(ref["mass_pos"], ref["cnt_pos"], ref["d"]), "dpos_w")
    with pytest.raises(AssertionError):
        assert_pos_bands(got, ref["dpos"], N, TOL[torch.float32], "dpos_w")


def test_shifted_bucket_fails(ref):
    got = ref["dts"].clone()
    lim = table_bound(ref["mass_ts"], ref["cnt_ts"], ref["d"])
    for b in range(got.numel() - 1):
        shifted = got.clone()
        shifted[b + 1] += shifted[b]
        shifted[b] = 0
        if ref["cnt_ts"][b] > 0:
            with pytest.raises(AssertionError):
                assert_table_entries(shifted, ref["dts"], lim, "dts_w")
    dropped_last = got.clone()
    dropped_last[-1] = 0  # a flush that skips the last (clamped) bucket
    with pytest.raises(AssertionError):
        assert_table_entries(dropped_last, ref["dts"], lim, "dts_w")


def test_single_nonzero_above_the_diagonal_fails(ref):
    got = ref["dpos"].clone()
    got[N + 5] = 1e-30
    with pytest.raises(AssertionError):
        assert_zero_from(got, N, "dpos_w")


def test_single_flipped_dropout_element_fails():
    g = torch.Generator().manual_seed(1)
    out = torch.rand(300, 64, generator=g) + 0.5
    out[torch.rand(300, 64, generator=g) < 0.2] = 0
    assert_same_zeros(out, out.clone() * 2, "same pattern")
    for (r, c) in ((0, 0), (123, 45), (299, 63)):
        flipped = out.clone()
        flipped[r, c] = 0 if flipped[r, c] != 0 else 1
        with pytest.raises(AssertionError, match=rf"\({r}, {c}\)"):
            assert_same_zeros(out, flipped, "one flipped element")


@pytest.mark.parametrize("concat_ua", [False, True], ids=["plain", "concat_ua"])
@pytest.mark.parametrize("config", ["ml20m", "amzn_books"])
def test_research_block_staged_oracle_distance(config, concat_ua):
    """How far bf16 storage of the forward activations alone moves the research block's gradients from fp64.  The bf16 GPU
    test allows the kernels twice this distance (measured on the same inputs): measured values 3.5e-3 .. 8.9e-3 (and 0 for the
    o.bias gradient, which the forward does not reach).  Pinned here so that a change of the staged oracle or of the inputs
    that made the derived bounds vacuous (much larger) or unattainable (zero) shows up without a GPU."""
    staged, exact, dist = research_reference(research_case(config, concat_ua))
    for name, d in dist.items():
        if name == "_o.bias":
            assert d == 0.0, (name, d)
        else:
            assert 1e-3 <= d <= 2e-2, (name, d)
    # the forward the staged oracle produces is the fp64 one up to bf16 storage (a few bf16 roundings)
    assert 0 < O.rel_l2(staged["y"], exact["y"]) <= 1e-2
