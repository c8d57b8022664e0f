"""The fp8 (e4m3) attention forward when the value head is wider than the query / key head (dqk < dv; DESIGN.md 3.5, "two
widths") on the GPU: attn_fwd_e4m3_mixed_wgmma_kernel for every pair, against the fp64 oracle on the dequantised values, on
the whole tensor (assert_rel) and per 64-row segment (assert_rel_segments), at the full bf16 bound.  Every mask option with
int32 offsets, lengths around the 64 / 128 tiles with exact zeros past max_seq_len and empty sequences, the rms(alpha S)
sweep (the P exponent bound reduces over dqk), tiny descales, the bitwise identities of the descales, NaN isolation, strided
views of one [L, H, 2 dqk + dv] buffer and the registered op."""
import pytest
import torch

from oracle import hstu_oracle as O
from test_gpu_attention_deterministic import _kernels_of
from test_gpu_attention_fp8 import FP8, check_parity, dequant, quantize, run
from util import assert_finite_rows, assert_rel, assert_rel_segments, offsets_from

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
PAIRS = [(32, 64), (32, 128), (32, 256), (64, 128), (64, 256), (128, 256)]
KERNEL = "attn_fwd_e4m3_mixed_wgmma_kernel"


def _case(lengths, targets, H, dqk, dv, sigma, seed, i32=False):
    """fp32 q, k ~ N(0, sigma^2) [L, H, dqk] and v ~ N(0, 1) [L, H, dv]; with alpha = 1/sqrt(dqk), rms(alpha S) = sigma^2."""
    g = torch.Generator().manual_seed(seed)
    idt = torch.int32 if i32 else torch.int64
    off = offsets_from(lengths, dtype=idt)
    L = int(off[-1])
    q, k = (sigma * torch.randn(L, H, dqk, generator=g) for _ in range(2))
    v = torch.randn(L, H, dv, generator=g)
    return q, k, v, off, None if targets is None else torch.tensor(targets, dtype=idt)


@pytest.mark.parametrize("dqk,dv", PAIRS)
def test_fp8_mixed_dims_run_their_kernel(dqk, dv):
    q, k, v, off, nt = _case([300, 0, 129], [3, 0, 1], 2, dqk, dv, 1.0, dqk + dv)
    res = {}
    names = _kernels_of(lambda: res.setdefault("out", check_parity(320, dqk**-0.5, q, k, v, off, nt, f"({dqk}, {dv})")))
    assert any(KERNEL in n for n in names), sorted(names)
    assert not any("attn_fwd_e4m3_wgmma_kernel" in n for n in names), sorted(names)
    assert tuple(res["out"].shape) == (q.shape[0], 2, dv)


MASKS = {
    "causal": dict(),
    "window_min_full": dict(max_attn_len=100, min_full_attn_seq_len=40),
    "contextual": dict(contextual_seq_len=17),
    "window_contextual_targets": dict(max_attn_len=64, contextual_seq_len=5, min_full_attn_seq_len=0),
}


@pytest.mark.parametrize("dqk,dv", PAIRS)
@pytest.mark.parametrize("mask", sorted(MASKS))
@pytest.mark.parametrize("i32", [False, True])
def test_fp8_mixed_dims_mask_options(dqk, dv, mask, i32):
    lengths = [700, 0, 260, 1100, 3]  # the first and fourth run past max_seq_len = 512: their rows >= 512 must be zero
    q, k, v, off, nt = _case(lengths, [9, 0, 4, 30, 1], 2, dqk, dv, 1.0, 5 + dqk + dv, i32=i32)
    out = check_parity(512, dqk**-0.5, q, k, v, off, nt, f"({dqk}, {dv}) {mask} i32={i32}", **MASKS[mask])
    assert (out[512:700] == 0).all() and (out[700 + 260 + 512:700 + 260 + 1100] == 0).all()


@pytest.mark.parametrize("dqk,dv", PAIRS)
def test_fp8_mixed_dims_lengths_around_the_tiles(dqk, dv):
    """Lengths 0, 1, 63, 64, 65, 127, 128, 129, one of max_seq_len and one past it: rows past max_seq_len are exact zeros
    (the output starts as NaN)."""
    lengths, targets, N = [640, 0, 1, 63, 64, 65, 127, 128, 129, 700], [9, 0, 1, 3, 0, 5, 1, 2, 7, 4], 640
    q, k, v, off, nt = _case(lengths, targets, 2, dqk, dv, 0.8, 77 + dqk + dv, i32=True)
    (q8, qd), (k8, kd), (v8, vd) = (quantize(t, off) for t in (q, k, v))
    out = torch.full((q.shape[0], 2, dv), float("nan"), device=DEV, dtype=torch.bfloat16)
    run(N, dqk**-0.5, q8, k8, v8, off, (qd, kd, vd), nt, out=out)
    out = out.cpu()
    ref = O.hstu_mha_fwd(N, dqk**-0.5, dequant(q8, qd, off), dequant(k8, kd, off), dequant(v8, vd, off), off.long(),
                         nt.long(), dtype=torch.float64)
    assert_rel(out, ref, f"lengths ({dqk}, {dv})")
    assert_rel_segments(out, ref, off, N, f"lengths ({dqk}, {dv})")
    last = slice(int(off[-2]) + N, int(off[-1]))
    assert torch.equal(out[last].float(), torch.zeros_like(out[last].float())), "rows past max_seq_len"


@pytest.mark.parametrize("dqk,dv", PAIRS)
def test_fp8_mixed_dims_empty_batch(dqk, dv):
    q, k, v, off, _ = _case([0, 0], None, 2, dqk, dv, 1.0, 1)
    (q8, qd), (k8, kd), (v8, vd) = (quantize(t, off) for t in (q, k, v))
    out = run(64, dqk**-0.5, q8, k8, v8, off, (qd, kd, vd))
    assert tuple(out.shape) == (0, 2, dv)


@pytest.mark.parametrize("dqk,dv", [(32, 256), (128, 256)])
@pytest.mark.parametrize("rms", [0.09, 1.0, 2.25, 4.0])
def test_fp8_mixed_dims_across_score_scales(dqk, dv, rms):
    """rms(alpha S) from 0.09 to 4: P' = 2^p P stays inside fp16 and keeps its precision at every scale.  p is bounded by
    the dqk terms of S; a bound taken over dv would scale P' down by 2^3 at (32, 256)."""
    q, k, v, off, nt = _case([1500, 731, 260, 1], [7, 3, 0, 1], 2, dqk, dv, rms**0.5, 2024 + dqk + int(10 * rms))
    check_parity(1536, dqk**-0.5, q, k, v, off, nt, f"({dqk}, {dv}) rms(alpha S)={rms}")


@pytest.mark.parametrize("dqk,dv", PAIRS)
def test_fp8_mixed_dims_tiny_descales_keep_full_precision(dqk, dv):
    # qd, kd scaled by 2^-66 each: alpha/2 qd kd is an fp32 subnormal, yet the logits keep full precision; vd 2^120 brings
    # the output back into bf16's normal range
    q, k, v, off, nt = _case([300, 129, 511], [3, 0, 7], 2, dqk, dv, 1.0, 31 + dv)
    (q8, qd), (k8, kd), (v8, vd) = (quantize(t, off) for t in (q, k, v))
    qd, kd, vd = qd * 2.0**-66, kd * 2.0**-66, vd * 2.0**120
    N, alpha = 512, dqk**-0.5
    out = run(N, alpha, q8, k8, v8, off, (qd, kd, vd), nt)
    ref = O.hstu_mha_fwd(N, alpha, dequant(q8, qd, off), dequant(k8, kd, off), dequant(v8, vd, off), off, nt,
                         dtype=torch.float64)
    assert torch.isfinite(out.float()).all()
    assert_rel(out, ref, f"tiny q / k descales ({dqk}, {dv})")
    assert_rel_segments(out, ref, off, N, f"tiny q / k descales ({dqk}, {dv})")


def _fixed(dqk, dv, lengths=(300, 129, 511), seed=13):
    q, k, v, off, _ = _case(list(lengths), None, 2, dqk, dv, 1.0, seed)
    (q8, qd), (k8, kd), (v8, vd) = (quantize(t, off) for t in (q, k, v))
    return q8, k8, v8, qd, kd, vd, off


def _bits(x):
    return x.view(torch.int16)


@pytest.mark.parametrize("dqk,dv", PAIRS)
def test_fp8_mixed_dims_none_descales_equal_ones_bitwise(dqk, dv):
    q8, k8, v8, qd, _, _, off = _fixed(dqk, dv)
    ones = torch.ones_like(qd)
    a = run(512, 0.125, q8, k8, v8, off, None)
    b = run(512, 0.125, q8, k8, v8, off, (ones, ones, ones))
    c = run(512, 0.125, q8, k8, v8, off, (None, ones, None))
    assert torch.equal(_bits(a), _bits(b)) and torch.equal(_bits(a), _bits(c))


@pytest.mark.parametrize("dqk,dv", PAIRS)
@pytest.mark.parametrize("e", [3, -5])
def test_fp8_mixed_dims_power_of_two_descale_changes_act_bitwise(dqk, dv, e):
    q8, k8, v8, qd, kd, vd, off = _fixed(dqk, dv)
    alpha, s = dqk**-0.5, 2.0**e
    out = run(512, alpha, q8, k8, v8, off, (qd, kd, vd))
    o1 = run(512, alpha, q8, k8, v8, off, (qd * s, kd / s, vd))
    assert torch.equal(_bits(o1), _bits(out))
    o2 = run(512, alpha, q8, k8, v8, off, (qd, kd, vd * s))
    assert torch.equal(_bits(o2), _bits(out * s))


@pytest.mark.parametrize("dqk,dv", [(32, 64), (64, 256), (128, 256)])
def test_fp8_mixed_dims_bad_values_stay_in_their_sequence_and_head(dqk, dv):
    N = 400
    lengths = [300, 500, 129, 260]  # the second runs past max_seq_len
    q8, k8, v8, qd, kd, vd, off = _fixed(dqk, dv, lengths, seed=21)
    o = [int(t) for t in off.tolist()]
    nan = torch.tensor([0x7F], dtype=torch.uint8).view(FP8)[0]  # the e4m3fn NaN
    poisoned = [(q8.clone(), k8.clone(), v8.clone(), qd.clone()) for _ in range(2)]
    # NaN in q, k and v inside sequence 0 (a column past dqk in v); NaN in every input past max_seq_len of sequence 1
    for val, (a, b_, c, _) in zip((nan, torch.zeros(1, dtype=FP8)[0]), poisoned):
        a[o[0] + 37, 1, 5] = val
        b_[o[0] + 37, 1, 5] = val
        c[o[0] + 37, 1, dv - 3] = val
        for t in (a, b_, c):
            t[o[1] + N: o[2]] = val
    # and a NaN descale of (sequence 2, head 0)
    poisoned[0][3][2, 0] = float("nan")
    poisoned[1][3][2, 0] = 0.0
    bad = run(N, 0.125, *poisoned[0][:3], off, (poisoned[0][3], kd, vd))
    zero = run(N, 0.125, *poisoned[1][:3], off, (poisoned[1][3], kd, vd))
    assert not torch.isfinite(bad[o[0]:o[1], 1].float()).all() and not torch.isfinite(bad[o[2]:o[3], 0].float()).all()
    keep = torch.ones(bad.shape[:2], dtype=torch.bool)
    keep[o[0]:o[1], 1] = False
    keep[o[2]:o[3], 0] = False
    assert torch.isfinite(bad[keep].float()).all()
    assert torch.equal(_bits(bad[keep]), _bits(zero[keep]))
    assert (bad[o[1] + N:o[2]] == 0).all()
    assert_finite_rows(bad[:, 0:1], off, {2}, "head 0 outside the NaN descale")


@pytest.mark.parametrize("dqk,dv", PAIRS)
def test_fp8_mixed_dims_strided_views_of_one_buffer(dqk, dv):
    """q, k, v as strided e4m3 views of one [L, H, 2 dqk + dv] buffer, descales as non-contiguous views, with targets."""
    q, k, v, off, nt = _case([200, 333, 64, 0], [2, 5, 0, 0], 2, dqk, dv, 1.0, 77 + dv, i32=True)
    check_parity(400, dqk**-0.5, q, k, v, off, nt, f"views ({dqk}, {dv})", views=True)


def test_fp8_mixed_dims_registered_op_equals_the_raw_entry_bitwise():
    from generative_recommenders_b200 import torch_ops

    torch_ops.register()
    dqk, dv, N, alpha = 128, 256, 512, 128**-0.5
    q8, k8, v8, qd, kd, vd, off = _fixed(dqk, dv)
    raw = run(N, alpha, q8, k8, v8, off, (qd, kd, vd))
    args = [t.to(DEV) for t in (q8, k8, v8)]
    off32 = off.to(DEV, torch.int32)
    a = torch.ops.hstu.hstu_mha_fwd(N, alpha, *args, off32, True, None, None, 0, 0, 0, qd.to(DEV), kd.to(DEV), vd.to(DEV), 0)
    b = torch.ops.hstu.hstu_mha(N, alpha, *args, off32, True, None, None, 0, 0, 0, qd.to(DEV), kd.to(DEV), vd.to(DEV), False,
                                False, 0)
    for x in (a, b):
        assert x.dtype == torch.bfloat16 and tuple(x.shape) == (q8.shape[0], 2, dv)
        assert torch.equal(_bits(x.cpu()), _bits(raw))
