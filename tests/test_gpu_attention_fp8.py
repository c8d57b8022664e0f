"""The fp8 (e4m3) attention forward (`hstu_attn_fwd_fp8`, DESIGN.md 3.5) on the GPU: parity with the fp64 oracle on the
dequantised values at the bf16 bound, every mask option, strided views, isolation of bad values, and bitwise identities of
the descales."""
import pytest
import torch

from oracle import hstu_oracle as O
from util import assert_finite_rows, assert_rel, assert_rel_segments, normal_case

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
FP8 = torch.float8_e4m3fn


def quantize(x, off):
    """Per (sequence, head) e4m3 quantisation: descale = amax / 448 (fp32, not a power of two), x8 = e4m3(x / descale).
    Returns (x8 [L, H, d], descale [B, H])."""
    o = [int(t) for t in off.tolist()]
    x = x.float()
    ds = torch.ones(len(o) - 1, x.shape[1])
    x8 = torch.zeros(x.shape, dtype=FP8)
    for b in range(len(o) - 1):
        s, e = o[b], o[b + 1]
        if e > s:
            amax = x[s:e].abs().amax(dim=(0, 2))
            ds[b] = torch.where(amax > 0, amax / 448.0, torch.ones_like(amax))
            x8[s:e] = (x[s:e] / ds[b][None, :, None]).clamp(-448, 448).to(FP8)
    return x8, ds


def dequant(x8, ds, off):
    o = [int(t) for t in off.tolist()]
    x = x8.double()
    for b in range(len(o) - 1):
        x[o[b]:o[b + 1]] *= ds[b].double()[None, :, None]
    return x


def run(N, alpha, q8, k8, v8, off, descales, nt=None, **kw):
    from generative_recommenders_b200.ops.hstu_attention import cuda_hstu_attention_fwd

    ds = None if descales is None else tuple(None if d is None else d.to(DEV) for d in descales)
    out = cuda_hstu_attention_fwd(N, alpha, q8.to(DEV), k8.to(DEV), v8.to(DEV), off.to(DEV),
                                  None if nt is None else nt.to(DEV), descales=ds, **kw)
    torch.cuda.synchronize()
    assert out.dtype == torch.bfloat16
    return out.cpu()


def check_parity(N, alpha, q, k, v, off, nt=None, what="", views=False, **kw):
    """Quantises q, k, v, runs the fp8 forward and holds it to the bf16 bound against the oracle on the dequantised values."""
    (q8, qd), (k8, kd), (v8, vd) = (quantize(t, off) for t in (q, k, v))
    if views:  # q, k, v as strided views of one [L, H, 3d] buffer; descales as non-contiguous views
        d = q.shape[2]
        buf = torch.cat([q8.view(torch.uint8), k8.view(torch.uint8), v8.view(torch.uint8)], dim=2).view(FP8).to(DEV)
        q8, k8, v8 = buf[:, :, :d], buf[:, :, d:2 * d], buf[:, :, 2 * d:]
        dsb = torch.stack([qd, kd, vd], dim=2).to(DEV)  # [B, H, 3]: each [:, :, i] has strides (3H, 3)
        qd, kd, vd = dsb[:, :, 0], dsb[:, :, 1], dsb[:, :, 2]
        assert not q8.is_contiguous() and not qd.is_contiguous()
    out = run(N, alpha, q8, k8, v8, off, (qd, kd, vd), nt, **kw)
    ref_kw = dict(max_attn_len=kw.get("max_attn_len", 0), contextual_seq_len=kw.get("contextual_seq_len", 0),
                  min_full_attn_seq_len=kw.get("min_full_attn_seq_len", 0))
    ref = O.hstu_mha_fwd(N, alpha, dequant(q8.cpu(), qd.cpu(), off), dequant(k8.cpu(), kd.cpu(), off),
                         dequant(v8.cpu(), vd.cpu(), off), off, nt, dtype=torch.float64, **ref_kw)
    assert_rel(out, ref, f"fp8 forward {what}")
    assert_rel_segments(out, ref, off, N, f"fp8 forward {what}")
    return out


LENGTHS = [300, 0, 129, 511, 64, 1]


@pytest.mark.parametrize("d", [32, 64, 128, 256])
@pytest.mark.parametrize("rms", [0.09, 1.0, 2.25, 4.0])
def test_parity_across_head_dims_and_logit_scales(d, rms):
    q, k, v, _, off, nt = normal_case(LENGTHS, [3, 0, 7, 20, 0, 1], 2, d, rms**0.5, torch.float32, seed=d + int(10 * rms))
    check_parity(512, 1.0 / d**0.5, q, k, v, off, nt, f"d={d} rms={rms}")


MASKS = {
    "window_min_full": dict(max_attn_len=100, min_full_attn_seq_len=40),
    "contextual": dict(contextual_seq_len=17),
    "window_contextual_targets": dict(max_attn_len=64, contextual_seq_len=5, min_full_attn_seq_len=0),
}


@pytest.mark.parametrize("d", [32, 128])
@pytest.mark.parametrize("mask", sorted(MASKS))
@pytest.mark.parametrize("i32", [False, True])
def test_mask_options_past_max_seq_len_and_empty_sequences(d, mask, i32):
    lengths = [700, 0, 260, 1100, 3]  # the first and fourth run past max_seq_len = 512: their rows >= 512 must be zero
    q, k, v, _, off, nt = normal_case(lengths, [9, 0, 4, 30, 1], 2, d, 1.0, torch.float32, seed=5, i32=i32)
    out = check_parity(512, 1.0 / d**0.5, q, k, v, off, nt, f"d={d} {mask} i32={i32}", **MASKS[mask])
    assert (out[512:700] == 0).all() and (out[700 + 260 + 512:700 + 260 + 1100] == 0).all()


@pytest.mark.parametrize("d", [32, 64, 128, 256])
def test_strided_views_of_one_buffer(d):
    q, k, v, _, off, nt = normal_case([200, 333, 64], [2, 5, 0], 2, d, 1.0, torch.float32, seed=77)
    check_parity(400, 1.0 / d**0.5, q, k, v, off, nt, f"views d={d}", views=True)


def test_long_sequence_wraps_the_ring():
    q, k, v, _, off, _ = normal_case([4096, 100], None, 2, 32, 1.0, torch.float32, seed=9)
    check_parity(4096, 1.0 / 32**0.5, q, k, v, off, None, "4096 rows d=32")


@pytest.mark.parametrize("d", [32, 64])
def test_tiny_descales_keep_full_precision(d):
    # qd, kd scaled by 2^-66 each: alpha/2 qd kd (~2^-146) is an fp32 subnormal with a few significant bits, yet the
    # logits still carry full precision; vd 2^120 brings the output back into bf16's normal range
    q, k, v, _, off, nt = normal_case([300, 129, 511], [3, 0, 7], 2, d, 1.0, torch.float32, seed=31)
    (q8, qd), (k8, kd), (v8, vd) = (quantize(t, off) for t in (q, k, v))
    qd, kd, vd = qd * 2.0**-66, kd * 2.0**-66, vd * 2.0**120
    N, alpha = 512, 1.0 / d**0.5
    out = run(N, alpha, q8, k8, v8, off, (qd, kd, vd), nt)
    ref = O.hstu_mha_fwd(N, alpha, dequant(q8, qd, off), dequant(k8, kd, off), dequant(v8, vd, off), off, nt,
                         dtype=torch.float64)
    assert torch.isfinite(out.float()).all()
    assert_rel(out, ref, f"fp8 forward, tiny q / k descales, d={d}")
    assert_rel_segments(out, ref, off, N, f"fp8 forward, tiny q / k descales, d={d}")


def _fixed(d=64, lengths=(300, 129, 511), seed=13):
    q, k, v, _, off, nt = normal_case(list(lengths), None, 2, d, 1.0, torch.float32, seed=seed)
    (q8, qd), (k8, kd), (v8, vd) = (quantize(t, off) for t in (q, k, v))
    return q8, k8, v8, qd, kd, vd, off


@pytest.mark.parametrize("d", [32, 128])
def test_none_descales_equal_ones_bitwise(d):
    q8, k8, v8, qd, _, _, off = _fixed(d)
    ones = torch.ones_like(qd)
    a = run(512, 0.125, q8, k8, v8, off, None)
    b = run(512, 0.125, q8, k8, v8, off, (ones, ones, ones))
    c = run(512, 0.125, q8, k8, v8, off, (None, ones, None))
    assert torch.equal(a.view(torch.int16), b.view(torch.int16)) and torch.equal(a.view(torch.int16), c.view(torch.int16))


@pytest.mark.parametrize("d", [32, 64, 256])
@pytest.mark.parametrize("e", [3, -5])
def test_power_of_two_descale_changes_act_bitwise(d, e):
    q8, k8, v8, qd, kd, vd, off = _fixed(d)
    alpha, s = 1.0 / d**0.5, 2.0**e
    out = run(512, alpha, q8, k8, v8, off, (qd, kd, vd))
    o1 = run(512, alpha, q8, k8, v8, off, (qd * s, kd / s, vd))
    assert torch.equal(o1.view(torch.int16), out.view(torch.int16))
    o2 = run(512, alpha, q8, k8, v8, off, (qd, kd, vd * s))
    assert torch.equal(o2.view(torch.int16), (out * s).view(torch.int16))


def test_bad_values_stay_in_their_sequence_and_head():
    d, N = 64, 400
    lengths = [300, 500, 129, 260]  # the second runs past max_seq_len
    q8, k8, v8, qd, kd, vd, off = _fixed(d, lengths, seed=21)
    o = [int(t) for t in off.tolist()]
    nan = torch.tensor([0x7F], dtype=torch.uint8).view(FP8)[0]  # the e4m3fn NaN
    poisoned = [(q8.clone(), k8.clone(), v8.clone(), qd.clone()) for _ in range(2)]
    # NaN in q, k and v inside sequence 0; NaN in every input past max_seq_len of sequence 1
    for val, (a, b_, c, _) in zip((nan, torch.zeros(1, dtype=FP8)[0]), poisoned):
        for t in (a, b_, c):
            t[o[0] + 37, 1, 5] = val
            t[o[1] + N: o[2]] = val
    # and a NaN descale of (sequence 2, head 0)
    poisoned[0][3][2, 0] = float("nan")
    poisoned[1][3][2, 0] = 0.0
    bad = run(N, 0.125, *poisoned[0][:3], off, (poisoned[0][3], kd, vd))
    zero = run(N, 0.125, *poisoned[1][:3], off, (poisoned[1][3], kd, vd))
    # NaN reaches only (sequence 0, head 1) and (sequence 2, head 0)
    assert not torch.isfinite(bad[o[0]:o[1], 1].float()).all() and not torch.isfinite(bad[o[2]:o[3], 0].float()).all()
    keep = torch.ones(bad.shape[:2], dtype=torch.bool)
    keep[o[0]:o[1], 1] = False
    keep[o[2]:o[3], 0] = False
    assert torch.isfinite(bad[keep].float()).all()
    assert torch.equal(bad[keep].view(torch.int16), zero[keep].view(torch.int16))
    assert (bad[o[1] + N:o[2]] == 0).all()
    assert_finite_rows(bad[:, 0:1], off, {2}, "head 0 outside the NaN descale")


def test_registered_ops_equal_the_raw_entry_bitwise():
    from generative_recommenders_b200 import torch_ops

    torch_ops.register()
    q8, k8, v8, qd, kd, vd, off = _fixed(64)
    N, alpha = 512, 0.125
    raw = run(N, alpha, q8, k8, v8, off, (qd, kd, None))
    args = [t.to(DEV) for t in (q8, k8, v8)]
    off32 = off.to(DEV, torch.int32)
    a = torch.ops.hstu.hstu_mha_fwd(N, alpha, *args, off32, True, None, None, 0, 0, 0, qd.to(DEV), kd.to(DEV), None, 0)
    b = torch.ops.hstu.hstu_mha(N, alpha, *args, off32, True, None, None, 0, 0, 0, qd.to(DEV), kd.to(DEV), None, False,
                                False, 0)
    for x in (a, b):
        assert x.dtype == torch.bfloat16 and torch.equal(x.cpu().view(torch.int16), raw.view(torch.int16))
    meta = torch.ops.hstu.hstu_mha_fwd(N, alpha, *(t.to("meta") for t in args), off32.to("meta"), True, None, None, 0, 0, 0,
                                       None, None, None, 0)
    assert meta.dtype == torch.bfloat16


def test_misuse_raises_with_a_message():
    from generative_recommenders_b200 import torch_ops
    from generative_recommenders_b200.ops.hstu_attention import cuda_hstu_attention_fwd

    torch_ops.register()
    q8, k8, v8, qd, kd, vd, off = _fixed(64)
    N, offd = 512, off.to(DEV)
    qg, kg, vg = (t.to(DEV) for t in (q8, k8, v8))
    qb = qg.to(torch.bfloat16)
    with pytest.raises(RuntimeError, match="float8_e4m3fn"):  # descales with bf16 inputs
        torch.ops.hstu.hstu_mha_fwd(N, 0.1, qb, qb, qb, offd, True, None, None, 0, 0, 0, qd.to(DEV), None, None, 0)
    with pytest.raises(RuntimeError, match="float8_e4m3fn"):
        cuda_hstu_attention_fwd(N, 0.1, qb, qb, qb, offd, descales=(None, None, None))
    with pytest.raises(RuntimeError, match="forward only"):  # a gradient through fp8
        torch.ops.hstu.hstu_mha(N, 0.1, qg.clone().requires_grad_(), kg, vg, offd, True, None, None, 0, 0, 0, None, None,
                                None, False, False, 0)
    with pytest.raises(RuntimeError, match="float8_e4m3fn"):  # mixed dtypes
        cuda_hstu_attention_fwd(N, 0.1, qg, kg, qb, offd)
    with pytest.raises(RuntimeError, match=r"\[B, H\]"):  # descale shape
        cuda_hstu_attention_fwd(N, 0.1, qg, kg, vg, offd, descales=(qd.to(DEV)[:, :1], None, None))
    with pytest.raises(RuntimeError, match="dqk == dv"):
        cuda_hstu_attention_fwd(N, 0.1, qg, kg, vg[:, :, :32].contiguous(), offd)
    L = qg.shape[0]
    q96 = torch.zeros(L, 2, 96, dtype=FP8, device=DEV)
    with pytest.raises(RuntimeError, match="dqk == dv"):
        cuda_hstu_attention_fwd(N, 0.1, q96, q96, q96, offd)
    wide = torch.zeros(L, 2, 72, dtype=FP8, device=DEV)  # row stride 144, head stride 72: not multiples of 16
    mis = wide[:, :, 8:72]
    with pytest.raises(RuntimeError, match="multiples of 16"):
        cuda_hstu_attention_fwd(N, 0.1, mis, mis, mis, offd)
