"""The KV-cached (delta-q) attention forward with bf16 / fp16 queries over a float8 e4m3 K / V cache (DESIGN.md 3.8): parity
with the fp64 oracle of pytorch_cached_hstu_mha on the dequantised cache, key chunks, masks, strided views of a fused cache,
descale folding, isolation of bad values, determinism, and the refusals of hstu_attn_fwd_delta_fp8_kv.

The file sorts after the attention test files that check kernel names with torch.profiler: a profiler session loses its first
device records in an older process, so GPU tests added ahead of those checks make them miss kernels more often."""
import ctypes as C
import math

import pytest
import torch

from oracle import hstu_oracle as O
from util import assert_rel, assert_rel_segments, normal_case, offsets_from

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
FP8 = torch.float8_e4m3fn


def _mods():
    from generative_recommenders_b200 import _lib
    from generative_recommenders_b200.ops import hstu_attention as HA

    return _lib, HA


def last_rows(x, off, delta):
    o = [int(t) for t in off.tolist()]
    return torch.cat([x[e - delta:e] for e in o[1:]])


def row_batch(off):
    """The sequence of every row of a jagged tensor."""
    lens = (off[1:] - off[:-1]).long()
    return torch.repeat_interleave(torch.arange(len(lens)), lens)


def quantise(x, off, scale=None):
    """x (float) -> e4m3 codes and the per (sequence, head) descale that maps them back: x ~ codes * descale[b, h].  scale:
    the descale to use instead of amax / 448."""
    B, H = len(off) - 1, x.shape[1]
    rb = row_batch(off)
    if scale is None:
        amax = torch.zeros(B, H)
        for b in range(B):
            seg = x[int(off[b]):int(off[b + 1])].float().abs()
            if seg.numel():
                amax[b] = seg.amax(dim=(0, 2))
        scale = torch.where(amax > 0, amax / 448.0, torch.ones_like(amax))
    codes = (x.float() / scale[rb][:, :, None]).to(FP8)
    return codes, scale.float()


def dequant(codes, ds, off):
    rb = row_batch(off)
    d = torch.ones(len(off) - 1, codes.shape[1], dtype=torch.float64) if ds is None else ds.double()
    return codes.double() * d[rb][:, :, None]


def case(lengths, delta, dqk, dv, dtype, seed=0, targets=None, i32=False, H=2):
    q, k, _, _, off, nt = normal_case(lengths, targets, H, dqk, 1.0, dtype, seed, i32=i32)
    v = torch.randn(k.shape[0], H, dv, generator=torch.Generator().manual_seed(seed + 1)).to(dtype)
    k8, kd = quantise(k, off)
    v8, vd = quantise(v, off)
    return last_rows(q, off, delta), k8, v8, kd, vd, off, nt


def run(dq, k8, v8, off, delta, N, alpha, nt=None, kv_descales=None, **kw):
    _, HA = _mods()
    ds = None if kv_descales is None else tuple(None if d is None else d.to(DEV) for d in kv_descales)
    out = HA.cuda_hstu_attention_fwd(N, alpha, dq.to(DEV), k8.to(DEV), v8.to(DEV), off.to(DEV),
                                     None if nt is None else nt.to(DEV), delta_q_len=delta,
                                     descales=None if ds is None else (None, *ds), **kw)
    torch.cuda.synchronize()
    return out


def oracle(dq, k8, v8, kd, vd, off, delta, N, alpha, nt=None, **mask):
    return O.delta_hstu_mha_fwd(N, alpha, dq, dequant(k8, kd, off), dequant(v8, vd, off), off, nt, dtype=torch.float64, **mask)


def check(lengths, delta, dqk, dv, dtype, seed=0, targets=None, i32=False, H=2, N=None, what="", **mask):
    dq, k8, v8, kd, vd, off, nt = case(lengths, delta, dqk, dv, dtype, seed, targets, i32, H)
    N = N or max(lengths)
    alpha = 1.0 / dqk**0.5
    out = run(dq, k8, v8, off, delta, N, alpha, nt, (kd, vd), **mask)
    assert out.dtype == dtype
    ref = oracle(dq, k8, v8, kd, vd, off, delta, N, alpha, nt, **mask)
    what = f"fp8 kv delta={delta} ({dqk}, {dv}) {dtype} {what}"
    assert_rel(out, ref, what)
    assert_rel_segments(out, ref, offsets_from([delta] * (len(off) - 1)), delta, what)
    return out, (dq, k8, v8, kd, vd, off, nt, N, alpha)


def params(dtype, dqk, dv, delta=16, B=4, H=8, N=8192):
    """hstu_attn_params of an fp8-KV delta call with placeholder (aligned, never dereferenced) device addresses."""
    _lib, _ = _mods()
    p = _lib.AttnParams()
    p.abi_version, p.dtype, p.impl = _lib.ABI_VERSION, dtype, _lib.IMPL_AUTO
    p.batch, p.heads, p.dqk, p.dv, p.max_seq_len = B, H, dqk, dv, N
    p.total_rows, p.alpha, p.delta_q_len = B * N, 0.1, delta
    p.seq_offsets = p.q = p.k = p.v = p.out = 1 << 20
    p.q_row_stride, p.q_head_stride = H * dqk, dqk
    p.k_row_stride, p.k_head_stride = H * dqk, dqk
    p.v_row_stride, p.v_head_stride = H * dv, dv
    p.o_row_stride, p.o_head_stride = H * dv, dv
    return p


def expected_workspace(B, H, delta, N, dv):
    """The chunk rule of the 16-bit delta-q forward: split only below 264 CTAs per chunk, into at most 264 / CTAs and
    ceil(N / 512) chunks."""
    ctas = B * H * math.ceil(delta / 128)
    chunks = 1 if ctas >= 264 else max(1, min(math.ceil(N / 512), 264 // ctas))
    return 0 if chunks == 1 else chunks * B * delta * H * dv * 4


# ---------------------------------------------------------------------------------------------------------------- parity
DIMS = [(32, 32), (64, 64), (128, 128), (256, 256), (128, 256)]
DELTAS = [1, 5, 16, 64, 100, 256]


@pytest.mark.parametrize("dims", DIMS)
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("delta", DELTAS)
def test_parity_across_head_dims_and_deltas(dims, dtype, delta):
    # len == delta, lengths one short of / at / one past a 64-key tile and a 512-key chunk from the queries
    lengths = [delta, delta + 63, delta + 64, delta + 65, delta + 511, delta + 512, delta + 513]
    check(lengths, delta, *dims, dtype, seed=dims[0] + dims[1] + delta, targets=[min(3, delta)] * len(lengths))


MASKS = {
    "none": ({}, None),
    "targets": ({}, "half"),
    "window": (dict(max_attn_len=100), "half"),
    "contextual": (dict(contextual_seq_len=17), None),
    "window_contextual": (dict(max_attn_len=64, contextual_seq_len=5), "delta"),
}


@pytest.mark.parametrize("mask", sorted(MASKS))
@pytest.mark.parametrize("dims", [(32, 32), (128, 128)])
@pytest.mark.parametrize("i32", [False, True])
def test_mask_options(mask, dims, i32):
    kw, tg = MASKS[mask]
    delta = 16
    lengths = [delta + 3, delta + 200, delta + 1000, delta + 64]
    targets = None if tg is None else [delta if tg == "delta" else max(1, delta // 2)] * len(lengths)
    check(lengths, delta, *dims, torch.bfloat16, seed=len(mask), targets=targets, i32=i32, what=mask, **kw)


@pytest.mark.parametrize("dims", [(32, 32), (128, 256)])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("B", [2, 40])
def test_one_chunk_and_several(dims, dtype, B):
    """B = 2: the 8192-key caches split into chunks (fp32 partials and the reduction); B = 40 (40 x 8 CTAs): one chunk."""
    _lib, _ = _mods()
    H, delta, N = 8, 16, 2048
    g = torch.Generator().manual_seed(B)
    lengths = torch.randint(delta, N + 1, (B,), generator=g).tolist()
    lengths[0] = N
    out, (dq, k8, v8, kd, vd, off, nt, N, alpha) = check(lengths, delta, *dims, dtype, seed=B, H=H, N=N, what=f"B={B}")
    p = params(_lib.BF16 if dtype == torch.bfloat16 else _lib.F16, *dims, delta=delta, B=B, H=H, N=N)
    p.total_rows = int(off[-1])
    want = expected_workspace(B, H, delta, N, dims[1])
    assert _lib.lib().hstu_attn_fp8_kv_workspace_bytes(C.byref(p)) == want
    assert (want > 0) == (B == 2)


@pytest.mark.parametrize("dims", DIMS)
def test_workspace_rule(dims):
    _lib, _ = _mods()
    lib = _lib.lib()
    for dt in (_lib.BF16, _lib.F16):
        for B, H, delta, N in ((1, 8, 1, 8192), (16, 8, 64, 8192), (128, 8, 16, 8192), (16, 4, 256, 8192), (2, 2, 5, 300)):
            p = params(dt, *dims, delta=delta, B=B, H=H, N=N)
            assert lib.hstu_attn_fp8_kv_workspace_bytes(C.byref(p)) == expected_workspace(B, H, delta, N, dims[1])


# ---------------------------------------------------------------------------------------------------------------- views
@pytest.mark.parametrize("dims", [(32, 32), (64, 64), (128, 256)])
def test_kv_views_of_one_fused_cache(dims):
    """k and v as 16-element-strided views of one e4m3 [rows, H, dqk + 16 + dv] cache buffer."""
    dqk, dv = dims
    delta, H = 16, 2
    dq, k8, v8, kd, vd, off, nt = case([500, 33, 129], delta, dqk, dv, torch.bfloat16, seed=21, targets=[5, 1, 16], H=H)
    fused = torch.zeros(k8.shape[0], H, dqk + 16 + dv, dtype=torch.uint8)
    fused[:, :, :dqk] = k8.view(torch.uint8)
    fused[:, :, dqk + 16:] = v8.view(torch.uint8)
    fused = fused.to(DEV).view(FP8)
    kv, vv = fused[:, :, :dqk], fused[:, :, dqk + 16:]
    assert not kv.is_contiguous() and not vv.is_contiguous()
    N = 600
    out = run(dq, kv, vv, off, delta, N, 1 / dqk**0.5, nt, (kd, vd))
    ref = run(dq, k8, v8, off, delta, N, 1 / dqk**0.5, nt, (kd, vd))
    assert torch.equal(out, ref)
    assert_rel(out, oracle(dq, k8, v8, kd, vd, off, delta, N, 1 / dqk**0.5, nt), "fused cache views")


# ---------------------------------------------------------------------------------------------------------------- scales
@pytest.mark.parametrize("dims", [(64, 64), (128, 256)])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_descales_none(dims, dtype):
    dq, k8, v8, kd, vd, off, nt = case([300, 90, 700], 16, *dims, dtype, seed=5)
    N, alpha = 700, 1 / dims[0]**0.5
    out = run(dq, k8, v8, off, 16, N, alpha, nt)
    assert_rel(out, oracle(dq, k8, v8, None, None, off, 16, N, alpha, nt), "no descales")
    part = run(dq, k8, v8, off, 16, N, alpha, nt, (None, vd))
    assert_rel(part, oracle(dq, k8, v8, None, vd, off, 16, N, alpha, nt), "v descale only")


@pytest.mark.parametrize("which", ["k", "v"])
@pytest.mark.parametrize("dims", [(32, 32), (256, 256)])
def test_tiny_descales(which, dims):
    """A descale of 2^-60 (bf16 output: fp16 cannot hold such results) stays out of fp32 subnormals."""
    dq, k8, v8, kd, vd, off, nt = case([300, 90, 2000], 16, *dims, torch.bfloat16, seed=6, H=2)
    tiny = torch.full_like(kd, 2.0**-60)
    kd, vd = (tiny, vd) if which == "k" else (kd, tiny)
    N, alpha = 2000, 1 / dims[0]**0.5
    out = run(dq, k8, v8, off, 16, N, alpha, nt, (kd, vd))
    ref = oracle(dq, k8, v8, kd, vd, off, 16, N, alpha, nt)
    assert ref.abs().max() > 0
    assert_rel(out, ref, f"tiny {which} descale")


@pytest.mark.parametrize("dims", [(32, 32), (128, 256)])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("lengths", [[300, 90, 700], [8192, 100]])  # one chunk / several
def test_descale_folding_is_exact(dims, dtype, lengths):
    """kd 2^e with alpha 2^-e leaves out bitwise unchanged; vd 2^e scales it by exactly 2^e."""
    dq, k8, v8, kd, vd, off, nt = case(lengths, 16, *dims, dtype, seed=7)
    N, alpha = max(lengths), 1 / dims[0]**0.5
    base = run(dq, k8, v8, off, 16, N, alpha, nt, (kd, vd))
    for e in (-5, 3):
        assert torch.equal(run(dq, k8, v8, off, 16, N, alpha * 2.0**-e, nt, (kd * 2.0**e, vd)), base), e
    # outputs that are normal numbers of the output type scale exactly (a subnormal one is rounded on a coarser grid)
    normal = base.float().abs() >= (2.0**-14 if dtype == torch.float16 else 2.0**-126)
    assert normal.float().mean() > 0.9
    for e in (1, 3):
        scaled = run(dq, k8, v8, off, 16, N, alpha, nt, (kd, vd * 2.0**e))
        assert torch.equal(scaled.float()[normal], base.float()[normal] * 2.0**e), e


# ---------------------------------------------------------------------------------------------------------------- isolation
@pytest.mark.parametrize("dims", [(32, 32), (256, 256)])
@pytest.mark.parametrize("lengths", [[100, 8000, 77], [70, 130, 201, 65]])
def test_bad_values_stay_in_their_sequence(dims, lengths):
    """A NaN code in one sequence's cache, and NaN codes past every other sequence's end (the next sequence's rows, written
    by the poisoned run into the bad sequence), leave every other sequence bitwise equal to a clean run."""
    delta, H, N = 5, 2, 8192
    dq, k8, v8, kd, vd, off, nt = case(lengths, delta, *dims, torch.bfloat16, seed=8, targets=[1] * len(lengths), H=H)
    o = [int(t) for t in off.tolist()]
    bad = 1
    clean_k, clean_v = k8.clone(), v8.clone()
    pk, pv = k8.clone().view(torch.uint8), v8.clone().view(torch.uint8)
    pk[o[bad]:o[bad + 1]] = 0x7F  # e4m3fn NaN
    pv[o[bad]:o[bad + 1]] = 0xFF  # -NaN
    a = run(dq, clean_k, clean_v, off, delta, N, 1 / dims[0]**0.5, nt, (kd, vd)).cpu()
    b = run(dq, pk.view(FP8), pv.view(FP8), off, delta, N, 1 / dims[0]**0.5, nt, (kd, vd)).cpu()
    keep = torch.ones(a.shape[0], dtype=torch.bool)
    keep[bad * delta:(bad + 1) * delta] = False
    assert torch.isfinite(a.float()).all()
    assert torch.equal(a[keep], b[keep])
    assert torch.isnan(b[~keep].float()).any()  # NaN stays NaN through the widening


@pytest.mark.parametrize("dims", [(32, 32), (128, 128)])
def test_bitwise_repeatable(dims):
    dq, k8, v8, kd, vd, off, nt = case([8192, 300, 16, 40], 16, *dims, torch.bfloat16, seed=4, targets=[3, 0, 16, 2])
    outs = [run(dq, k8, v8, off, 16, 8192, 1 / dims[0]**0.5, nt, (kd, vd)) for _ in range(2)]
    assert torch.isfinite(outs[0].float()).all()
    assert torch.equal(outs[0], outs[1])


def test_delta_hstu_mha_takes_an_fp8_cache():
    from generative_recommenders_b200.ops.hstu_attention import delta_hstu_mha

    dq, k8, v8, kd, vd, off, nt = case([400, 64, 1000], 16, 64, 64, torch.float16, seed=9)
    out = delta_hstu_mha(1000, 0.125, dq.to(DEV), k8.to(DEV), v8.to(DEV), off.to(DEV), nt, kv_descales=(kd.to(DEV), vd.to(DEV)))
    assert_rel(out, oracle(dq, k8, v8, kd, vd, off, 16, 1000, 0.125, nt), "delta_hstu_mha")


# ---------------------------------------------------------------------------------------------------------------- refusals
def test_refusals_launch_nothing():
    _lib, HA = _mods()
    lib = _lib.lib()
    ERR_INVALID, ERR_UNSUPPORTED = -1, -2
    ds = _lib.Descales()

    def rc(p, d=ds):
        return lib.hstu_attn_fwd_delta_fp8_kv(C.byref(p), C.byref(d), None)

    p = params(_lib.BF16, 64, 64, delta=0)
    assert rc(p) == ERR_UNSUPPORTED and b"delta_q_len" in lib.hstu_last_error()
    p = params(_lib.BF16, 64, 64)
    p.pos_w = 1 << 20
    assert rc(p) == ERR_UNSUPPORTED and b"bias" in lib.hstu_last_error()
    for dims in ((64, 32), (256, 128), (40, 40)):
        assert rc(params(_lib.F16, *dims)) == ERR_UNSUPPORTED and b"dqk" in lib.hstu_last_error()
    for dt in (_lib.E4M3, _lib.F32):
        assert rc(params(dt, 64, 64)) == ERR_UNSUPPORTED
    p = params(_lib.BF16, 64, 64)
    p.k_row_stride += 8  # half of a 16-byte unit of e4m3
    assert rc(p) == ERR_UNSUPPORTED and b"multiples of 16" in lib.hstu_last_error()
    p = params(_lib.BF16, 64, 64)
    p.q += 2
    assert rc(p) == ERR_UNSUPPORTED and b"multiples of 8" in lib.hstu_last_error()
    p = params(_lib.BF16, 64, 64)
    p.impl = _lib.IMPL_GENERIC
    assert rc(p) == ERR_UNSUPPORTED and b"wgmma" in lib.hstu_last_error()
    qd = _lib.Descales()
    qd.q = 1 << 20
    assert rc(params(_lib.BF16, 64, 64), qd) == ERR_INVALID and b"descale" in lib.hstu_last_error()
    for p in (params(_lib.BF16, 64, 64, delta=0), params(_lib.F16, 64, 32)):
        assert lib.hstu_attn_fp8_kv_workspace_bytes(C.byref(p)) == 0
    # the routing of the existing entries is unchanged: fp8 delta-q through hstu_attn_select_impl stays refused
    assert lib.hstu_attn_select_impl(C.byref(params(_lib.E4M3, 64, 64)), 0) == ERR_UNSUPPORTED
    # python: fp8 queries, an fp8 cache without delta, and mixed cache dtypes stay RuntimeErrors
    dq, k8, v8, kd, vd, off, nt = case([100, 50], 16, 32, 32, torch.bfloat16)
    k16 = dequant(k8, kd, off).to(torch.bfloat16)
    for args, kw in (((dq.to(FP8), k8, v8), dict(delta_q_len=16)), ((last_rows(k16, off, 16), k8, v8), {}),
                     ((dq, k16, v8), dict(delta_q_len=16)), ((dq, k8, v8), dict(delta_q_len=16, impl=_lib.IMPL_GENERIC))):
        with pytest.raises(RuntimeError):
            HA.cuda_hstu_attention_fwd(100, 0.1, *(t.to(DEV) for t in args), off.to(DEV), **kw)
