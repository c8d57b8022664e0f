"""The delta-q (KV-cached) attention forward on the wgmma kernels (DESIGN.md 3.6): routing and workspace, parity with the fp64
oracle of pytorch_cached_hstu_mha and with the generic kernel, key chunks, strided views, isolation of bad values,
determinism, and the cached forward of an STU stack."""
import ctypes as C
import math

import pytest
import torch

from oracle import hstu_oracle as O
from util import assert_rel, assert_rel_segments, normal_case, offsets_from

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")


def _mods():
    from generative_recommenders_b200 import _lib
    from generative_recommenders_b200.ops.hstu_attention import cuda_hstu_attention_fwd

    return _lib, cuda_hstu_attention_fwd


def last_rows(x, off, delta):
    """The last `delta` rows of every sequence of a jagged [L, ...] tensor: the delta_q layout [B * delta, ...]."""
    o = [int(t) for t in off.tolist()]
    return torch.cat([x[e - delta:e] for e in o[1:]])


def run(x_q, k, v, off, delta, N, alpha, nt=None, impl=None, **kw):
    _lib, fwd = _mods()
    impl = _lib.IMPL_UMMA if impl is None else impl
    out = fwd(N, alpha, x_q.to(DEV), k.to(DEV), v.to(DEV), off.to(DEV), None if nt is None else nt.to(DEV), impl=impl,
              delta_q_len=delta, **kw)
    torch.cuda.synchronize()
    return out


def lib_workspace(dq, k, v, off, delta, N, nt=None, **mask):
    """The library's hstu_attn_workspace_bytes for this call (0: one key chunk, the attention kernel writes out itself)."""
    _lib, _ = _mods()
    from generative_recommenders_b200.ops.hstu_attention import _fill_common

    p = _lib.AttnParams()
    _fill_common(p, N, 0.1, dq, k, v, off, nt, mask.get("max_attn_len", 0), mask.get("contextual_seq_len", 0), 0,
                 _lib.IMPL_AUTO, delta)
    p.out, p.o_row_stride, p.o_head_stride = 1 << 20, dq.shape[1] * v.shape[2], v.shape[2]
    return int(_lib.lib().hstu_attn_workspace_bytes(C.byref(p), 0))


def case(lengths, delta, d, dtype, sigma=1.0, seed=0, targets=None, i32=False, H=2):
    q, k, v, _, off, nt = normal_case(lengths, targets, H, d, sigma, dtype, seed, i32=i32)
    return last_rows(q, off, delta), k, v, off, nt


def check(lengths, delta, d, dtype, sigma=1.0, seed=0, targets=None, i32=False, H=2, N=None, what="", **mask):
    dq, k, v, off, nt = case(lengths, delta, d, dtype, sigma, seed, targets, i32, H)
    N = N or max(lengths)
    alpha = 1.0 / d**0.5
    out = run(dq, k, v, off, delta, N, alpha, nt, **mask)
    ref = O.delta_hstu_mha_fwd(N, alpha, dq, k, v, off, nt, dtype=torch.float64, **mask)
    what = f"delta={delta} d={d} {dtype} {what}"
    assert_rel(out, ref, what)
    assert_rel_segments(out, ref, offsets_from([delta] * (len(off) - 1)), delta, what)
    return out, (dq, k, v, off, nt, N, alpha)


# ---------------------------------------------------------------------------------------------------------------- routing
def params(dtype, d, dv=None, delta=16, B=4, H=8, N=8192, impl=0):
    """hstu_attn_params of a delta call with placeholder (aligned, never dereferenced) device addresses."""
    _lib, _ = _mods()
    p = _lib.AttnParams()
    p.abi_version, p.dtype, p.impl = _lib.ABI_VERSION, dtype, impl
    p.batch, p.heads, p.dqk, p.dv, p.max_seq_len = B, H, d, dv or d, N
    p.total_rows, p.alpha, p.delta_q_len = B * N, 0.1, delta
    p.seq_offsets = p.q = p.k = p.v = p.out = 1 << 20
    p.q_row_stride = p.k_row_stride = p.v_row_stride = p.o_row_stride = H * d
    p.q_head_stride = p.k_head_stride = p.v_head_stride = p.o_head_stride = d
    return p


def expected_workspace(B, H, delta, N, d):
    """The documented chunk rule: split only below 264 CTAs per chunk, into at most 264 / CTAs and ceil(N / 512) chunks."""
    ctas = B * H * math.ceil(delta / 128)
    chunks = 1 if ctas >= 264 else max(1, min(math.ceil(N / 512), 264 // ctas))
    return 0 if chunks == 1 else chunks * B * delta * H * d * 4


@pytest.mark.parametrize("d", [32, 64, 128, 256])
def test_select_impl_and_workspace(d):
    _lib, _ = _mods()
    lib = _lib.lib()
    for dt in (_lib.BF16, _lib.F16):
        assert lib.hstu_attn_select_impl(C.byref(params(dt, d)), 0) == _lib.IMPL_UMMA
        assert lib.hstu_attn_select_impl(C.byref(params(dt, d, impl=_lib.IMPL_GENERIC)), 0) == _lib.IMPL_GENERIC
        for B, H, delta, N in ((1, 8, 1, 8192), (16, 8, 64, 8192), (128, 8, 16, 8192), (16, 4, 256, 8192), (2, 2, 5, 300),
                               (3, 1, 100, 100)):
            p = params(dt, d, delta=delta, B=B, H=H, N=N)
            assert lib.hstu_attn_workspace_bytes(C.byref(p), 0) == expected_workspace(B, H, delta, N, d), (B, H, delta, N)
    # B * H * query tiles >= 264: one chunk, no workspace; the bound of the rule at d = 256
    assert lib.hstu_attn_workspace_bytes(C.byref(params(_lib.BF16, d, delta=64, B=33, H=8)), 0) == 0
    assert expected_workspace(1, 1, 128, 1 << 20, 256) <= 264 * 128 * 256 * 4


def test_unsupported_shapes_route_to_generic():
    _lib, _ = _mods()
    lib = _lib.lib()
    for p in (params(_lib.F32, 64), params(_lib.BF16, 48), params(_lib.BF16, 25), params(_lib.F16, 64, dv=32)):
        assert lib.hstu_attn_select_impl(C.byref(p), 0) == _lib.IMPL_GENERIC
        assert lib.hstu_attn_workspace_bytes(C.byref(p), 0) == 0
        p.impl = _lib.IMPL_UMMA
        assert lib.hstu_attn_select_impl(C.byref(p), 0) == -2
    p = params(_lib.E4M3, 64)  # fp8 delta-q stays refused
    assert lib.hstu_attn_select_impl(C.byref(p), 0) == -2


# ---------------------------------------------------------------------------------------------------------------- parity
DELTAS = [1, 5, 16, 64, 100, 256]


@pytest.mark.parametrize("d", [32, 64, 128, 256])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("delta", DELTAS)
def test_parity_across_head_dims_and_deltas(d, dtype, delta):
    # len == delta, lengths one short of / at / one past a 64-key tile and a 512-key chunk from the queries
    lengths = [delta, delta + 63, delta + 64, delta + 65, delta + 511, delta + 700]
    check(lengths, delta, d, dtype, seed=d + delta, targets=[min(3, delta)] * 6)


MASKS = {
    "none": ({}, None),
    "targets_eq_delta": ({}, "delta"),
    "targets_lt_delta": ({}, "half"),
    "window": (dict(max_attn_len=100), "half"),
    "contextual": (dict(contextual_seq_len=17), None),
    "window_contextual": (dict(max_attn_len=64, contextual_seq_len=5), "delta"),
}


@pytest.mark.parametrize("mask", sorted(MASKS))
@pytest.mark.parametrize("d", [32, 128])
@pytest.mark.parametrize("delta", [5, 64, 100])
@pytest.mark.parametrize("i32", [False, True])
def test_mask_options(mask, d, delta, i32):
    kw, tg = MASKS[mask]
    lengths = [delta + 3, delta + 200, delta + 1000, delta + 64]
    targets = None if tg is None else [delta if tg == "delta" else max(1, delta // 2)] * len(lengths)
    check(lengths, delta, d, torch.bfloat16, seed=len(mask) + delta, targets=targets, i32=i32, what=mask, **kw)


@pytest.mark.parametrize("rms", [0.09, 1.0, 2.25, 4.0])
@pytest.mark.parametrize("d", [32, 64, 128, 256])
def test_logit_scales(rms, d):
    check([600, 80, 1500], 16, d, torch.bfloat16, sigma=rms**0.5, seed=int(10 * rms) + d, targets=[4, 0, 16],
          what=f"rms={rms}")


@pytest.mark.parametrize("d", [32, 128])
@pytest.mark.parametrize("lengths", [[8192], [8192, 70, 300]])
def test_long_cache_splits_into_chunks(d, lengths):
    _lib, _ = _mods()
    out, (dq, k, v, off, nt, N, alpha) = check(lengths, 16, d, torch.bfloat16, seed=3, H=2, N=8192, what="split")
    assert lib_workspace(dq, k, v, off, 16, N, nt) > 0  # the call really ran on more than one chunk
    # the generic kernel on the same inputs agrees within the same bound
    gen = run(dq, k, v, off, 16, N, alpha, nt, impl=_lib.IMPL_GENERIC)
    assert_rel(out, gen.float(), "delta wgmma vs generic")


@pytest.mark.parametrize("d", [32, 64, 128, 256])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_agrees_with_generic_kernel(d, dtype):
    _lib, _ = _mods()
    dq, k, v, off, nt = case([300, 64, 1029, 17], 17, d, dtype, seed=11, targets=[2, 17, 5, 0])
    kw = dict(max_attn_len=200, contextual_seq_len=3)
    a = run(dq, k, v, off, 17, 1100, 0.2, nt, **kw)
    g = run(dq, k, v, off, 17, 1100, 0.2, nt, impl=_lib.IMPL_GENERIC, **kw)
    ref = O.delta_hstu_mha_fwd(1100, 0.2, dq, k, v, off, nt, dtype=torch.float64, **kw)
    assert_rel(a, ref, "wgmma")
    assert_rel(g, ref, "generic")
    assert_rel(a, g.float(), "wgmma vs generic")


# ---------------------------------------------------------------------------------------------------------------- views
@pytest.mark.parametrize("d", [32, 64, 128, 256])
def test_delta_q_view_of_a_fused_projection(d):
    delta, H = 16, 2
    dq, k, v, off, nt = case([500, 33, 129], delta, d, torch.bfloat16, seed=21, targets=[5, 1, 16], H=H)
    # [rows, u | q | k | v] as hstu_compute_uqvk leaves it: q is a strided view (row stride 4 H d, head stride d)
    fused = torch.randn(dq.shape[0], 4 * H * d).to(torch.bfloat16)
    fused[:, H * d:2 * H * d] = dq.reshape(dq.shape[0], -1)
    fused = fused.to(DEV)
    view = fused[:, H * d:2 * H * d].view(dq.shape[0], H, d)
    assert not view.is_contiguous()
    N = 600
    out = run(view, k, v, off, delta, N, 1 / d**0.5, nt)
    ref = run(dq, k, v, off, delta, N, 1 / d**0.5, nt)
    assert torch.equal(out, ref)
    assert_rel(out, O.delta_hstu_mha_fwd(N, 1 / d**0.5, dq, k, v, off, nt, dtype=torch.float64), "view")


# ---------------------------------------------------------------------------------------------------------------- isolation
@pytest.mark.parametrize("d", [32, 256])
@pytest.mark.parametrize("lengths", [[100, 8000, 77], [70, 130, 201, 65]])
def test_bad_values_stay_in_their_sequence(d, lengths):
    delta, H, N = 5, 2, 8192
    dq, k, v, off, nt = case(lengths, delta, d, torch.bfloat16, seed=8, targets=[1] * len(lengths), H=H)
    o = [int(t) for t in off.tolist()]
    bad = 1  # sequence 1: zeros in the reference run, NaN / Inf in the other
    clean = [t.clone() for t in (dq, k, v)]
    clean[0][bad * delta:(bad + 1) * delta] = 0
    clean[1][o[bad]:o[bad + 1]] = 0
    clean[2][o[bad]:o[bad + 1]] = 0
    poisoned = [t.clone() for t in clean]
    poisoned[0][bad * delta:(bad + 1) * delta] = float("nan")
    poisoned[1][o[bad]:o[bad + 1]] = float("nan")
    poisoned[2][o[bad]:o[bad + 1]] = float("inf")
    a = run(*clean, off, delta, N, 1 / d**0.5, nt).cpu()
    b = run(*poisoned, off, delta, N, 1 / d**0.5, nt).cpu()
    keep = torch.ones(a.shape[0], dtype=torch.bool)
    keep[bad * delta:(bad + 1) * delta] = False
    assert torch.isfinite(a[keep].float()).all()
    assert torch.equal(a[keep], b[keep])


# ---------------------------------------------------------------------------------------------------------------- determinism
@pytest.mark.parametrize("d", [32, 128])
def test_bitwise_repeatable_with_a_poisoned_allocator(d, monkeypatch):
    """Every fp32 partial the reduction reads has been written by the attention kernel: the workspace holds NaN when the
    kernels start.  The sequences of one or a few key tiles leave most of their 16 chunk shares empty (zero partials)."""
    _lib, _ = _mods()
    from generative_recommenders_b200.ops import hstu_attention as HA

    delta, N = 16, 8192
    dq, k, v, off, nt = (t.to(DEV) for t in case([8192, 300, delta, 40], delta, d, torch.bfloat16, seed=4, H=2,
                                                  targets=[3, 0, 16, 2]))
    nbytes = lib_workspace(dq, k, v, off, delta, N, nt)
    assert nbytes > 0

    def poison_allocator():  # freed NaN blocks of exactly the workspace request (its size class and rounding)
        junk = [torch.empty(nbytes + 256, dtype=torch.uint8, device=DEV).fill_(0xFF) for _ in range(8)]
        del junk

    orig, filled = HA._workspace, []

    def nan_workspace(p, bwd, device):  # and the workspace itself NaN (0xFFFFFFFF) on the stream of the kernels
        ws = orig(p, bwd, device)
        if ws is not None:
            ws.fill_(0xFF)
            filled.append(ws.numel())
        return ws

    monkeypatch.setattr(HA, "_workspace", nan_workspace)
    outs = []
    for _ in range(2):
        poison_allocator()
        outs.append(run(dq, k, v, off, delta, N, 1 / d**0.5, nt))
    assert filled == [nbytes + 256] * 2
    assert torch.isfinite(outs[0].float()).all()
    assert torch.equal(outs[0], outs[1])
    gen = run(dq, k, v, off, delta, N, 1 / d**0.5, nt, impl=_lib.IMPL_GENERIC)
    assert_rel(outs[0], gen.float(), "poisoned workspace vs generic")
    ref = O.delta_hstu_mha_fwd(N, 1 / d**0.5, dq.cpu(), k.cpu(), v.cpu(), off.cpu(), nt.cpu(), dtype=torch.float64)
    assert_rel(outs[0], ref, "poisoned workspace vs oracle")
    assert_rel_segments(outs[0], ref, offsets_from([delta] * 4), delta, "poisoned workspace vs oracle")


# ---------------------------------------------------------------------------------------------------------------- one chunk
def check_one_chunk(lengths, delta, d, dtype, N, H, seed, what, **mask):
    """A call with a single key chunk (no workspace: the attention kernel scales by 1/N and writes out itself), with out and
    delta_q as strided views of wider buffers; nothing outside the out view may be touched."""
    _lib, fwd = _mods()
    dq, k, v, off, nt = case(lengths, delta, d, dtype, seed=seed, H=H, targets=[min(4, delta)] * len(lengths))
    assert lib_workspace(dq, k, v, off, delta, N, nt, **mask) == 0
    rows = dq.shape[0]
    qbuf = torch.randn(rows, H, 3 * d).to(dtype)
    qbuf[:, :, d:2 * d] = dq
    qbuf = qbuf.to(DEV)
    obuf = torch.full((rows, H, 2 * d), 7.0, dtype=dtype, device=DEV)
    out_view, q_view = obuf[:, :, d:], qbuf[:, :, d:2 * d]
    assert not out_view.is_contiguous() and not q_view.is_contiguous()
    alpha = 1.0 / d**0.5
    res = fwd(N, alpha, q_view, k.to(DEV), v.to(DEV), off.to(DEV), nt.to(DEV), impl=_lib.IMPL_UMMA, delta_q_len=delta,
              out=out_view, **mask)
    torch.cuda.synchronize()
    assert res.data_ptr() == out_view.data_ptr()
    assert (obuf[:, :, :d] == 7).all(), "a write outside the out view"
    ref = O.delta_hstu_mha_fwd(N, alpha, dq, k, v, off, nt, dtype=torch.float64, **mask)
    what = f"one chunk, delta={delta} d={d} {dtype} {what}"
    assert_rel(res, ref, what)
    assert_rel_segments(res, ref, offsets_from([delta] * len(lengths)), delta, what)


@pytest.mark.parametrize("d", [32, 64, 128, 256])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("delta", [16, 200])  # 16: the second warpgroup is padding only; 200: two query tiles
def test_one_chunk_short_cache(d, dtype, delta):
    # N <= 512: one chunk whatever the batch
    check_one_chunk([delta, delta + 63, delta + 130, 512], delta, d, dtype, 512, 2, seed=d + delta, what="N=512",
                    max_attn_len=300, contextual_seq_len=2)


@pytest.mark.parametrize("d", [32, 128])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_one_chunk_large_batch(d, dtype):
    # B * H * query tiles = 34 * 8 = 272 >= 264: one chunk on long caches
    g = torch.Generator().manual_seed(d)
    lengths = torch.randint(600, 1300, (34,), generator=g).tolist()
    check_one_chunk(lengths, 5, d, dtype, 1300, 8, seed=d + 1, what="B=34 H=8")


# ---------------------------------------------------------------------------------------------------------------- end to end
@pytest.mark.parametrize("d", [32, 64])
def test_stu_stack_cached_forward_bf16(d):
    from generative_recommenders_b200.modules.stu import STULayer, STULayerConfig, STUStack

    torch.manual_seed(5)
    D, H, delta = 256, 8, 16
    stack = STUStack([STULayer(STULayerConfig(embedding_dim=D, num_heads=H, hidden_dim=d, attention_dim=d,
                                              output_dropout_ratio=0.0, target_aware=True)) for _ in range(2)])
    stack = stack.to(DEV).to(torch.bfloat16).eval()
    lengths = torch.tensor([700, 129, 1000, 64], device=DEV)
    full_len = lengths + delta
    nt = torch.full((4,), delta, device=DEV)
    off = offsets_from(full_len.tolist(), DEV)
    N = 1000 + delta
    x = torch.randn(int(off[-1]), D, device=DEV).to(torch.bfloat16)
    with torch.no_grad():
        y_full = stack(x=x, x_lengths=full_len, x_offsets=off, max_seq_len=N, num_targets=nt)
        for layer in stack._stu_layers:
            layer.reset_kv_cache()
        stack(x=x, x_lengths=full_len, x_offsets=off, max_seq_len=N, num_targets=nt, max_kv_caching_len=1000,
              kv_caching_lengths=lengths)
        rows = torch.cat([torch.arange(int(off[i + 1]) - delta, int(off[i + 1]), device=DEV) for i in range(4)])
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            y_delta = stack.cached_forward(delta_x=x[rows], num_targets=nt)
            torch.cuda.synchronize()
    names = {e.key for e in prof.key_averages()}
    assert any("attn_fwd_delta_wgmma_kernel" in n for n in names), sorted(names)
    assert not any("attn_fwd_generic_kernel" in n for n in names), sorted(names)
    assert_rel(y_delta, y_full[rows].float(), "cached vs full forward, bf16", tol=1.5e-2)
