"""The deterministic attention backward on the wgmma kernels (d = 32, 64, 128; bf16 and fp16).

`cuda_hstu_attention_bwd(..., deterministic=True)`, `torch.use_deterministic_algorithms(True)` and
`torch.ops.hstu.hstu_mha(deterministic=True)` run the atomic-free attn_bwd_dkdv_wgmma_kernel + attn_bwd_dq_wgmma_kernel pair
at every head dim the wgmma backward covers.  Checked here: which kernels run, bitwise repeatability on long sequences, parity
with the oracle in fp64 (targets, window, contextual prefix, int32 / int64 offsets, strided views of one uvqk / duvqk buffer,
rows past max_seq_len), the score-scale sweep and the sequence isolation of tests/test_gpu_attention_numerics.py on the new
kernels, and the global torch flag through a 2-layer STU stack.
"""
import ctypes as C

import pytest
import torch

from test_gpu_attention_numerics import (ISO_LENGTHS, ISO_N, ISO_TARGETS, SIGMAS, SWEEP_N, _check_isolated, _compare,
                                         _oracle, _poison, _sweep_case)
from util import assert_rel, assert_rel_segments, normal_case, offsets_from

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda")
DIMS = [32, 64, 128]
DTYPES = [torch.bfloat16, torch.float16]
SPLIT = ("attn_bwd_dkdv_wgmma_kernel", "attn_bwd_dq_wgmma_kernel")
NOT_SPLIT = ("attn_bwd_wgmma_kernel", "dq_convert_kernel", "attn_bwd_kv_generic_kernel", "attn_bwd_q_generic_kernel")


def _ops():
    from generative_recommenders_b200 import _lib
    from generative_recommenders_b200.ops import hstu_attention as ha

    return _lib, ha


def _kernels_of(fn, attempts=3):
    """Names of the CUDA kernels `fn` launches (torch.profiler).  Every caller's `fn` launches kernels, so a session that
    recorded no kernel at all (nothing, or only some of the copies around the kernels) lost its records in the profiler; it
    is profiled again (`fn` runs again: each caller's `fn` can be repeated).  The names of a session that recorded a kernel
    are returned as they are."""
    from torch.profiler import ProfilerActivity, profile

    for _ in range(attempts):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        names = {ev.name for ev in prof.events() if ev.device_type == torch.autograd.DeviceType.CUDA}
        if any(not n.startswith(("Memcpy", "Memset")) for n in names):
            break
    return names


def _assert_split_path(names, what):
    for k in SPLIT:
        assert any(k in n for n in names), f"{what}: {k} did not run ({sorted(names)})"
    for k in NOT_SPLIT:
        assert not any(k in n for n in names), f"{what}: {k} ran ({sorted(names)})"


def _bwd(N, alpha, do, q, k, v, off, nt, win=0, ctx=0, min_full=0, grads=None, **kw):
    _, ha = _ops()
    dq, dk, dv = grads if grads is not None else (torch.full_like(t, float("nan")) for t in (q, k, v))
    ha.cuda_hstu_attention_bwd(N, alpha, do, q, k, v, dq, dk, dv, off, num_targets=nt, max_attn_len=win,
                               contextual_seq_len=ctx, min_full_attn_seq_len=min_full, **kw)
    return dq, dk, dv


def _params(N, alpha, q, k, v, off, deterministic, impl=None, bias=False):
    """hstu_attn_params of a backward over device tensors (select_impl / workspace queries)."""
    _lib, ha = _ops()
    p = _lib.AttnParams()
    ha._fill_common(p, N, alpha, q, k, v, off, None, 0, 0, 0, _lib.IMPL_AUTO if impl is None else impl)
    p.dout, p.dq, p.dk, p.dv_out = q.data_ptr(), q.data_ptr(), k.data_ptr(), v.data_ptr()
    for name, t in (("do", q), ("dq", q), ("dk", k), ("dv", v)):
        setattr(p, f"{name}_row_stride", t.stride(0))
        setattr(p, f"{name}_head_stride", t.stride(1))
    p.deterministic = int(deterministic)
    if bias:
        p.pos_w = q.data_ptr()
    return p


@pytest.mark.parametrize("d", DIMS)
@pytest.mark.parametrize("dtype", DTYPES)
def test_deterministic_backward_runs_the_split_wgmma_kernels(d, dtype):
    _lib, _ = _ops()
    q, k, v, do, off, nt = (t.to(DEV) for t in normal_case([700, 300], [5, 2], 2, d, 0.5, dtype, 5))
    N, alpha = 768, d**-0.5
    _assert_split_path(_kernels_of(lambda: _bwd(N, alpha, do, q, k, v, off, nt, deterministic=True)),
                       f"deterministic=True d={d} {dtype}")
    lib = _lib.lib()
    p = _params(N, alpha, q, k, v, off, True)
    assert lib.hstu_attn_select_impl(C.byref(p), 1) == _lib.IMPL_UMMA
    if dtype == torch.float16 or d > 32:  # bf16 at d = 32: the scaled fp16 copies are the workspace, with or without the flag
        assert lib.hstu_attn_workspace_bytes(C.byref(p), 1) == 0
    p.deterministic = 0
    if d > 32:
        assert lib.hstu_attn_workspace_bytes(C.byref(p), 1) == q.shape[0] * q.shape[1] * d * 4  # the fused kernel's dQ


@pytest.mark.parametrize("d", DIMS)
@pytest.mark.parametrize("dtype", DTYPES)
def test_deterministic_backward_is_bitwise_repeatable(d, dtype):
    """Long sequences with targets: every dq element sums up to N / 64 key tiles."""
    N = 4096 if d == 128 else 8192
    lengths = [N, N - 500, N - 64, 3 * N // 4]
    q, k, v, do, off, nt = normal_case(lengths, [3, 17, 1, 9], 2, d, 0.6, dtype, 11 + d)
    q, k, v, do, off, nt = (t.to(DEV) for t in (q, k, v, do, off, nt))
    runs = [_bwd(N, d**-0.5, do, q, k, v, off, nt, deterministic=True) for _ in range(2)]
    torch.cuda.synchronize()
    for name, a, b in zip(("dq", "dk", "dv"), *runs):
        assert torch.isfinite(a).all(), f"{name}: non-finite values"
        assert torch.equal(a.view(torch.int16), b.view(torch.int16)), f"{name}: two calls differ"


PARITY = {  # (lengths, targets, N, window, min_full, ctx, int32 offsets, strided uvqk views)
    "targets_window_context_i32_strided": ([1100, 517, 300, 70], [9, 0, 4, 2], 1024, 150, 64, 37, True, True),
    "targets_causal_i64": ([1024, 700, 129, 1], [20, 3, 0, 1], 1024, 0, 0, 0, False, False),
}


@pytest.mark.parametrize("case", sorted(PARITY))
@pytest.mark.parametrize("d", DIMS)
@pytest.mark.parametrize("dtype", DTYPES)
def test_deterministic_backward_matches_the_oracle(case, d, dtype):
    """The first sequence of the first case runs past max_seq_len: its rows there must come out as zeros (the gradient
    buffers start as NaN).  Strided: q / k / v and dq / dk / dv are column slices of one [L, H * (2 dv + 2 dqk)] buffer."""
    lengths, targets, N, win, min_full, ctx, i32, strided = PARITY[case]
    H, alpha = 2, d**-0.5
    q, k, v, do, off, nt = normal_case(lengths, targets, H, d, 1.0, dtype, 101 + d, i32=i32)
    L = q.shape[0]
    if strided:
        def views(buf):
            _, vv, qq, kk = torch.split(buf, [d * H, d * H, d * H, d * H], dim=1)
            return tuple(t.view(L, H, d) for t in (qq, kk, vv))

        uvqk = torch.empty(L, 4 * H * d, device=DEV, dtype=dtype)
        qd, kd, vd = views(uvqk)
        for dst, src in zip((qd, kd, vd), (q, k, v)):
            dst.copy_(src)
        duvqk = torch.full((L, 4 * H * d), float("nan"), device=DEV, dtype=dtype)
        grads = views(duvqk)
        assert grads[0].stride(0) == 4 * H * d
    else:
        qd, kd, vd = (t.to(DEV) for t in (q, k, v))
        grads = None
    got = _bwd(N, alpha, do.to(DEV), qd, kd, vd, off.to(DEV), nt.to(DEV), win, ctx, min_full, grads=grads, deterministic=True)
    torch.cuda.synchronize()
    ref = _oracle(N, alpha, q, k, v, do, off.long(), nt, win, ctx, min_full)[1:]
    for name, a, r in zip(("dq", "dk", "dv"), got, ref):
        assert_rel(a, r, f"{case} d={d} {dtype} {name}")
        assert_rel_segments(a, r, off, N, f"{case} d={d} {dtype} {name}")


def _fwd_bwd_det(N, alpha, q, k, v, dout, off, nt):
    _, ha = _ops()
    qd, kd, vd, dod, offd = (t.to(DEV) for t in (q, k, v, dout, off))
    ntd = None if nt is None else nt.to(DEV)
    out = ha.cuda_hstu_attention_fwd(N, alpha, qd, kd, vd, offd, ntd)
    grads = _bwd(N, alpha, dod, qd, kd, vd, offd, ntd, deterministic=True)
    torch.cuda.synchronize()
    return (out,) + tuple(grads)


@pytest.mark.parametrize("sigma", SIGMAS)
@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("dtype", DTYPES)
def test_deterministic_backward_across_score_scales(sigma, d, dtype):
    """The sweep of test_wgmma_vs_oracle_across_score_scales, rms(alpha S) up to 4, on the split kernels at d = 64 / 128."""
    q, k, v, dout, off, nt = _sweep_case(sigma, d, dtype)
    alpha = d**-0.5
    got = _fwd_bwd_det(SWEEP_N, alpha, q, k, v, dout, off, nt)
    ref = _oracle(SWEEP_N, alpha, q, k, v, dout, off, nt)
    _compare(got, ref, off, SWEEP_N, f"deterministic d={d} {dtype} rms(alpha S)={sigma**2:g}")


@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("value", ["nan", "inf"])
def test_deterministic_non_finite_rows_stay_in_their_sequence(d, dtype, value):
    """test_non_finite_rows_stay_in_their_sequence on the split kernels: without atomics dq too is bitwise that of the run
    whose poisoned rows hold zeros."""
    q, k, v, dout, off, nt = normal_case(ISO_LENGTHS, ISO_TARGETS, 2, d, 0.7, dtype, 300 + d)
    alpha = d**-0.5
    clean = [_poison(t, 0.0, 0) for t in (q, k, v, dout)]
    dirty = [_poison(t, value, i) for i, t in enumerate((q, k, v, dout))]
    got = _fwd_bwd_det(ISO_N, alpha, *dirty, off, nt)
    base = _fwd_bwd_det(ISO_N, alpha, *clean, off, nt)
    ref = _oracle(ISO_N, alpha, *clean, off, nt)
    _check_isolated(got, base, ref, f"deterministic d={d} {dtype} {value}")


HSTU_ERR_UNSUPPORTED = -2


def test_unsupported_deterministic_requests_are_refused():
    _lib, _ = _ops()
    lib = _lib.lib()
    q = torch.zeros(256, 2, 64, device=DEV, dtype=torch.bfloat16)
    off = torch.tensor([0, 256], device=DEV)
    p = _params(256, 0.125, q, q, q, off, True, bias=True)
    assert lib.hstu_attn_select_impl(C.byref(p), 1) == HSTU_ERR_UNSUPPORTED
    assert b"relative bias" in lib.hstu_last_error()
    q256 = torch.zeros(256, 2, 256, device=DEV, dtype=torch.bfloat16)
    p = _params(256, 0.0625, q256, q256, q256, off, True)
    assert lib.hstu_attn_select_impl(C.byref(p), 1) == _lib.IMPL_GENERIC
    p.impl = _lib.IMPL_UMMA
    assert lib.hstu_attn_select_impl(C.byref(p), 1) == HSTU_ERR_UNSUPPORTED


def test_global_flag_makes_an_stu_stack_bitwise_reproducible(monkeypatch):
    """torch.use_deterministic_algorithms(True): a bf16 2-layer STU stack at d = 64 gives bitwise identical dx and parameter
    gradients over two forward + backward runs, on the split wgmma kernels."""
    from generative_recommenders_b200.modules.stu import STULayer, STULayerConfig, STUStack

    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")  # deterministic cuBLAS for the block's GEMMs
    torch.manual_seed(5)
    D, H, d, N = 256, 2, 64, 4096
    stack = STUStack([STULayer(STULayerConfig(embedding_dim=D, num_heads=H, hidden_dim=d, attention_dim=d,
                                              output_dropout_ratio=0.0, target_aware=True)) for _ in range(2)])
    stack = stack.to(DEV).to(torch.bfloat16)
    lengths = torch.tensor([4096, 3000, 3900, 2048], device=DEV)
    off = torch.zeros(5, dtype=torch.int64, device=DEV)
    off[1:] = torch.cumsum(lengths, 0)
    nt = torch.tensor([4, 11, 1, 20], device=DEV)
    x0 = torch.randn(int(off[-1]), D, device=DEV, dtype=torch.bfloat16)
    dy = torch.randn(int(off[-1]), D, device=DEV, dtype=torch.bfloat16)

    def run():
        stack.zero_grad(set_to_none=True)
        x = x0.clone().requires_grad_()
        y = stack(x=x, x_lengths=lengths, x_offsets=off, max_seq_len=N, num_targets=nt)
        y.backward(dy)
        torch.cuda.synchronize()
        return [x.grad.clone()] + [p.grad.clone() for p in stack.parameters()]

    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    try:
        torch.use_deterministic_algorithms(True)
        a, b = run(), []

        def again():
            b[:] = run()

        names = _kernels_of(again)
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=prev_warn)
    _assert_split_path({n for n in names if "attn_bwd" in n or "convert" in n}, "STU stack under the global flag")
    assert len(a) == len(b)
    for i, (g0, g1) in enumerate(zip(a, b)):
        assert torch.isfinite(g0.float()).all(), f"gradient {i} is not finite"
        assert torch.equal(g0.view(torch.int16), g1.view(torch.int16)), f"gradient {i} differs between two runs"


def test_torch_ops_hstu_mha_deterministic_at_d128():
    from generative_recommenders_b200 import torch_ops

    torch_ops.register()
    q, k, v, do, off, nt = normal_case([4096, 3500, 2900], [7, 1, 30], 2, 128, 0.6, torch.bfloat16, 128, i32=True)
    N = 4096
    grads = []

    def run():
        qd, kd, vd = (t.to(DEV).requires_grad_() for t in (q, k, v))
        out = torch.ops.hstu.hstu_mha(N, 128**-0.5, qd, kd, vd, off.to(DEV), True, nt.to(DEV), None, 0, 0, 0, None, None, None,
                                      True, True, 0)
        out.backward(do.to(DEV))
        torch.cuda.synchronize()
        grads.append((qd.grad, kd.grad, vd.grad))

    run()
    _assert_split_path(_kernels_of(run), "torch.ops.hstu.hstu_mha(deterministic=True) d=128")
    for name, a, b in zip(("dq", "dk", "dv"), *grads):
        assert torch.isfinite(a.float()).all(), f"{name}: non-finite values"
        assert torch.equal(a.view(torch.int16), b.view(torch.int16)), f"{name}: two calls differ"
