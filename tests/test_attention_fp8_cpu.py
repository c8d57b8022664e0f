"""The fp8 (e4m3) attention forward (DESIGN.md 3.5) without a GPU: its P exponent rule, an fp64 emulation of its arithmetic
held to the bf16 parity bound, the host-side checks of `hstu_attn_fwd_fp8`, and the compiler output of its kernels."""
import ctypes as C
import math
import os
import subprocess
import tempfile

import numpy as np
import pytest
import torch

from conftest import ROOT
from oracle import hstu_oracle as O
from util import TOL

FP8 = torch.float8_e4m3fn
E4M3_MAX = 448.0


# ---------------------------------------------------------------------------------------------------------------------
# the P exponent (csrc/attn_fp16_operands.cuh, e4m3_p_exp)
# ---------------------------------------------------------------------------------------------------------------------
def e4m3_p_exp(alpha, q_descale, k_descale, d):
    """p with |alpha qd kd| d 448^2 2^p in [2^11, 2^15): frexp exponents of the fp32 factors, d <= 2^ld; 0 for a zero, Inf or
    NaN factor; clamped to fp32's normal exponents."""
    s = 0
    for x in (alpha, q_descale, k_descale):
        x = abs(float(np.float32(x)))
        if x == 0.0 or not math.isfinite(x):
            return 0
        s += math.frexp(x)[1]
    ld = (d - 1).bit_length()
    return max(-126, min(127, -3 - (s + ld)))


def _bound(alpha, qd, kd, d):
    return abs(float(np.float32(alpha)) * float(np.float32(qd)) * float(np.float32(kd))) * d * E4M3_MAX**2


@pytest.mark.parametrize("d", [32, 64, 128, 256])
def test_p_exponent_puts_the_bound_in_2_11_to_2_15(d):
    rng = np.random.default_rng(d)
    cases = [(1 / d**0.5, 1 / 448, 1 / 448), (-0.125, 0.01, 3.0), (1.0, 1.0, 1.0), (-1 / d, 2e-3, 7e-4)]
    cases += [tuple(float(np.float32(x)) * s for x, s in zip(rng.lognormal(0, 3, 3), (1, 1, -1))) for _ in range(200)]
    cases += [(0.2, 1e-20, 3e-18), (0.2, 1e18, 4e15), (1.0, 1e-40, 1e10)]  # tiny (a subnormal descale), huge
    for alpha, qd, kd in cases:
        p = e4m3_p_exp(alpha, qd, kd, d)
        scaled = math.ldexp(_bound(alpha, qd, kd, d), p)
        assert 2.0**11 <= scaled < 2.0**15, (alpha, qd, kd, d, p, scaled)
        # p stays within fp32's normal exponents
        assert -126 <= p <= 127


def test_p_exponent_edge_cases():
    for bad in (0.0, -0.0, float("inf"), -float("inf"), float("nan")):
        assert e4m3_p_exp(bad, 1.0, 1.0, 64) == 0
        assert e4m3_p_exp(0.125, bad, 1.0, 64) == 0
        assert e4m3_p_exp(0.125, 1.0, bad, 64) == 0
    # a negative alpha or descale has the exponent of its magnitude
    assert e4m3_p_exp(-0.125, -0.01, 0.3, 32) == e4m3_p_exp(0.125, 0.01, 0.3, 32)
    # power-of-two changes move p by the same amount, and q 2^e with k 2^-e leaves it as it is
    assert e4m3_p_exp(0.125, 0.01 * 8, 0.3 / 8, 128) == e4m3_p_exp(0.125, 0.01, 0.3, 128)
    assert e4m3_p_exp(0.125, 0.01 * 8, 0.3, 128) == e4m3_p_exp(0.125, 0.01, 0.3, 128) - 3
    # clamped at fp32's normal exponents
    assert e4m3_p_exp(1e-30, 1e-30, 1e-30, 32) == 127
    assert e4m3_p_exp(1e30, 1e30, 1e30, 256) == -126


def _nvcc():
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    return None


def test_p_exponent_restatement_matches_the_header():
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not installed")
    vals = [0.0, float("inf"), float("nan"), 1e-40, 3e-20, 1 / 448, 0.01, -0.125, 1.0, 3.0, 7e5, 1e30]
    cases = [(a, q, k, d) for a in vals[3:] for q in vals for k in vals[::3] for d in (32, 64, 128, 256)]
    src = ('#include <stdio.h>\n#include <math.h>\n#include "attn_fp16_operands.cuh"\n'
           "int main() { float a, q, k; int d; while (scanf(\"%a %a %a %d\", &a, &q, &k, &d) == 4) "
           "printf(\"%d\\n\", hstu::e4m3_p_exp(a, q, k, d)); return 0; }\n")
    with tempfile.TemporaryDirectory() as tmp:
        with open(os.path.join(tmp, "p.cu"), "w") as f:
            f.write(src)
        exe = os.path.join(tmp, "p")
        subprocess.run([nvcc, "-std=c++20", "-I", os.path.join(ROOT, "generative_recommenders_b200", "csrc"),
                        os.path.join(tmp, "p.cu"), "-o", exe], check=True, capture_output=True)
        inp = "".join(f"{float(np.float32(a)).hex()} {float(np.float32(q)).hex()} {float(np.float32(k)).hex()} {d}\n"
                      for a, q, k, d in cases)
        out = subprocess.run([exe], input=inp, capture_output=True, text=True, check=True).stdout.split()
    assert [int(x) for x in out] == [e4m3_p_exp(*c) for c in cases]


# ---------------------------------------------------------------------------------------------------------------------
# fp64 emulation of the kernel's arithmetic
# ---------------------------------------------------------------------------------------------------------------------
def quantize(x):
    """Per-head e4m3 quantisation as the tests and the bench do it: descale = amax / 448 (fp32), x8 = e4m3(x / descale)."""
    ds = (x.float().abs().amax(dim=(0, 2)) / E4M3_MAX).clamp_min(1e-30)  # [H]
    return (x.float() / ds[None, :, None]).to(FP8), ds


def emulate(q8, k8, v8, qd, kd, vd, alpha, n_max, p_format=torch.float16):
    """One sequence, one head, causal mask, as attn_fwd_e4m3_wgmma_kernel computes it: S exact from the e4m3 values, x = S
    alpha/2 qd kd and x 2^p (fp32 scalars), P' = 2^p x (1 + tanh x) rounded to `p_format` (fp16: the kernel; e4m3: what an
    fp8 P would cost), V exact (its fp16 copy), O (1/N) vd 2^-p -> bf16."""
    n, d = q8.shape
    s = q8.double() @ k8.double().T
    p = e4m3_p_exp(alpha, qd, kd, d)
    if p_format == FP8:
        p -= 7  # the bound maps below 2^8 < 448, the largest e4m3 value
    # the kernel's scalars: frexp mantissas multiplied in fp32, exponents applied exactly
    (ma, ea), (mq, eq), (mk, ek) = (math.frexp(float(np.float32(f))) for f in (alpha / 2, qd, kd))
    m_s = float(np.float32(np.float32(np.float32(ma) * np.float32(mq)) * np.float32(mk)))
    c_s, c_sp = (float(np.float32(math.ldexp(m_s, ea + eq + ek + e))) for e in (0, p))
    x, xp = (s * c_s).float(), (s * c_sp).float()
    pp = xp * (1 + torch.tanh(x))
    pp = torch.where(torch.ones(n, n).tril().bool(), pp, 0.0).to(p_format).double()
    mv, ev = math.frexp(float(np.float32(vd)))
    out = (pp @ v8.double()) * float(np.float32(np.float32(1.0 / n_max) * np.float32(mv))) * math.ldexp(1.0, ev - p)
    return out.to(torch.bfloat16)


def _fp8_case(n, d, rms, seed):
    g = torch.Generator().manual_seed(seed)
    sigma = rms**0.5  # q, k ~ N(0, sigma^2), alpha = 1/sqrt(d): rms(alpha S) = sigma^2
    q, k = (sigma * torch.randn(n, 1, d, generator=g) for _ in range(2))
    v = torch.randn(n, 1, d, generator=g)
    return [quantize(t) for t in (q, k, v)], 1.0 / d**0.5


def _error(n, d, rms, seed, p_format):
    ((q8, qd), (k8, kd), (v8, vd)), alpha = _fp8_case(n, d, rms, seed)
    deq = [t.double() * s.double()[None, :, None] for t, s in ((q8, qd), (k8, kd), (v8, vd))]
    ref = O.hstu_mha_fwd(n, alpha, *deq, torch.tensor([0, n]), dtype=torch.float64)[:, 0].float()
    got = emulate(q8[:, 0], k8[:, 0], v8[:, 0], float(qd[0]), float(kd[0]), float(vd[0]), alpha, n, p_format)
    lim = math.hypot(TOL[torch.bfloat16], O.storage_quantisation(ref, torch.bfloat16))
    return O.rel_l2(got.float(), ref), lim


@pytest.mark.parametrize("rms", [0.09, 1.0, 2.25, 4.0])
def test_fp16_p_emulation_within_the_bf16_bound(rms):
    err, lim = _error(1024, 64, rms, 11, torch.float16)
    assert err <= lim, f"rms {rms}: {err:.3e} > {lim:.3e}"


@pytest.mark.parametrize("rms", [0.09, 1.0, 2.25, 4.0])
def test_e4m3_p_would_break_the_bf16_bound(rms):
    # why P . V stays 16-bit: P rounded to e4m3 (3 significand bits) alone is far outside the parity bound
    err, lim = _error(1024, 64, rms, 11, FP8)
    assert err > 2 * lim, f"rms {rms}: {err:.3e} <= 2 x {lim:.3e}"


def test_e4m3_values_widen_to_fp16_exactly():
    allb = torch.arange(256, dtype=torch.uint8).view(FP8)
    f = allb.float()
    fin = torch.isfinite(f)
    assert int(fin.sum()) == 254  # every byte but the two NaNs (0x7f, 0xff)
    assert torch.equal(f[fin].half().float(), f[fin])
    nz = f[fin].abs()
    nz = nz[nz > 0]
    assert float(nz.max()) == E4M3_MAX and float(nz.min()) == 2.0**-9 > 2.0**-14  # normal fp16 values


# ---------------------------------------------------------------------------------------------------------------------
# host-side checks of the C ABI (no device needed)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    from generative_recommenders_b200 import _lib
    from generative_recommenders_b200.build import build

    build()
    return _lib.lib()


def _params(d=64, dv=None, impl=0, rs=None, L=1000, H=4):
    from generative_recommenders_b200 import _lib

    p = _lib.AttnParams()
    p.abi_version, p.dtype, p.impl = 1, _lib.E4M3, impl
    p.batch, p.heads, p.dqk, p.dv, p.max_seq_len, p.total_rows = 3, H, d, dv or d, 512, L
    p.alpha = 0.125
    # never dereferenced: every call below is rejected (or sized) before anything touches the device
    p.seq_offsets, p.q, p.k, p.v, p.out = 1 << 20, 1 << 21, 1 << 22, 1 << 23, 1 << 24
    p.dout, p.dq, p.dk, p.dv_out = 1 << 25, 1 << 26, 1 << 27, 1 << 28
    r = rs if rs is not None else H * d
    p.q_row_stride = p.k_row_stride = p.v_row_stride = p.o_row_stride = r
    p.q_head_stride = p.k_head_stride = p.v_head_stride = p.o_head_stride = d
    return p


def test_e4m3_is_rejected_by_the_other_entries(lib):
    from generative_recommenders_b200 import _lib

    p = _params()
    assert lib.hstu_attn_bwd(C.byref(p), None) == -2
    assert b"no backward" in lib.hstu_last_error()
    assert lib.hstu_attn_select_impl(C.byref(p), 1) == -2
    assert lib.hstu_attn_fwd(C.byref(p), None) == -1
    assert b"hstu_attn_fwd_fp8" in lib.hstu_last_error()
    p = _params(impl=_lib.IMPL_GENERIC)
    assert lib.hstu_attn_select_impl(C.byref(p), 0) == -2
    assert b"generic" in lib.hstu_last_error()
    assert lib.hstu_attn_fwd_fp8(C.byref(p), None, None) == -2
    for impl in (_lib.IMPL_AUTO, _lib.IMPL_UMMA):
        assert lib.hstu_attn_select_impl(C.byref(_params(impl=impl)), 0) == _lib.IMPL_UMMA
    # the fp8 entry takes fp8 inputs only
    p = _params()
    p.dtype = _lib.BF16
    assert lib.hstu_attn_fwd_fp8(C.byref(p), None, None) == -1
    assert b"HSTU_E4M3" in lib.hstu_last_error()


@pytest.mark.parametrize("kw,what", [(dict(d=96), b"dqk == dv"), (dict(d=64, dv=32), b"dqk == dv"),
                                     (dict(d=64, rs=4 * 64 + 8), b"multiples of 16")])
def test_unsupported_shapes_are_refused_with_a_message(lib, kw, what):
    p = _params(**kw)
    assert lib.hstu_attn_select_impl(C.byref(p), 0) == -2
    assert what in lib.hstu_last_error()
    assert lib.hstu_attn_fwd_fp8(C.byref(p), None, None) == -2
    assert lib.hstu_attn_workspace_bytes(C.byref(p), 0) == 0


def test_malformed_descales_are_rejected(lib):
    from generative_recommenders_b200 import _lib

    p = _params()
    for field, val, msg in (("k_head_stride", -1, b"negative stride"), ("v_batch_stride", -4, b"negative stride"),
                            ("q", (1 << 30) + 2, b"not a float pointer")):
        ds = _lib.Descales()
        setattr(ds, field, val)
        assert lib.hstu_attn_fwd_fp8(C.byref(p), C.byref(ds), None) == -1, field
        assert msg in lib.hstu_last_error(), (field, lib.hstu_last_error())


@pytest.mark.parametrize("d", [32, 64, 128, 256])
def test_workspace_is_the_fp16_copy_of_v(lib, d):
    for L in (1, 1000, 4097):
        p = _params(d=d, L=L)
        assert lib.hstu_attn_workspace_bytes(C.byref(p), 0) == (L * 4 * d * 2 + 255) // 256 * 256
        assert lib.hstu_attn_workspace_bytes(C.byref(p), 1) == 0


def test_meta_output_is_bf16_and_descales_need_fp8_inputs():
    from generative_recommenders_b200 import torch_ops

    torch_ops.register()
    L, H, d, N = 100, 2, 64, 128
    q = torch.empty(L, H, d, dtype=FP8, device="meta")
    off = torch.empty(3, dtype=torch.int32, device="meta")
    ds = torch.empty(2, H, device="meta")
    out = torch.ops.hstu.hstu_mha_fwd(N, 0.125, q, q, q, off, True, None, None, 0, 0, 0, ds, ds, ds, 0)
    assert out.dtype == torch.bfloat16 and tuple(out.shape) == (L, H, d)
    qb = torch.zeros(L, H, d, dtype=torch.bfloat16)
    with pytest.raises(RuntimeError, match="float8_e4m3fn"):
        torch_ops._check(True, off, None, (ds, None, None), (qb, qb, qb))
    with pytest.raises(RuntimeError, match="attn_scale"):
        torch_ops._check(True, off, torch.ones(1), (None, None, None), (q, q, q))
    torch_ops._check(True, off, None, (ds, None, ds), (q, q, q))  # fp8 with descales: accepted
    from generative_recommenders_b200.ops.hstu_attention import cuda_hstu_attention_fwd

    with pytest.raises(RuntimeError, match="float8_e4m3fn"):  # mixed dtypes
        cuda_hstu_attention_fwd(N, 0.125, torch.zeros(L, H, d, dtype=FP8), qb, qb, torch.tensor([0, 50, 100]))


# ---------------------------------------------------------------------------------------------------------------------
# compiler output of the fp8 kernels (scripts/sass_report.py)
# ---------------------------------------------------------------------------------------------------------------------
def _sass_report():
    import importlib.util

    spec = importlib.util.spec_from_file_location("sass_report", os.path.join(ROOT, "scripts", "sass_report.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="module")
def report():
    sr = _sass_report()
    if sr.tools() is None:
        pytest.skip("nvcc / cuobjdump not installed")
    return sr.report("attn_fwd_e4m3")


def _check_schedule(report, name, dv):
    """No spills, no wgmma serialisation, and no more registers or per-tile instructions than the kernels compiled to when
    each carried its own copy of the K / V ring (CUDA 12.9, the flags of build.py): <= 128 registers at dv <= 64 (two CTAs
    per SM), 210 instructions per tile with the merged MMA batch (dv <= 64) and 203 without."""
    found = [r for n, r in report.items() if name in n]
    assert len(found) == 1, (name, sorted(report))
    r = found[0]
    assert r["spill_stores"] == 0 and r["spill_loads"] == 0, r
    assert not set(r["notes"]) & {"C7510", "C7512", "C7515"}, r
    if dv <= 64:
        assert r["registers"] <= 128, r
    assert r["iter_instrs"] is not None and r["iter_instrs"] <= (210 if dv <= 64 else 203), r
    return r


@pytest.mark.parametrize("d", [32, 64, 128, 256])
def test_e4m3_kernel_schedule(report, d):
    r = _check_schedule(report, f"attn_fwd_e4m3_wgmma_kernel<(int){d}>", d)
    if d == 32:
        assert r["tanh_per_block"] >= 8, r


@pytest.mark.parametrize("dqk,dv", [(32, 64), (32, 128), (32, 256), (64, 128), (64, 256), (128, 256)])
def test_e4m3_mixed_kernel_schedule(report, dqk, dv):
    _check_schedule(report, f"attn_fwd_e4m3_mixed_wgmma_kernel<(int){dqk}, (int){dv}>", dv)
