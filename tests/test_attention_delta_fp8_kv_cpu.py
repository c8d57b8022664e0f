"""The delta-q forward over an fp8 K / V cache without a GPU (DESIGN.md 3.8): the exact widening of every e4m3 code to bf16
and fp16, the folding of the descales into the kernel's scalars (fp64 emulation), the workspace rule of
hstu_attn_fp8_kv_workspace_bytes, and the compiler output of its kernels (scripts/sass_report.py; needs nvcc)."""
import ctypes as C
import importlib.util
import math
import os

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_spec = importlib.util.spec_from_file_location("sass_report", os.path.join(ROOT, "scripts", "sass_report.py"))
sass_report = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(sass_report)

CODES = torch.arange(256, dtype=torch.int32).to(torch.uint8).view(torch.float8_e4m3fn)


@pytest.mark.parametrize("wide", [torch.bfloat16, torch.float16])
def test_every_e4m3_code_widens_exactly(wide):
    x = CODES.float()
    w = CODES.to(wide).float()
    nan = torch.isnan(x)
    assert int(nan.sum()) == 2  # 0x7F and 0xFF: e4m3fn has NaN and no Inf
    assert torch.isnan(w[nan]).all()
    assert torch.equal(w[~nan], x[~nan])
    assert not torch.isinf(x).any()
    if wide == torch.float16:  # and every finite nonzero value is a normal fp16 value (>= 2^-14), as the kernel assumes
        nz = x[~nan & (x != 0)].abs()
        assert nz.min() == 2.0**-9 and nz.max() == 448.0


def _frexp(x):
    m, e = math.frexp(x)
    return m, e


def _fp32(x):
    return float(torch.tensor(x, dtype=torch.float64).float())


def scalars(alpha, kd, vd, inv_n):
    """The kernel's scalars, as it forms them: c_s = alpha/2 kd (the tanh argument), c_sp = alpha/2 kd 2^-e_k (P' = 2^-e_k P),
    and the output as a mantissa c_o and an exponent e_o ((1/N) vd 2^e_k)."""
    ma, ea = _frexp(_fp32(alpha / 2))
    mk, ek = _frexp(_fp32(kd))
    mv, ev = _frexp(_fp32(vd))
    m_s = _fp32(ma * mk)
    return _fp32(math.ldexp(m_s, ea + ek)), _fp32(math.ldexp(m_s, ea)), _fp32(inv_n * mv), ev + ek


@pytest.mark.parametrize("kd", [2.0**-60, 2.0**-8 * 1.37, 1.0, 3.0e3])
def test_descale_folding(kd):
    alpha, vd, inv_n = 0.125, 0.7, 1 / 8192
    c_s, c_sp, c_o, e_o = scalars(alpha, kd, vd, inv_n)
    # the product of the scales, whatever their size, with no fp32 subnormal on the way
    assert c_s == pytest.approx(alpha / 2 * kd, rel=1e-6)
    assert c_sp == pytest.approx(alpha / 2 * kd / 2.0 ** math.frexp(kd)[1], rel=1e-6)
    assert 2.0**-126 < c_sp < 1  # P' has the magnitude of the unscaled scores
    assert math.ldexp(c_o, e_o) * c_sp / c_s == pytest.approx(inv_n * vd, rel=1e-6)
    # kd 2^e with alpha 2^-e: the same c_s, P' scaled by 2^-e, the output scale by 2^e -- an unchanged output
    for e in (-5, 3):
        c_s2, c_sp2, c_o2, e_o2 = scalars(alpha * 2.0**-e, kd * 2.0**e, vd, inv_n)
        assert c_s2 == c_s and c_sp2 == math.ldexp(c_sp, -e) and c_o2 == c_o and e_o2 == e_o + e
    # vd 2^e: only the output exponent moves
    c_s3, c_sp3, c_o3, e_o3 = scalars(alpha, kd, vd * 8, inv_n)
    assert (c_s3, c_sp3, c_o3, e_o3) == (c_s, c_sp, c_o, e_o + 3)


def _lib_or_skip():
    from generative_recommenders_b200 import _lib

    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("libhstu_b200.so is not built")
    return _lib


def _params(_lib, dtype, dqk, dv, delta, B, H, N):
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


@pytest.mark.parametrize("dims", [(32, 32), (64, 64), (128, 128), (256, 256), (32, 256), (128, 256)])
def test_workspace_rule(dims):
    """The partials of the key chunks, by the rule of the 16-bit delta-q forward (sizes only: no device needed)."""
    _lib = _lib_or_skip()
    lib = _lib.lib()
    for dt in (_lib.BF16, _lib.F16):
        for B, H, delta, N in ((1, 8, 1, 8192), (16, 8, 64, 8192), (128, 8, 16, 8192), (16, 4, 256, 8192), (2, 2, 5, 300),
                               (3, 1, 100, 100)):
            ctas = B * H * math.ceil(delta / 128)
            chunks = 1 if ctas >= 264 else max(1, min(math.ceil(N / 512), 264 // ctas))
            want = 0 if chunks == 1 else chunks * B * delta * H * dims[1] * 4
            assert lib.hstu_attn_fp8_kv_workspace_bytes(C.byref(_params(_lib, dt, *dims, delta, B, H, N))) == want
    # refused calls need nothing: no delta, fp8 queries, dqk > dv
    for args in ((_lib.BF16, *dims, 0, 2, 2, 4096), (_lib.E4M3, *dims, 16, 2, 2, 4096), (_lib.F16, 64, 32, 16, 2, 2, 4096)):
        assert lib.hstu_attn_fp8_kv_workspace_bytes(C.byref(_params(_lib, *args))) == 0


@pytest.fixture(scope="module")
def report():
    if sass_report.tools() is None:
        pytest.skip("nvcc / cuobjdump not installed")
    return sass_report.report("attn_fwd_delta_e4m3kv_wgmma_kernel")


DIMS = [(32, 32), (64, 64), (128, 128), (256, 256), (32, 64), (32, 128), (32, 256), (64, 128), (64, 256), (128, 256)]


@pytest.mark.parametrize("dims", DIMS)
@pytest.mark.parametrize("bf16", [False, True])
def test_kernel_compiler_output(report, dims, bf16):
    dqk, dv = dims
    found = [r for name, r in report.items() if f"attn_fwd_delta_e4m3kv_wgmma_kernel<(int){dqk}, (int){dv}, (bool){int(bf16)}>" in name]
    assert len(found) == 1, sorted(report)
    r = found[0]
    assert r["spill_stores"] == 0 and r["spill_loads"] == 0, r
    assert not set(r["notes"]) & {"C7510", "C7512", "C7515"}, r  # no wgmma serialisation
    assert r["tanh_per_block"] >= 8, r
    if dv == 32 or (dv == 64 and not bf16):
        assert r["registers"] <= 128, r  # two CTAs per SM
