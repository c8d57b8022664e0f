"""The fp8 (e4m3) attention forward at dqk < dv (DESIGN.md 3.5, "two widths") without a GPU: the dispatch and workspace of
the C ABI, what stays refused (the swapped pairs, dims outside the set, delta-q, the relative bias, the backward), and the
compiler output of attn_fwd_e4m3_mixed_wgmma_kernel (attn_wgmma_mixed_fwd_e4m3.cu).

The fp8 forward runs on the wgmma kernels only, so its dispatch does not depend on the device."""
import ctypes as C
import importlib.util
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PAIRS = [(32, 64), (32, 128), (32, 256), (64, 128), (64, 256), (128, 256)]
HSTU_ERR_UNSUPPORTED = -2


@pytest.fixture(scope="module")
def lib():
    from generative_recommenders_b200 import _lib
    from generative_recommenders_b200.build import build

    build()
    return _lib.lib()


def _params(dqk, dv, L=1000, H=4, **kw):
    """e4m3 q, k [L, H, dqk] and v [L, H, dv] as contiguous tensors, bf16 out [L, H, dv]; never dereferenced: every call
    below is sized or refused before anything touches the device."""
    from generative_recommenders_b200 import _lib

    p = _lib.AttnParams()
    p.abi_version, p.dtype, p.impl = _lib.ABI_VERSION, _lib.E4M3, kw.pop("impl", _lib.IMPL_AUTO)
    p.batch, p.heads, p.dqk, p.dv, p.max_seq_len, p.total_rows = 3, H, dqk, dv, 512, L
    p.alpha = dqk**-0.5
    p.seq_offsets, p.q, p.k, p.v, p.out = 1 << 20, 1 << 21, 1 << 22, 1 << 23, 1 << 24
    p.dout, p.dq, p.dk, p.dv_out = 1 << 25, 1 << 26, 1 << 27, 1 << 28
    p.q_row_stride = p.k_row_stride = H * dqk
    p.q_head_stride = p.k_head_stride = dqk
    p.v_row_stride = p.o_row_stride = H * dv
    p.v_head_stride = p.o_head_stride = dv
    for k, v in kw.items():
        setattr(p, k, v)
    return p


@pytest.mark.parametrize("dqk,dv", PAIRS)
def test_fp8_mixed_dims_select_the_wgmma_kernels_with_the_dv_copy_of_v(lib, dqk, dv):
    from generative_recommenders_b200 import _lib

    for impl in (_lib.IMPL_AUTO, _lib.IMPL_UMMA):
        assert lib.hstu_attn_select_impl(C.byref(_params(dqk, dv, impl=impl)), 0) == _lib.IMPL_UMMA
    # the workspace is the fp16 copy of v, [L, H, dv], whatever dqk is
    for L in (1, 1000, 4097):
        assert lib.hstu_attn_workspace_bytes(C.byref(_params(dqk, dv, L=L)), 0) == (L * 4 * dv * 2 + 255) // 256 * 256
    # no generic kernel takes fp8, and there is no backward
    assert lib.hstu_attn_select_impl(C.byref(_params(dqk, dv, impl=_lib.IMPL_GENERIC)), 0) == HSTU_ERR_UNSUPPORTED
    assert b"generic" in lib.hstu_last_error()
    p = _params(dqk, dv)
    assert lib.hstu_attn_select_impl(C.byref(p), 1) == HSTU_ERR_UNSUPPORTED
    assert lib.hstu_attn_bwd(C.byref(p), None) == HSTU_ERR_UNSUPPORTED
    assert b"no backward" in lib.hstu_last_error()
    assert lib.hstu_attn_workspace_bytes(C.byref(p), 1) == 0


@pytest.mark.parametrize("dqk,dv", [(dv, dqk) for dqk, dv in PAIRS] + [(32, 96), (16, 64), (48, 128), (64, 512)])
def test_swapped_pairs_and_dims_outside_the_set_are_refused(lib, dqk, dv):
    p = _params(dqk, dv)
    if dv > 256:  # the shared head-dim check of every attention entry comes first
        assert lib.hstu_attn_select_impl(C.byref(p), 0) == -1
        return
    assert lib.hstu_attn_select_impl(C.byref(p), 0) == HSTU_ERR_UNSUPPORTED
    msg = lib.hstu_last_error()
    assert b"dqk == dv" in msg and f"dqk={dqk}, dv={dv}".encode() in msg, msg
    assert lib.hstu_attn_fwd_fp8(C.byref(p), None, None) == HSTU_ERR_UNSUPPORTED
    assert lib.hstu_attn_workspace_bytes(C.byref(p), 0) == 0


@pytest.mark.parametrize("dqk,dv", [(32, 64), (128, 256)])
@pytest.mark.parametrize("what", ["delta_q", "bias"])
def test_delta_q_and_the_relative_bias_stay_refused(lib, dqk, dv, what):
    p = _params(dqk, dv, **({"delta_q_len": 16} if what == "delta_q" else {"pos_w": 1 << 29}))
    assert lib.hstu_attn_select_impl(C.byref(p), 0) == HSTU_ERR_UNSUPPORTED
    assert b"delta_q and the relative bias are not supported" in lib.hstu_last_error()
    assert lib.hstu_attn_fwd_fp8(C.byref(p), None, None) == HSTU_ERR_UNSUPPORTED
    assert lib.hstu_attn_workspace_bytes(C.byref(p), 0) == 0


def test_v_view_alignment_is_checked_at_its_own_width(lib):
    # v's row stride 2 dv + 8 is no multiple of 16 bytes; q and k are fine
    p = _params(64, 128, v_row_stride=4 * 128 + 8)
    assert lib.hstu_attn_select_impl(C.byref(p), 0) == HSTU_ERR_UNSUPPORTED
    assert b"multiples of 16" in lib.hstu_last_error()


def test_meta_output_has_the_value_width():
    import torch

    from generative_recommenders_b200 import torch_ops

    torch_ops.register()
    L, H, N = 100, 2, 128
    q = torch.empty(L, H, 128, dtype=torch.float8_e4m3fn, device="meta")
    v = torch.empty(L, H, 256, dtype=torch.float8_e4m3fn, device="meta")
    off = torch.empty(3, dtype=torch.int32, device="meta")
    out = torch.ops.hstu.hstu_mha_fwd(N, 0.125, q, q, v, off, True, None, None, 0, 0, 0, None, None, None, 0)
    assert out.dtype == torch.bfloat16 and tuple(out.shape) == (L, H, 256)


# ---- compiler output of the dqk < dv fp8 kernels (needs nvcc, no GPU) ----
def _sass_report():
    spec = importlib.util.spec_from_file_location("sass_report", os.path.join(ROOT, "scripts", "sass_report.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="module")
def report():
    sr = _sass_report()
    if sr.tools() is None:
        pytest.skip("nvcc / cuobjdump not installed")
    return sr.report("attn_fwd_e4m3_mixed_wgmma_kernel")


@pytest.mark.parametrize("dqk,dv", PAIRS)
def test_fp8_mixed_dims_kernel_compiler_output(report, dqk, dv):
    """No spills, no wgmma serialisation, at most 128 registers at dv = 64 (two CTAs per SM) and 255 elsewhere, and an
    elementwise stage whose tanh ptxas can overlap.  Shared memory is checked by static_asserts."""
    found = [r for name, r in report.items() if f"attn_fwd_e4m3_mixed_wgmma_kernel<(int){dqk}, (int){dv}>" in name]
    assert len(found) == 1, (dqk, dv, sorted(report))
    r = found[0]
    assert r["spill_stores"] == 0 and r["spill_loads"] == 0, r
    assert not set(r["notes"]) & {"C7510", "C7512", "C7515"}, r
    assert r["registers"] <= (128 if dv == 64 else 255), r
    assert r["tanh_per_block"] >= 8, r
