"""CPU side of the deterministic attention backward (hstu_attn_params.deterministic): dispatch and workspace of the C ABI, the
barrier models of the split kernels at their ring depths, and the compiler output of the d = 64 / 128 split kernels.

Without an sm_90 device the wgmma kernels are never selected, so there the dispatch test checks that a deterministic call
falls back to the generic kernels and that the refusals do not depend on the device."""
import ctypes as C
import importlib.util
import os

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _load(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, "scripts", f"{name}.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="module")
def lib():
    from generative_recommenders_b200 import _lib
    from generative_recommenders_b200.build import build

    build()
    return _lib.lib()


HSTU_ERR_UNSUPPORTED = -2
SM90 = torch.cuda.is_available() and torch.cuda.get_device_capability() == (9, 0)


def _params(dtype, dqk, dv=None, deterministic=1, impl=0, rows=4096, bias=False):
    """A backward problem with 16-byte aligned placeholder pointers and strides (nothing is dereferenced)."""
    from generative_recommenders_b200 import _lib

    dv = dqk if dv is None else dv
    p = _lib.AttnParams()
    p.abi_version, p.dtype, p.impl = _lib.ABI_VERSION, dtype, impl
    p.batch, p.heads, p.dqk, p.dv, p.max_seq_len, p.total_rows = 2, 2, dqk, dv, 2048, rows
    p.alpha = dqk**-0.5
    base = 1 << 24
    for i, f in enumerate(("seq_offsets", "q", "k", "v", "out", "dout", "dq", "dk", "dv_out")):
        setattr(p, f, base * (i + 1))
    for f, w in (("q", dqk), ("k", dqk), ("v", dv), ("o", dv), ("do", dv), ("dq", dqk), ("dk", dqk), ("dv", dv)):
        setattr(p, f"{f}_row_stride", p.heads * w)
        setattr(p, f"{f}_head_stride", w)
    p.deterministic = deterministic
    if bias:
        p.pos_w = base * 16
    return p


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("d", [32, 64, 128])
def test_deterministic_dispatch_of_wgmma_shapes(lib, dtype, d):
    from generative_recommenders_b200 import _lib

    code = _lib.BF16 if dtype == "bf16" else _lib.F16
    want = _lib.IMPL_UMMA if SM90 else _lib.IMPL_GENERIC
    assert lib.hstu_attn_select_impl(C.byref(_params(code, d)), 1) == want
    # a relative bias cannot be reproducible (its table gradients are added with atomics), whatever the device
    for impl in (_lib.IMPL_AUTO, _lib.IMPL_GENERIC, _lib.IMPL_UMMA):
        assert lib.hstu_attn_select_impl(C.byref(_params(code, d, impl=impl, bias=True)), 1) == HSTU_ERR_UNSUPPORTED
        assert b"relative bias" in lib.hstu_last_error()
    # the forward is reproducible anyway: the flag changes nothing there, with or without a bias
    assert lib.hstu_attn_select_impl(C.byref(_params(code, d, bias=True)), 0) == _lib.IMPL_GENERIC


@pytest.mark.parametrize("case", ["d256", "fp32", "dqk_ne_dv", "odd"])
def test_deterministic_dispatch_of_other_shapes(lib, case):
    from generative_recommenders_b200 import _lib

    p = {"d256": lambda **kw: _params(_lib.BF16, 256, **kw), "fp32": lambda **kw: _params(_lib.F32, 64, **kw),
         "dqk_ne_dv": lambda **kw: _params(_lib.F16, 64, 128, **kw), "odd": lambda **kw: _params(_lib.BF16, 40, **kw)}[case]
    assert lib.hstu_attn_select_impl(C.byref(p()), 1) == _lib.IMPL_GENERIC
    assert lib.hstu_attn_select_impl(C.byref(p(impl=_lib.IMPL_GENERIC)), 1) == _lib.IMPL_GENERIC
    assert lib.hstu_attn_select_impl(C.byref(p(impl=_lib.IMPL_UMMA)), 1) == HSTU_ERR_UNSUPPORTED
    assert lib.hstu_attn_workspace_bytes(C.byref(p()), 1) == 0


def test_deterministic_flag_must_be_0_or_1(lib):
    from generative_recommenders_b200 import _lib

    assert lib.hstu_attn_select_impl(C.byref(_params(_lib.BF16, 64, deterministic=2)), 1) < 0
    assert b"deterministic" in lib.hstu_last_error()


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("d", [64, 128])
def test_deterministic_backward_needs_no_workspace(lib, dtype, d):
    from generative_recommenders_b200 import _lib

    code = _lib.BF16 if dtype == "bf16" else _lib.F16
    assert lib.hstu_attn_workspace_bytes(C.byref(_params(code, d)), 1) == 0
    fused = lib.hstu_attn_workspace_bytes(C.byref(_params(code, d, deterministic=0)), 1)
    assert fused == (4096 * 2 * d * 4 if SM90 else 0)  # the fused kernel's fp32 dQ accumulator


def test_bf16_d32_workspace_does_not_depend_on_the_flag(lib):
    from generative_recommenders_b200 import _lib

    a = lib.hstu_attn_workspace_bytes(C.byref(_params(_lib.BF16, 32, deterministic=0)), 1)
    b = lib.hstu_attn_workspace_bytes(C.byref(_params(_lib.BF16, 32, deterministic=1)), 1)
    assert a == b
    assert (a > 0) == SM90  # the scaled fp16 copies of the wgmma path


# ---- barrier models of the split kernels at the ring depths of every head dim (csrc/attn_wgmma_bwd.cu) ----
bwd_model = _load("sim_bwd_protocol")
fwd_model = _load("sim_fwd_protocol")
TILES = (1, 2, 3, 4, 5, 8, 13, 40)
DEPTHS = (2, 3, 4)  # the kernels use 4 (dK / dV) and 3 (dQ) at every d; their neighbours are checked too


@pytest.mark.parametrize("stages", DEPTHS)
def test_split_protocols_at_each_ring_depth(stages):
    for tiles in TILES:
        for seed in range(15):
            bwd_model.run_dkdv(tiles, seed, stages=stages)
            fwd_model.run_dq(tiles, seed, stages=stages)


def test_models_default_to_the_kernel_depths():
    assert bwd_model.DKDV_STAGES == 4 and fwd_model.DQ_STAGES == 3


DKDV_BREAKS = {"break_release": "TMA load into q|wait on qf", "first_releaser": "TMA load into q|wait on qf",
               "early_release": "TMA load into q|wait on qf", "break_zero": "(reads|writes) q|TMA load into q"}
DQ_BREAKS = {"break_k_refill": "TMA load into k|wait on kf", "first_releaser": "TMA load into [kv]|wait on [kv]f",
             "early_release": "TMA load into k|wait on kf", "break_zero": "(reads|writes) k|TMA load into k"}


@pytest.mark.parametrize("stages", DEPTHS)
@pytest.mark.parametrize("brk", sorted(DKDV_BREAKS))
def test_dkdv_model_catches_its_seeded_breaks(stages, brk):
    with pytest.raises(bwd_model.Violation, match=DKDV_BREAKS[brk]):
        for seed in range(200):
            bwd_model.run_dkdv(8, seed, stages=stages, **{brk: True})


@pytest.mark.parametrize("stages", DEPTHS)
@pytest.mark.parametrize("brk", sorted(DQ_BREAKS))
def test_dq_model_catches_its_seeded_breaks(stages, brk):
    with pytest.raises(fwd_model.Violation, match=DQ_BREAKS[brk]):
        for seed in range(200):
            fwd_model.run_dq(8, seed, stages=stages, **{brk: True})


# ---- compiler output of the split kernels at d = 64 / 128 (needs nvcc, no GPU) ----
sass_report = _load("sass_report")
SERIALISATION = ("C7510", "C7512", "C7515")


@pytest.fixture(scope="module")
def report():
    if sass_report.tools() is None:
        pytest.skip("nvcc / cuobjdump not installed")
    return sass_report.report()


@pytest.mark.parametrize("bf16", [0, 1])
@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("kernel", ["attn_bwd_dkdv_wgmma_kernel", "attn_bwd_dq_wgmma_kernel"])
def test_split_kernel_schedule(report, kernel, d, bf16):
    name = f"{kernel}<(int){d}, (bool){bf16}>"
    found = [r for n, r in report.items() if name in n]
    assert len(found) == 1, (name, sorted(report))
    r = found[0]
    assert r["spill_stores"] == 0 and r["spill_loads"] == 0, r
    assert not set(r["notes"]) & set(SERIALISATION), r
    assert r["tanh_per_block"] >= 8, r
