"""CPU side of the attention backward at head dim 256 on the wgmma kernels: dispatch and workspace of the C ABI, the compiler
output of the d = 256 split kernels (attn_bwd_dkdv_wgmma_kernel, attn_bwd_dq_wgmma_kernel), and the barrier models at their
ring depths.

Without an sm_90 device the wgmma kernels are never selected, so there the dispatch test checks the generic fall-back and
that the refusals do not depend on the device."""
import ctypes as C
import importlib.util
import os

import pytest
import torch

from test_attention_deterministic_cpu import HSTU_ERR_UNSUPPORTED, SM90, _params

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


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
def test_d256_backward_dispatch(lib, dtype):
    from generative_recommenders_b200 import _lib

    code = _lib.BF16 if dtype == "bf16" else _lib.F16
    p = _params(code, 256, deterministic=0)
    assert lib.hstu_attn_select_impl(C.byref(p), 1) == (_lib.IMPL_UMMA if SM90 else _lib.IMPL_GENERIC)
    assert lib.hstu_attn_workspace_bytes(C.byref(p), 1) == 0  # the split kernels: no fp32 dQ accumulator
    # deterministic = 1 stays on the generic kernels, and forcing the wgmma kernels with it is refused
    assert lib.hstu_attn_select_impl(C.byref(_params(code, 256)), 1) == _lib.IMPL_GENERIC
    assert lib.hstu_attn_select_impl(C.byref(_params(code, 256, impl=_lib.IMPL_UMMA)), 1) == HSTU_ERR_UNSUPPORTED
    # dqk != dv and fp32 route as before: generic kernels
    assert lib.hstu_attn_select_impl(C.byref(_params(code, 256, 128, deterministic=0)), 1) == _lib.IMPL_GENERIC
    assert lib.hstu_attn_select_impl(C.byref(_params(_lib.F32, 256, deterministic=0)), 1) == _lib.IMPL_GENERIC


# ---- compiler output of the d = 256 split kernels (needs nvcc, no GPU) ----
sass_report = _load("sass_report")
SERIALISATION = ("C7510", "C7512", "C7515")


@pytest.fixture(scope="module")
def report():
    if sass_report.tools() is None:
        pytest.skip("nvcc / cuobjdump not installed")
    return sass_report.report()


@pytest.mark.parametrize("bf16", [0, 1])
@pytest.mark.parametrize("kernel", ["attn_bwd_dkdv_wgmma_kernel", "attn_bwd_dq_wgmma_kernel"])
def test_d256_split_kernel_compiler_output(report, kernel, bf16):
    """No spills, no wgmma serialisation, at most 255 registers (one CTA of 256 threads per SM), and an elementwise stage
    whose tanh ptxas can overlap.  Shared memory (224 KB + barriers) is checked against kSmemPerSm by static_asserts."""
    name = f"{kernel}<(int)256, (bool){bf16}>"
    found = [r for n, r in report.items() if name in n]
    assert len(found) == 1, (name, sorted(report))
    r = found[0]
    assert r["spill_stores"] == 0 and r["spill_loads"] == 0, r
    assert not set(r["notes"]) & set(SERIALISATION), r
    assert r["registers"] <= 255, r
    assert r["tanh_per_block"] >= 8, r


# ---- barrier models at the d = 256 ring depths (csrc/attn_wgmma_bwd.cu: BwdCfg<256, false>, DqCfg<256>) ----
bwd_model = _load("sim_bwd_protocol")
fwd_model = _load("sim_fwd_protocol")
TILES = (1, 2, 3, 4, 5, 8, 13, 64)  # 64 query tiles of 32 rows: a 2048-row causal key range


def test_d256_protocols_at_their_ring_depths():
    assert bwd_model.DKDV_STAGES_D256 == 3 and fwd_model.DQ_STAGES == 3
    for tiles in TILES:
        for seed in range(25):
            for straddle in (False, True):
                bwd_model.run_dkdv(tiles, seed, stages=bwd_model.DKDV_STAGES_D256, straddle=straddle)
                fwd_model.run_dq(tiles, seed, stages=fwd_model.DQ_STAGES, straddle=straddle)


DKDV_BREAKS = {"break_release": "TMA load into q|wait on qf", "first_releaser": "TMA load into q|wait on qf",
               "early_release": "TMA load into q|wait on qf", "break_zero": "(reads|writes) q|TMA load into q"}


@pytest.mark.parametrize("brk", sorted(DKDV_BREAKS))
def test_d256_dkdv_model_catches_its_seeded_breaks(brk):
    with pytest.raises(bwd_model.Violation, match=DKDV_BREAKS[brk]):
        for seed in range(200):
            bwd_model.run_dkdv(8, seed, stages=bwd_model.DKDV_STAGES_D256, **{brk: True})
