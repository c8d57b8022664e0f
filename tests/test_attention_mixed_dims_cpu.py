"""CPU side of attention on the wgmma kernels at dqk < dv: dispatch and workspace of the C ABI, the compiler output of the new
kernels (attn_wgmma_mixed_fwd.cu, attn_wgmma_mixed_bwd.cu), and the barrier models at their ring depths.

Without an sm_90 device the wgmma kernels are never selected, so there the dispatch test checks the generic fall-back and
that the refusals do not depend on the device."""
import ctypes as C
import importlib.util
import os

import pytest

from test_attention_deterministic_cpu import HSTU_ERR_UNSUPPORTED, SM90, _params

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PAIRS = [(32, 64), (32, 128), (32, 256), (64, 128), (64, 256), (128, 256)]


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


def _delta(p, B, delta):
    p.batch, p.delta_q_len = B, delta
    return p


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("dqk,dv", PAIRS)
def test_mixed_dims_dispatch(lib, dtype, dqk, dv):
    from generative_recommenders_b200 import _lib

    code = _lib.BF16 if dtype == "bf16" else _lib.F16
    umma = _lib.IMPL_UMMA if SM90 else _lib.IMPL_GENERIC
    # forward and non-deterministic backward: the wgmma kernels, no workspace
    for bwd in (0, 1):
        p = _params(code, dqk, dv, deterministic=0)
        assert lib.hstu_attn_select_impl(C.byref(p), bwd) == umma
        assert lib.hstu_attn_workspace_bytes(C.byref(p), bwd) == 0
    # delta-q: one chunk at B = 128, H = 2 (256 CTAs); at B = 1 the keys of the 2048-row sequences split into 4 chunks, whose
    # fp32 partials are chunks * B * delta * H * dv * 4 bytes
    assert lib.hstu_attn_select_impl(C.byref(_delta(_params(code, dqk, dv, deterministic=0), 128, 16)), 0) == umma
    if SM90:
        assert lib.hstu_attn_workspace_bytes(C.byref(_delta(_params(code, dqk, dv, deterministic=0), 128, 16)), 0) == 0
        assert lib.hstu_attn_workspace_bytes(C.byref(_delta(_params(code, dqk, dv, deterministic=0), 1, 16)), 0) == 4 * 1 * 16 * 2 * dv * 4
    # deterministic = 1 stays on the generic kernels, forcing the wgmma kernels with it is refused, and it needs no workspace
    assert lib.hstu_attn_select_impl(C.byref(_params(code, dqk, dv)), 1) == _lib.IMPL_GENERIC
    assert lib.hstu_attn_select_impl(C.byref(_params(code, dqk, dv, impl=_lib.IMPL_UMMA)), 1) == HSTU_ERR_UNSUPPORTED
    assert lib.hstu_attn_workspace_bytes(C.byref(_params(code, dqk, dv)), 1) == 0
    # dqk > dv stays generic in every direction, and forcing the wgmma kernels there is refused
    for bwd in (0, 1):
        assert lib.hstu_attn_select_impl(C.byref(_params(code, dv, dqk, deterministic=0)), bwd) == _lib.IMPL_GENERIC
        assert lib.hstu_attn_select_impl(C.byref(_params(code, dv, dqk, deterministic=0, impl=_lib.IMPL_UMMA)), bwd) == HSTU_ERR_UNSUPPORTED
    # fp32 and a relative bias keep the generic kernels
    assert lib.hstu_attn_select_impl(C.byref(_params(_lib.F32, dqk, dv, deterministic=0)), 1) == _lib.IMPL_GENERIC
    assert lib.hstu_attn_select_impl(C.byref(_params(code, dqk, dv, deterministic=0, bias=True)), 0) == _lib.IMPL_GENERIC


def test_dims_outside_the_set_stay_generic(lib):
    from generative_recommenders_b200 import _lib

    for dqk, dv in ((16, 64), (32, 96), (48, 128)):
        assert lib.hstu_attn_select_impl(C.byref(_params(_lib.BF16, dqk, dv, deterministic=0)), 0) == _lib.IMPL_GENERIC


# ---- compiler output of the dqk < dv kernels (needs nvcc, no GPU) ----
sass_report = _load("sass_report")
SERIALISATION = ("C7510", "C7512", "C7515")
KERNELS = ("attn_fwd_mixed_wgmma_kernel", "attn_fwd_delta_mixed_wgmma_kernel", "attn_bwd_dkdv_mixed_wgmma_kernel",
           "attn_bwd_dq_mixed_wgmma_kernel")


@pytest.fixture(scope="module")
def report():
    if sass_report.tools() is None:
        pytest.skip("nvcc / cuobjdump not installed")
    return sass_report.report()


@pytest.mark.parametrize("bf16", [0, 1])
@pytest.mark.parametrize("dqk,dv", PAIRS)
@pytest.mark.parametrize("kernel", KERNELS)
def test_mixed_dims_kernel_compiler_output(report, kernel, dqk, dv, bf16):
    """No spills, no wgmma serialisation, at most 255 registers (128 for the forward at dv = 64, which runs two CTAs per
    SM), and an elementwise stage whose tanh ptxas can overlap.  Shared memory is checked by static_asserts."""
    name = f"{kernel}<(int){dqk}, (int){dv}, (bool){bf16}>"
    found = [r for n, r in report.items() if name in n]
    assert len(found) == 1, (name, sorted(report))
    r = found[0]
    assert r["spill_stores"] == 0 and r["spill_loads"] == 0, r
    assert not set(r["notes"]) & set(SERIALISATION), r
    assert r["registers"] <= (128 if "fwd" in kernel and dv == 64 else 255), r
    assert r["tanh_per_block"] >= 8, r


# ---- barrier models at the ring depths of the dqk < dv kernels ----
# forward: FwdCfg<dqk, dv>::STAGES = 3, with the merged MMA batch at dv <= 64 (the model's d = 64) and without it above
# (d = 128); dK / dV: BwdCfg<dqk, dv, false>::STAGES = 4; dQ: DqCfg<dqk, dv>::STAGES = 3
bwd_model = _load("sim_bwd_protocol")
fwd_model = _load("sim_fwd_protocol")
TILES = (1, 2, 3, 4, 5, 8, 13, 64)


def test_mixed_dims_protocols_at_their_ring_depths():
    assert fwd_model.STAGES[64] == fwd_model.STAGES[128] == 3
    assert bwd_model.DKDV_STAGES == 4 and fwd_model.DQ_STAGES == 3
    for tiles in TILES:
        for seed in range(25):
            for straddle in (False, True):
                for d in (64, 128):
                    fwd_model.run(tiles, d, seed, straddle=straddle)
                    fwd_model.run_delta(tiles, d, seed, straddle=straddle)
                bwd_model.run_dkdv(tiles, seed, stages=4, straddle=straddle)
                fwd_model.run_dq(tiles, seed, stages=3, straddle=straddle)


@pytest.mark.parametrize("brk", ["break_release", "first_releaser", "early_release", "break_zero"])
def test_mixed_dims_dkdv_model_catches_its_seeded_breaks(brk):
    with pytest.raises(bwd_model.Violation):
        for seed in range(200):
            bwd_model.run_dkdv(8, seed, stages=4, **{brk: True})


@pytest.mark.parametrize("brk", ["break_k_refill", "first_releaser", "early_release", "break_zero"])
def test_mixed_dims_dq_model_catches_its_seeded_breaks(brk):
    with pytest.raises(fwd_model.Violation):
        for seed in range(200):
            fwd_model.run_dq(8, seed, stages=3, **{brk: True})


@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("brk", ["break_refill", "first_releaser", "break_zero"])
def test_mixed_dims_fwd_model_catches_its_seeded_breaks(d, brk):
    with pytest.raises(fwd_model.Violation):
        for seed in range(200):
            fwd_model.run(8, d, seed, **{brk: True})
