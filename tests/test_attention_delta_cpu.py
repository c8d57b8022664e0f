"""The delta-q (KV-cached) wgmma forward without a GPU: its ring protocol under random schedules, with the warpgroup of padding
rows that releases stages it never reads (scripts/sim_fwd_protocol.py run_delta), and the compiler output of its kernels
(scripts/sass_report.py; needs nvcc)."""
import importlib.util
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _load(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, "scripts", f"{name}.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


sim = _load("sim_fwd_protocol")
sass_report = _load("sass_report")


@pytest.mark.parametrize("d", [32, 64, 128, 256])
@pytest.mark.parametrize("idle_warps", [0, 4])
def test_delta_protocol_has_no_deadlock_or_phase_aliasing(d, idle_warps):
    for tiles in (1, 2, 3, 4, 5, 8, 13):
        for straddle in (False, True):
            for seed in range(15):
                sim.run_delta(tiles, d, seed, idle_warps=idle_warps, straddle=straddle)


@pytest.mark.parametrize("d", [32, 256])
def test_model_catches_idle_releases_that_do_not_wait_for_the_stage(d):
    """An idle warp that releases a stage before its load has landed can complete the release of the stage's next use while
    an active warp still reads it."""
    with pytest.raises(sim.Violation):
        for seed in range(100):
            sim.run_delta(8, d, seed, break_idle_wait=True)


@pytest.fixture(scope="module")
def report():
    if sass_report.tools() is None:
        pytest.skip("nvcc / cuobjdump not installed")
    return sass_report.report("attn_fwd_delta_wgmma_kernel")


@pytest.mark.parametrize("d", [32, 64, 128, 256])
@pytest.mark.parametrize("bf16", [False, True])
def test_delta_kernel_compiler_output(report, d, bf16):
    found = [r for name, r in report.items() if f"attn_fwd_delta_wgmma_kernel<(int){d}, (bool){int(bf16)}>" in name]
    assert len(found) == 1, sorted(report)
    r = found[0]
    assert r["spill_stores"] == 0 and r["spill_loads"] == 0, r
    assert not set(r["notes"]) & {"C7510", "C7512", "C7515"}, r  # no wgmma serialisation
    assert r["tanh_per_block"] >= 8, r
    if d <= 64:
        assert r["registers"] <= 128, r  # two CTAs per SM
