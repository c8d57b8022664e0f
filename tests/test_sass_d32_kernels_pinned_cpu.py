"""The three d = 32 wgmma attention kernels as the compiler builds them (scripts/sass_report.py; needs nvcc, no GPU): their
registers, no spills, and the instructions of one steady-state tile iteration, pinned at the values of CUDA 12.9 with the
flags of build.py.  The pre-pass and the operand handoff of DESIGN.md 3.0 live outside these kernels and must leave them as
they are; a change to a kernel itself updates these numbers on purpose."""
import importlib.util
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_spec = importlib.util.spec_from_file_location("sass_report", os.path.join(ROOT, "scripts", "sass_report.py"))
sass_report = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(sass_report)

# kernel: (registers, iter_instrs)
PINNED = {
    "attn_fwd_wgmma_kernel<(int)32, (bool)0>": (123, 204),
    "attn_bwd_dq_wgmma_kernel<(int)32, (bool)0>": (128, 279),
    "attn_bwd_dkdv_wgmma_kernel<(int)32, (bool)0>": (127, 427),
}


@pytest.fixture(scope="module")
def report():
    if sass_report.tools() is None:
        pytest.skip("nvcc / cuobjdump not installed")
    return sass_report.report()


@pytest.mark.parametrize("kernel", sorted(PINNED))
def test_d32_kernel_pinned(report, kernel):
    found = [r for name, r in report.items() if kernel in name]
    assert len(found) == 1, (kernel, sorted(report))
    r = found[0]
    assert r["spill_stores"] == 0 and r["spill_loads"] == 0, r
    assert (r["registers"], r["iter_instrs"]) == PINNED[kernel], (kernel, r)
