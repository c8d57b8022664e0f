"""Compiler-output guard of the d = 32 wgmma attention kernels (scripts/sass_report.py; needs nvcc, no GPU).

The elementwise stage issues one tanh per score.  It must stay free of per-score branches, so that the tanh of a thread's
scores share a basic block and ptxas can overlap their latency (DESIGN.md section 3.2); and each kernel must keep the
register budget of two CTAs per SM without spilling.
"""
import importlib.util
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_spec = importlib.util.spec_from_file_location("sass_report", os.path.join(ROOT, "scripts", "sass_report.py"))
sass_report = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(sass_report)

D32_KERNELS = ("attn_fwd_wgmma_kernel<(int)32,", "attn_bwd_dkdv_wgmma_kernel<(int)32,", "attn_bwd_dq_wgmma_kernel<(int)32,")
SERIALISATION = ("C7510", "C7512", "C7515")


@pytest.fixture(scope="module")
def report():
    if sass_report.tools() is None:
        pytest.skip("nvcc / cuobjdump not installed")
    return sass_report.report()


@pytest.mark.parametrize("kernel", D32_KERNELS)
def test_d32_kernel_schedule(report, kernel):
    found = [r for name, r in report.items() if kernel in name]
    assert len(found) == 1, (kernel, sorted(report))
    r = found[0]
    assert r["tanh_per_block"] >= 8, r
    assert r["spill_stores"] == 0 and r["spill_loads"] == 0, r
    assert r["registers"] <= 128, r
    assert not set(r["notes"]) & set(SERIALISATION), r


def test_block_count_sees_branches():
    # two tanh separated by a predicated branch are two blocks; the branch target starts a third
    sass = """
        /*0000*/                   MUFU.TANH R1, R0 ;
        /*0010*/                   MUFU.TANH R2, R0 ;
        /*0020*/              @!P0 BRA 0x50 ;
        /*0030*/                   MUFU.TANH R3, R0 ;
        /*0040*/                   FMUL R3, R3, R3 ;
        /*0050*/                   MUFU.TANH R4, R0 ;
        /*0060*/                   MUFU.TANH R5, R0 ;
        /*0070*/                   MUFU.TANH R6, R0 ;
        /*0080*/                   EXIT ;
    """
    assert sass_report.max_tanh_per_block(sass) == 3
