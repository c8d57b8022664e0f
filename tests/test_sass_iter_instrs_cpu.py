"""Bookkeeping guard of the d = 32 wgmma attention kernels (scripts/sass_report.py, iter_instrs; needs nvcc, no GPU).

iter_instrs counts the instructions one thread issues in one steady-state tile iteration on the full-tile path.  About
half of it is the elementwise stage (one tanh per score and its FMAs), which these bounds leave alone; the rest is ring,
descriptor and branch bookkeeping around the MMAs, which the bounds keep from creeping back (DESIGN.md section 3.1).
"""
import importlib.util
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_spec = importlib.util.spec_from_file_location("sass_report", os.path.join(ROOT, "scripts", "sass_report.py"))
sass_report = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(sass_report)

# upper bounds at the values the current kernels compile to (CUDA 12.9, the flags of build.py)
ITER_BOUNDS = {
    "attn_fwd_wgmma_kernel<(int)32,": 204,
    "attn_bwd_dq_wgmma_kernel<(int)32,": 279,
    "attn_bwd_dkdv_wgmma_kernel<(int)32,": 427,
}


@pytest.fixture(scope="module")
def report():
    if sass_report.tools() is None:
        pytest.skip("nvcc / cuobjdump not installed")
    return sass_report.report()


@pytest.mark.parametrize("kernel", sorted(ITER_BOUNDS))
def test_d32_iter_instrs(report, kernel):
    found = [r for name, r in report.items() if kernel in name]
    assert len(found) == 1, (kernel, sorted(report))
    n = found[0]["iter_instrs"]
    assert n is not None and n <= ITER_BOUNDS[kernel], (kernel, n, ITER_BOUNDS[kernel])


def test_iter_instrs_path():
    # tile loop 0x10 .. 0xd0: the spin loop (0x20 -> 0x20) counts once; the masked case (0x80, fewer tanh) and the refill
    # (0xc0) are off the path, and the path with the HGMMA is taken over the shorter one that skips it (0x90 -> 0xb0)
    sass = """
        /*0000*/                   MOV R0, RZ ;
        /*0010*/                   IADD3 R1, R1, 0x1, RZ ;
        /*0020*/                   SYNCS.PHASECHK.TRANS64.TRYWAIT P0, [R2], R3 ;
        /*0030*/              @!P0 BRA 0x20 ;
        /*0040*/               @P1 BRA 0x80 ;
        /*0050*/                   MUFU.TANH R4, R4 ;
        /*0060*/                   MUFU.TANH R5, R5 ;
        /*0070*/                   BRA 0x90 ;
        /*0080*/                   MUFU.TANH R4, R4 ;
        /*0090*/               @P2 BRA 0xb0 ;
        /*00a0*/                   HGMMA.64x32x16.F32 R8, R4, gdesc[UR4], R8 ;
        /*00b0*/               @P3 BRA 0xd0 ;
        /*00c0*/                   ATOMS.ADD R6, [R7], R6 ;
        /*00d0*/              @!P4 BRA 0x10 ;
        /*00e0*/                   EXIT ;
        /*00f0*/                   NOP ;
    """
    # 0x10, 0x20 and 0x30 (one try-wait), 0x40, 0x50 .. 0x70, 0x90, 0xa0, 0xb0, 0xd0
    assert sass_report.iter_instrs(sass) == 11
