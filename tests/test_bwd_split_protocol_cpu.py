"""The synchronisation protocols of the two d = 32 backward kernels, model-checked on the CPU under random schedules:
attn_bwd_dkdv_wgmma_kernel (scripts/sim_bwd_protocol.py, run_dkdv) and attn_bwd_dq_wgmma_kernel
(scripts/sim_fwd_protocol.py, run_dq), both in csrc/attn_wgmma_bwd.cu."""
import importlib.util
import os

import pytest


def _load(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(os.path.dirname(__file__), "..", "scripts", f"{name}.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


bwd = _load("sim_bwd_protocol")
fwd = _load("sim_fwd_protocol")

TILES = (1, 2, 3, 4, 5, 8, 13, 64)


def test_dkdv_protocol_has_no_deadlock_or_phase_aliasing():
    for tiles in TILES:
        for seed in range(25):
            bwd.run_dkdv(tiles, seed)


def test_dq_protocol_has_no_deadlock_or_phase_aliasing():
    for tiles in TILES:
        for seed in range(25):
            fwd.run_dq(tiles, seed)


def test_dkdv_model_catches_a_refill_after_one_release():
    """Thread 0 refilling a Q / dO stage once only its own warpgroup has released it overwrites a tile the other reads, or
    completes a phase of the stage's full barrier that the other warpgroup has not waited for yet."""
    with pytest.raises(bwd.Violation, match="TMA load into q|wait on qf"):
        for seed in range(100):
            bwd.run_dkdv(8, seed, break_release=True)


def test_dq_model_catches_a_k_refill_before_the_dq_mma():
    """A K refill that waits for the release of V (after S / dP) instead of K (after dQ) lands under a dQ MMA."""
    with pytest.raises(fwd.Violation, match="TMA load into k|wait on kf"):
        for seed in range(100):
            fwd.run_dq(8, seed, break_k_refill=True)
