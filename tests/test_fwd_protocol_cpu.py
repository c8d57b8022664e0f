"""The synchronisation protocol of the wgmma forward kernel, model-checked on the CPU under random schedules
(scripts/sim_fwd_protocol.py mirrors the mbarrier waits / arrives and TMA refills of csrc/attn_wgmma_fwd.cu)."""
import importlib.util
import os

import pytest

_spec = importlib.util.spec_from_file_location(
    "sim_fwd_protocol", os.path.join(os.path.dirname(__file__), "..", "scripts", "sim_fwd_protocol.py"))
sim = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(sim)


@pytest.mark.parametrize("d", [32, 64, 128, 256])
def test_forward_protocol_has_no_deadlock_or_phase_aliasing(d):
    for tiles in (1, 2, 3, 4, 5, 8, 13, 64):
        for seed in range(25):
            sim.run(tiles, d, seed)


@pytest.mark.parametrize("d", [32, 256])
def test_model_catches_a_refill_before_the_release(d):
    """Thread 0 refilling a K / V stage without waiting for both warpgroups to release it is caught."""
    with pytest.raises(sim.Violation):  # an overwrite of a tile in use, or a barrier overrun
        for seed in range(100):
            sim.run(8, d, seed, break_refill=True)
