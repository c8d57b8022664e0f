"""The synchronisation protocol of the wgmma backward kernel, model-checked on the CPU under random schedules
(scripts/sim_bwd_protocol.py mirrors the mbarrier waits / arrives, TMA loads, named barrier and dS buffers of
csrc/attn_wgmma_bwd.cu for d = 32, 64, 128)."""
import importlib.util
import os

import pytest

_spec = importlib.util.spec_from_file_location(
    "sim_bwd_protocol", os.path.join(os.path.dirname(__file__), "..", "scripts", "sim_bwd_protocol.py"))
sim = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(sim)


@pytest.mark.parametrize("d", [32, 64, 128])
def test_protocol_has_no_deadlock_or_phase_aliasing(d):
    for tiles in (1, 2, 3, 4, 5, 8, 13, 64):
        for seed in range(25):
            sim.run(tiles, d, seed)


@pytest.mark.parametrize("d", [32, 64, 128])
def test_model_catches_a_single_ds_buffer(d):
    """With one dS buffer instead of two, a warpgroup overwrites dS while the other one's dQ MMA still reads it."""
    with pytest.raises(sim.Violation, match="ds0"):
        for seed in range(100):
            sim.run(8, d, seed, break_ds=True)
