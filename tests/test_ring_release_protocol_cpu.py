"""The ring protocol of the wgmma attention kernels without a waiting producer, model-checked on the CPU: every warp releases a
K / V (forward, dQ) or Q / dO (dK/dV) stage once the MMAs that read it have completed, and the warp whose release is the
last of the eight refills the stage (scripts/sim_fwd_protocol.py run / run_dq, scripts/sim_bwd_protocol.py run_dkdv).  Each
model is shown to catch the two ways this protocol can be broken: a refill by the first warp to release, and a release
before the wait of the MMAs that read the stage."""
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
Violation = (fwd.Violation, bwd.Violation)  # each module loads its own copy of the engine

MODELS = {
    "fwd32": lambda T, s, **kw: fwd.run(T, 32, s, **kw),
    "fwd64": lambda T, s, **kw: fwd.run(T, 64, s, **kw),
    "dq": lambda T, s, **kw: fwd.run_dq(T, s, **kw),
    "dkdv": lambda T, s, **kw: bwd.run_dkdv(T, s, **kw),
}


@pytest.mark.parametrize("model", sorted(MODELS))
def test_release_protocol_holds_under_many_schedules(model):
    for tiles in (1, 2, 3, 4, 6, 9, 17):
        for seed in range(100):
            MODELS[model](tiles, 1000 + seed)


@pytest.mark.parametrize("model", sorted(MODELS))
def test_model_catches_a_refill_by_the_first_releaser(model):
    with pytest.raises(Violation, match="TMA load into|wait on"):
        for seed in range(100):
            MODELS[model](8, seed, first_releaser=True)


@pytest.mark.parametrize("model", sorted(MODELS))
def test_model_catches_a_release_before_the_wait(model):
    """Forward: K_{i+1} released before the wait of the batch that also holds O += P_i V_i; dQ: K_i before the wait of the dQ
    MMAs; dK/dV: Q_j / dO_j before the wait of the dV / dK MMAs.  The refill then lands under an MMA that still reads it."""
    with pytest.raises(Violation, match="TMA load into"):
        for seed in range(100):
            MODELS[model](8, seed, early_release=True)


@pytest.mark.parametrize("d", [128, 256])
def test_unmerged_forward_catches_a_refill_by_the_first_releaser(d):
    with pytest.raises(Violation, match="TMA load into|wait on"):
        for seed in range(100):
            fwd.run(8, d, seed, first_releaser=True)


ZERO_MODELS = dict(MODELS, fused64=lambda T, s, **kw: bwd.run(T, 64, s, **kw),
                   fused128=lambda T, s, **kw: bwd.run(T, 128, s, **kw))


@pytest.mark.parametrize("model", sorted(ZERO_MODELS))
def test_zeroing_rows_past_the_sequence_end_holds_under_many_schedules(model):
    """All warps zero the rows past the sequence end of the tile that crosses it (the last key tile of the forward and the dQ
    kernel; the key tile and the last query tile of the key-stationary kernels), then meet at one named barrier."""
    for straddle in (False, True):
        for tiles in (1, 2, 3, 4, 5, 9):
            for seed in range(60):
                ZERO_MODELS[model](tiles, 2000 + seed, straddle=straddle)


@pytest.mark.parametrize("model", sorted(ZERO_MODELS))
def test_model_catches_zeroing_without_the_barrier(model):
    with pytest.raises(Violation, match="while it is being (written|read)"):
        for seed in range(200):
            for tiles in (1, 3):
                ZERO_MODELS[model](tiles, seed, break_zero=True)
