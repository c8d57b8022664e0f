#!/usr/bin/env python3
"""Discrete simulation of the synchronisation protocol of attn_fwd_wgmma_kernel (csrc/attn_wgmma_fwd.cu) on the CPU, on the
engine of sim_bwd_protocol.py: no deadlock, no mbarrier parity aliasing, and no TMA load into a K or V stage that a warpgroup
still reads.

Actors: the two warpgroups W0 / W1 (one arrival each on the 256-count empty barriers); thread 0 of W0 issues the TMA loads of
Q, of the first STAGES key tiles and, once both warpgroups have released stage i % STAGES, of key tile i + STAGES.
usage: sim_fwd_protocol.py [--d 32|64|128|256] [--tiles T] [--seeds N] [--break-refill]"""
import argparse
import importlib.util
import os
import random

_spec = importlib.util.spec_from_file_location("sim_bwd_protocol", os.path.join(os.path.dirname(os.path.abspath(__file__)),
                                                                                 "sim_bwd_protocol.py"))
_eng = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(_eng)
Bar, Violation = _eng.Bar, _eng.Violation

STAGES = {32: 3, 64: 3, 128: 3, 256: 2}  # FwdCfg<D>::STAGES


def run(T, d, seed, break_refill=False):
    """One query-tile CTA over T key tiles.  break_refill: thread 0 refills a stage without waiting for its release."""
    NST = STAGES[d]
    rnd = random.Random(seed)
    B = {"q": Bar(1)}
    for i in range(NST):
        B[f"kf{i}"], B[f"vf{i}"] = Bar(1), Bar(1)
        B[f"ke{i}"], B[f"ve{i}"] = Bar(2), Bar(2)

    def load(i):
        st = i % NST
        if i >= NST and not break_refill:
            yield ("wait", f"ke{st}", i // NST - 1)
        yield ("tma", f"kf{st}", f"k{st}")
        if i >= NST and not break_refill:
            yield ("wait", f"ve{st}", i // NST - 1)
        yield ("tma", f"vf{st}", f"v{st}")

    def W(w):
        if w == 0:
            yield ("async", "q")
            for i in range(min(T, NST)):
                yield from load(i)
        yield ("wait", "q", 0)
        for i in range(T):
            st = i % NST
            yield ("wait", f"kf{st}", i // NST)
            yield ("read", f"k{st}", 1)          # S = Q K^T, waited for
            yield ("read", f"k{st}", -1)
            yield ("arrive", f"ke{st}")
            yield ("wait", f"vf{st}", i // NST)
            yield ("read", f"v{st}", 1)          # O += P V, waited for
            yield ("read", f"v{st}", -1)
            yield ("arrive", f"ve{st}")
            if w == 0 and i + NST < T:
                yield from load(i + NST)

    return _eng._simulate({"W0": W(0), "W1": W(1)}, B, rnd)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--d", type=int, default=32, choices=sorted(STAGES))
    ap.add_argument("--tiles", type=int, default=8)
    ap.add_argument("--seeds", type=int, default=200)
    ap.add_argument("--break-refill", action="store_true")
    a = ap.parse_args()
    for s in range(a.seeds):
        run(a.tiles, a.d, s, break_refill=a.break_refill)
    print(f"ok: d={a.d} tiles={a.tiles} seeds={a.seeds}")


if __name__ == "__main__":
    main()
