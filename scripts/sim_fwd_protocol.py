#!/usr/bin/env python3
"""Discrete simulation of the synchronisation protocol of attn_fwd_wgmma_kernel (csrc/attn_wgmma_fwd.cu) on the CPU, on the
engine of sim_bwd_protocol.py: no deadlock, no mbarrier parity aliasing, and no TMA load into a K or V stage that a warp
still reads.

Actors: the eight warps W0..W7.  Thread 0 (in W0) issues the TMA loads of Q and of the first STAGES key tiles; afterwards
each warp releases the K (V) stage of tile i once its MMAs that read it have completed, and the warp whose release is the last
of the eight loads tile i + STAGES into the stage.  With d <= 64 the MMAs O += P_i V_i and S_{i+1} = Q K_{i+1}^T form one
batch with one wait, so V_i and K_{i+1} are read together and released together.
usage: sim_fwd_protocol.py [--d 32|64|128|256] [--tiles T] [--seeds N] [--break-refill]"""
import argparse
import importlib.util
import os
import random

_spec = importlib.util.spec_from_file_location("sim_bwd_protocol", os.path.join(os.path.dirname(os.path.abspath(__file__)),
                                                                                 "sim_bwd_protocol.py"))
_eng = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(_eng)
Bar, Violation, Release, WARPS, release, zero_rows = (_eng.Bar, _eng.Violation, _eng.Release, _eng.WARPS, _eng.release,
                                                      _eng.zero_rows)

STAGES = {32: 3, 64: 3, 128: 3, 256: 2}  # FwdCfg<D>::STAGES


def run(T, d, seed, break_refill=False, first_releaser=False, early_release=False, straddle=True, break_zero=False):
    """One query-tile CTA over T key tiles; with `straddle` the last key tile crosses the sequence end, and all warps zero
    its V rows past the end and meet at a named barrier before O += P V reads them.  Seeded breaks (each must be caught):
      break_zero                    no named barrier between that zeroing and the MMAs;
      break_refill, first_releaser  the first warp to release a stage refills it;
      early_release                 (d <= 64) K_{i+1} is released before the wait of the batch that reads it."""
    NST = STAGES[d]
    merge = d <= 64
    refill_at = 1 if (break_refill or first_releaser) else WARPS
    rnd = random.Random(seed)
    B = {"q": Bar(1), "zb": Bar(WARPS)}
    R = {}
    for i in range(NST):
        B[f"kf{i}"], B[f"vf{i}"] = Bar(1), Bar(1)
        R[f"k{i}"], R[f"v{i}"] = Release(refill_at), Release(refill_at)

    def rel(kind, i):  # release of stage K / V of tile i; the refilling warp loads tile i + NST
        if i + NST < T:
            st = i % NST
            yield from release(R[f"{kind}{st}"], [("tma", f"{kind}f{st}", f"{kind}{st}")])

    def W(w):
        if w == 0:
            yield ("async", "q")
            for i in range(min(T, NST)):
                yield ("tma", f"kf{i}", f"k{i}")
                yield ("tma", f"vf{i}", f"v{i}")
        yield ("wait", "q", 0)
        yield ("wait", "kf0", 0)
        yield ("read", "k0", 1)                      # S_0, waited for
        yield ("read", "k0", -1)
        yield from rel("k", 0)
        for i in range(T):
            st, nst = i % NST, (i + 1) % NST
            nxt = i + 1 < T
            yield ("wait", f"vf{st}", i // NST)
            if straddle and not nxt:
                yield from zero_rows(f"v{st}", "zb", 0, break_zero)
            if merge and nxt:
                yield ("wait", f"kf{nst}", (i + 1) // NST)
            yield ("read", f"v{st}", 1)              # O += P_i V_i ...
            if merge and nxt:
                yield ("read", f"k{nst}", 1)         # ... and S_{i+1} in the same batch
                if early_release:
                    yield from rel("k", i + 1)
            yield ("read", f"v{st}", -1)             # one wait for the batch
            if merge and nxt:
                yield ("read", f"k{nst}", -1)
            yield from rel("v", i)
            if not merge and nxt:                    # d >= 128: S_{i+1} in a batch of its own
                yield ("wait", f"kf{nst}", (i + 1) // NST)
                yield ("read", f"k{nst}", 1)
                yield ("read", f"k{nst}", -1)
            if nxt and not (merge and early_release):
                yield from rel("k", i + 1)

    return _eng._simulate({f"W{w}": W(w) for w in range(WARPS)}, B, rnd)


DQ_STAGES = 3  # DqCfg<D>::STAGES (csrc/attn_wgmma_bwd.cu, every d)


def run_dq(T, seed, break_k_refill=False, first_releaser=False, early_release=False, straddle=True, break_zero=False,
           stages=DQ_STAGES):
    """attn_bwd_dq_wgmma_kernel: the forward's ring (`stages` deep) with Q and dO resident; S / dP read K and V and are waited for,
    V is released, then dQ += dS K reads K, is waited for, and K is released.  With `straddle` the last key tile crosses the
    sequence end, and all warps zero its K rows past the end and meet at a named barrier first.  Seeded breaks (each must be
    caught):
      break_zero      no named barrier between that zeroing and the MMAs;
      break_k_refill  the K stage is refilled by the warp that completes the release of V (after S / dP) instead of K, so
                      the load may land while another warp's dQ MMA still reads K;
      first_releaser  the first warp to release a stage refills it;
      early_release   K is released before the wait of the dQ MMAs that read it."""
    NST = stages
    refill_at = 1 if first_releaser else WARPS
    rnd = random.Random(seed)
    B = {"qd": Bar(1), "zb": Bar(WARPS)}
    R = {}
    for i in range(NST):
        B[f"kf{i}"], B[f"vf{i}"] = Bar(1), Bar(1)
        R[f"k{i}"], R[f"v{i}"] = Release(refill_at), Release(refill_at)

    def W(w):
        if w == 0:
            yield ("async", "qd")
            for i in range(min(T, NST)):
                yield ("tma", f"kf{i}", f"k{i}")
                yield ("tma", f"vf{i}", f"v{i}")
        yield ("wait", "qd", 0)
        for i in range(T):
            st = i % NST
            k_load, v_load = [("tma", f"kf{st}", f"k{st}")], [("tma", f"vf{st}", f"v{st}")]
            yield ("wait", f"kf{st}", i // NST)
            yield ("wait", f"vf{st}", i // NST)
            if straddle and i == T - 1:
                yield from zero_rows(f"k{st}", "zb", 0, break_zero)
            yield ("read", f"k{st}", 1)          # S = Q K^T and dP = dO V^T, waited for
            yield ("read", f"v{st}", 1)
            yield ("read", f"v{st}", -1)
            if i + NST < T:
                yield from release(R[f"v{st}"], v_load + (k_load if break_k_refill else []))
            yield ("read", f"k{st}", -1)
            yield ("read", f"k{st}", 1)          # dQ += dS K ...
            if early_release and i + NST < T:
                yield from release(R[f"k{st}"], k_load)
            yield ("read", f"k{st}", -1)         # ... waited for
            if not early_release and not break_k_refill and i + NST < T:
                yield from release(R[f"k{st}"], k_load)

    return _eng._simulate({f"W{w}": W(w) for w in range(WARPS)}, B, rnd)


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
