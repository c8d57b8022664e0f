#!/usr/bin/env python3
"""Discrete simulation of the synchronisation protocol of attn_bwd_wgmma_kernel (csrc/attn_wgmma_bwd.cu) on the CPU.

Checks, under random schedules, that (1) nobody deadlocks, (2) no mbarrier parity wait "passes falsely" -- a waiter asking
for phase k while phase k-1 has not completed sees the parity test succeed at once --, (3) no waiter falls two phases behind,
(4) no TMA load is issued into a Q / dO stage that a warpgroup still reads, and (5) no dS buffer is written while the dQ
MMA of an earlier tile reads it, or read while it is written.

Actors: the eight warps W0..W7 of the two warpgroups (W0-W3 and W4-W7).  Thread 0 (in W0) issues the first TMA loads; after
that a stage is refilled by the warp whose release completes it (Release, below), so nobody waits for a free stage.
TMA completions are asynchronous: queued per issuing actor and fired later, in order.
usage: sim_bwd_protocol.py [--d 32|64|128] [--tiles T] [--seeds N] [--break-ds]"""
import argparse
import random

STAGES = {32: 4, 64: 3, 128: 2}  # BwdCfg<D>::STAGES


class Bar:
    def __init__(self, count):
        self.count, self.pending, self.phase = count, count, 0

    def arrive(self):
        self.pending -= 1
        if self.pending == 0:
            self.pending, self.phase = self.count, self.phase + 1


class Violation(Exception):
    pass


WARPS = 8  # one release per warp and use of a stage (release_is_last<8> in csrc/wgmma.cuh)


class Release:
    """Release counter of one ring stage: WARPS arrivals per use, and arrival number `refill_at` of a use (the last one in the
    kernels) is told to refill the stage.  A smaller `refill_at` seeds a break."""

    def __init__(self, refill_at=WARPS):
        self.refill_at, self.n = refill_at, 0

    def arrive(self):
        self.n += 1
        return (self.n - 1) % WARPS + 1 == self.refill_at


def zero_rows(res, barrier, phase, skip_barrier=False):
    """All eight warps zero the rows past the sequence end of stage `res` (zero_tile_rows, csrc/wgmma.cuh: plain stores, then
    fence.proxy.async), then meet at the CTA-wide named barrier `barrier` before any MMA reads the stage.  skip_barrier seeds
    the break of reading the stage without the barrier."""
    yield ("write", res, 1)
    yield ("write", res, -1)
    if not skip_barrier:
        yield ("arrive", barrier)
        yield ("wait", barrier, phase)


def release(ctr, refill):
    """One warp's release of a stage (an atomic step); if it is the refilling arrival, the warp then issues `refill` (a list of
    ops, usually TMA loads)."""
    got = []
    yield ("call", lambda: got.append(ctr.arrive()))
    if got[0]:
        yield from refill


def _simulate(actors, B, rnd):
    pending = {k: None for k in actors}
    queues = {k: [] for k in actors}
    readers, writers = {}, {}   # resource -> number of actors inside a read / write of it
    done = set()
    steps = 0
    while len(done) < len(actors) or any(queues.values()):
        steps += 1
        if steps > 400000:
            raise Violation("no progress (livelock?)")
        choices = [("run", k) for k in actors if k not in done] + [("fire", k) for k, q in queues.items() if q]
        rnd.shuffle(choices)
        progressed = False
        for kind, k in choices:
            if kind == "fire":
                B[queues[k].pop(0)].arrive()
                progressed = True
                break
            if pending[k] is None:
                try:
                    pending[k] = next(actors[k])
                except StopIteration:
                    done.add(k)
                    progressed = True
                    break
            op = pending[k]
            if op[0] == "wait":
                _, name, want = op
                bar = B[name]
                passes = (bar.phase & 1) != (want & 1)
                if passes and bar.phase <= want:
                    raise Violation(f"{k}: wait on {name} for phase {want} passed while the barrier is in phase {bar.phase} (false pass)")
                if not passes and bar.phase > want:
                    raise Violation(f"{k}: wait on {name} for phase {want} but the barrier is already in phase {bar.phase} (two ahead)")
                if not passes:
                    continue
            elif op[0] == "arrive":
                B[op[1]].arrive()
            elif op[0] == "call":        # an atomic step of the actor's own (a shared-memory atomic)
                op[1]()
            elif op[0] == "async":
                queues[k].append(op[1])
            elif op[0] == "tma":          # TMA load into stage op[2], completing on barrier op[1]
                if readers.get(op[2], 0):
                    raise Violation(f"{k}: TMA load into {op[2]} while it is being read")
                if writers.get(op[2], 0):
                    raise Violation(f"{k}: TMA load into {op[2]} while it is being written")
                queues[k].append(op[1])
            elif op[0] in ("read", "write"):
                _, res, delta = op
                if op[0] == "read":
                    if writers.get(res, 0):
                        raise Violation(f"{k}: reads {res} while it is being written")
                    readers[res] = readers.get(res, 0) + delta
                else:
                    if readers.get(res, 0):
                        raise Violation(f"{k}: writes {res} while it is being read")
                    writers[res] = writers.get(res, 0) + delta
            pending[k] = None
            progressed = True
            break
        if not progressed:
            state = {k: pending[k] for k in actors if k not in done}
            raise Violation(f"deadlock: {state}")
    return steps


def run(T, d, seed, break_ds=False, straddle=True, break_zero=False):
    """One key-tile CTA streaming T query tiles.  straddle: the key tile and the last query tile cross the sequence end, so K
    and that Q_j / dO_j stage get their rows past it zeroed.  Seeded breaks (each must be caught): break_ds, one dS buffer
    instead of two; break_zero, no named barrier between the zeroing and the MMAs."""
    NST = STAGES[d]
    NDS = 1 if break_ds else 2
    rnd = random.Random(seed)
    B = {"kv": Bar(1), "nb": Bar(WARPS), "zb": Bar(WARPS)}
    R = {}
    for i in range(NST):
        B[f"qf{i}"] = Bar(1)   # expect_tx arrival of the loading thread + TMA bytes: modelled as the TMA completion
        R[i] = Release()

    def W(w):
        if w == 0:                                   # thread 0: K / V and the first STAGES query tiles
            yield ("async", "kv")
            for j in range(min(T, NST)):
                yield ("tma", f"qf{j % NST}", f"q{j % NST}")
        yield ("wait", "kv", 0)
        if straddle:
            yield from zero_rows("k", "zb", 0, break_zero)
        for j in range(T):
            st = j % NST
            yield ("wait", f"qf{st}", j // NST)
            if straddle and j == T - 1:
                yield from zero_rows(f"q{st}", "zb", 1, break_zero)
            yield ("read", f"q{st}", 1)              # S^T, dP^T, dV, dK MMAs read Q_j / dO_j ...
            yield ("read", f"q{st}", -1)             # ... and complete within the iteration
            if j + NST < T:                          # the last warp to release the stage refills it
                yield from release(R[st], [("tma", f"qf{st}", f"q{st}")])
            b = f"ds{j % NDS}"
            yield ("write", b, 1)                    # dS^T of this warp's 16 keys
            yield ("write", b, -1)
            yield ("arrive", "nb")                   # named barrier of the 256 consumer threads
            yield ("wait", "nb", j)
            if j % 2 == w // 4:                      # dQ_j = dS K by warpgroup j % 2, waited for before the warp goes on
                yield ("read", b, 1)
                yield ("read", "k", 1)
                yield ("read", "k", -1)
                yield ("read", b, -1)

    return _simulate({f"W{w}": W(w) for w in range(WARPS)}, B, rnd)


DKDV_STAGES = 4  # BwdCfg<D, false>::STAGES (every d)


def run_dkdv(T, seed, break_release=False, first_releaser=False, early_release=False, straddle=True, break_zero=False,
             stages=DKDV_STAGES):
    """attn_bwd_dkdv_wgmma_kernel: the key-tile CTA of `run` without dS buffers, dS barrier or dQ, with a ring of `stages`;
    the warps meet at the Q / dO ring and, with `straddle`, once at the named barrier after zeroing the rows of the last
    query tile that lie past the sequence end.  Seeded breaks (each must be caught):
      break_zero      no named barrier between that zeroing and the MMAs;
      break_release   the stage is refilled once four warps (one warpgroup's worth) have released it;
      first_releaser  the first warp to release the stage refills it;
      early_release   a warp releases Q_j / dO_j before the wait of the MMAs that read them."""
    NST = stages
    refill_at = 1 if first_releaser else WARPS // 2 if break_release else WARPS
    rnd = random.Random(seed)
    B = {"kv": Bar(1), "zb": Bar(WARPS)}
    R = {}
    for i in range(NST):
        B[f"qf{i}"] = Bar(1)
        R[i] = Release(refill_at)

    def W(w):
        if w == 0:
            yield ("async", "kv")
            for j in range(min(T, NST)):
                yield ("tma", f"qf{j % NST}", f"q{j % NST}")
        yield ("wait", "kv", 0)
        for j in range(T):
            st = j % NST
            refill = [("tma", f"qf{st}", f"q{st}")]
            yield ("wait", f"qf{st}", j // NST)
            if straddle and j == T - 1:
                yield from zero_rows(f"q{st}", "zb", 0, break_zero)
            yield ("read", f"q{st}", 1)              # S^T, dP^T, dV, dK MMAs ...
            if early_release and j + NST < T:
                yield from release(R[st], refill)
            yield ("read", f"q{st}", -1)             # ... waited for
            if not early_release and j + NST < T:
                yield from release(R[st], refill)

    return _simulate({f"W{w}": W(w) for w in range(WARPS)}, B, rnd)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--d", type=int, default=32, choices=sorted(STAGES))
    ap.add_argument("--tiles", type=int, default=8)
    ap.add_argument("--seeds", type=int, default=200)
    ap.add_argument("--break-ds", action="store_true")
    a = ap.parse_args()
    for s in range(a.seeds):
        run(a.tiles, a.d, s, break_ds=a.break_ds)
    print(f"ok: d={a.d} tiles={a.tiles} seeds={a.seeds}")


if __name__ == "__main__":
    main()
