#!/usr/bin/env python3
"""Discrete simulation of the synchronisation protocol of attn_bwd_wgmma_kernel (csrc/attn_wgmma_bwd.cu) on the CPU.

Checks, under random schedules, that (1) nobody deadlocks, (2) no mbarrier parity wait "passes falsely" -- a waiter asking
for phase k while phase k-1 has not completed sees the parity test succeed at once --, (3) no waiter falls two phases behind,
(4) no TMA load is issued into a Q / dO stage that a warpgroup still reads, and (5) no dS buffer is written while the dQ
MMA of an earlier tile reads it, or read while it is written.

Actors: the two warpgroups W0 / W1 (128 threads each, modelled as one arrival each); thread 0 of W0 also issues the TMA loads.
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
            elif op[0] == "async":
                queues[k].append(op[1])
            elif op[0] == "tma":          # TMA load into stage op[2], completing on barrier op[1]
                if readers.get(op[2], 0):
                    raise Violation(f"{k}: TMA load into {op[2]} while it is being read")
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


def run(T, d, seed, break_ds=False):
    """One key-tile CTA streaming T query tiles.  break_ds: one dS buffer instead of two (must be caught)."""
    NST = STAGES[d]
    NDS = 1 if break_ds else 2
    rnd = random.Random(seed)
    B = {"kv": Bar(1), "nb": Bar(2)}
    for i in range(NST):
        B[f"qf{i}"] = Bar(1)   # expect_tx arrival of thread 0 + TMA bytes: modelled as the TMA completion
        B[f"qe{i}"] = Bar(2)   # 256 consumer threads: one arrival per warpgroup

    def W(w):
        if w == 0:                                   # thread 0: K / V and the first STAGES query tiles
            yield ("async", "kv")
            for j in range(min(T, NST)):
                yield ("tma", f"qf{j % NST}", f"q{j % NST}")
        yield ("wait", "kv", 0)
        for j in range(T):
            st = j % NST
            yield ("wait", f"qf{st}", j // NST)
            yield ("read", f"q{st}", 1)              # S^T, dP^T, dV, dK MMAs read Q_j / dO_j ...
            yield ("read", f"q{st}", -1)             # ... and complete within the iteration
            yield ("arrive", f"qe{st}")
            if w == 0 and j + NST < T:               # refill the stage once both warpgroups have released it
                yield ("wait", f"qe{st}", j // NST)
                yield ("tma", f"qf{st}", f"q{st}")
            b = f"ds{j % NDS}"
            yield ("write", b, 1)                    # dS^T of this warpgroup's 64 keys
            yield ("write", b, -1)
            yield ("arrive", "nb")                   # named barrier of the 256 consumer threads
            yield ("wait", "nb", j)
            if j % 2 == w:                           # dQ_j = dS K, waited for before the warpgroup goes on
                yield ("read", b, 1)
                yield ("read", b, -1)

    return _simulate({"W0": W(0), "W1": W(1)}, B, rnd)


DKDV_STAGES = 4  # BwdCfg<32, false>::STAGES


def run_dkdv(T, seed, break_release=False):
    """attn_bwd_dkdv_wgmma_kernel (d = 32): the key-tile CTA of `run` without dS buffers, named barrier or dQ; the two
    warpgroups meet only at the Q / dO empty barriers.  break_release: thread 0 refills a stage once its own warpgroup has
    released it, without waiting for the other one (must be caught)."""
    NST = DKDV_STAGES
    rnd = random.Random(seed)
    B = {"kv": Bar(1)}
    for i in range(NST):
        B[f"qf{i}"] = Bar(1)
        B[f"qe{i}"] = Bar(2)

    def W(w):
        if w == 0:
            yield ("async", "kv")
            for j in range(min(T, NST)):
                yield ("tma", f"qf{j % NST}", f"q{j % NST}")
        yield ("wait", "kv", 0)
        for j in range(T):
            st = j % NST
            yield ("wait", f"qf{st}", j // NST)
            yield ("read", f"q{st}", 1)              # S^T, dP^T, dV, dK MMAs, waited for
            yield ("read", f"q{st}", -1)
            yield ("arrive", f"qe{st}")
            if w == 0 and j + NST < T:
                if not break_release:
                    yield ("wait", f"qe{st}", j // NST)
                yield ("tma", f"qf{st}", f"q{st}")

    return _simulate({"W0": W(0), "W1": W(1)}, B, rnd)


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
