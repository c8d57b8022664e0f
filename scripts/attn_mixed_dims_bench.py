"""Attention with a value head wider than the query / key head (dqk < dv): the wgmma kernels against the generic CUDA-core
kernels, timed on the same inputs in one process.

    python scripts/attn_mixed_dims_bench.py [--rounds 5] [--window 0.5] [--out FILE]

Inputs: `synth_lengths` of bench.py (lengths U[0.9, 1) Lmax with 1-20 targets, seed 1001); q, k, v as strided views of one
[L, H, 2 dqk + dv] U(-0.01, 0.01) buffer split [dqk, dqk, dv] (the reference benchmark's split), dO ~ N(0, 1); alpha = 1/dqk,
H = 4, bf16 and fp16 (the fp16 inputs are the bf16 values converted).  Cells:
  forward and backward at (128, 256), Lmax 512 / 2048 / 8192 (the batches of attn_bwd_d256_bench.py);
  forward and backward at the other five pairs, Lmax 2048;
  delta-q forward at (128, 256), Lmax 8192, B in {16, 128}, delta in {16, 64}.
In every round the two implementations (AUTO: the wgmma kernels; IMPL_GENERIC: what AUTO ran before) are timed one after the
other with CUDA events, each over enough back-to-back calls to fill `--window` seconds; medians over rounds are reported, with
the achieved TFLOP/s of the wgmma path under bench.py's FLOP model (attn_flops) against the 989 TFLOP/s dense bf16 / fp16
data-sheet rate of the H100 SXM, and the rel-L2 distance between the two results.  Delta-q cells also report the bytes of
K and V read per call over the time (the bound that binds there).

Prints one JSON line (also written to --out) with the card's name, power limit and SM clock, read in the same run.
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)

HEADS = 4
PEAK_TFLOPS = 989.0  # H100 SXM data sheet, dense bf16 / fp16
PEAK_TBPS = 3.35  # H100 SXM data sheet, HBM3
MAIN = (128, 256)
CELLS = [(MAIN, 512, 512), (MAIN, 2048, 128), (MAIN, 8192, 16)] + [
    (pair, 2048, 128) for pair in [(32, 64), (32, 128), (32, 256), (64, 128), (64, 256)]]
DELTA = [(16, 16), (16, 64), (128, 16), (128, 64)]  # (B, delta) at Lmax 8192


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), (s.strip() for s in out.split(","))))
    except Exception as e:  # the timing itself does not depend on nvidia-smi
        return {"name": torch.cuda.get_device_name(0), "error": str(e)}


def rel_l2(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


def time_ms(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def compare(calls, rounds, window):
    """calls: {name: fn}; warm-up, calls per window, then `rounds` alternating windows.  Returns (iters, medians, all)."""
    iters = {}
    for name, fn in calls.items():
        fn()
        iters[name] = max(1, math.ceil(window * 1e3 / time_ms(fn, 1)))
    times = {name: [] for name in calls}
    for _ in range(rounds):
        for name, fn in calls.items():
            times[name].append(time_ms(fn, iters[name]))
    return iters, {n: statistics.median(t) for n, t in times.items()}, times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--window", type=float, default=0.5, help="seconds of back-to-back calls per timed window")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from bench import attn_flops, ensure_built, synth_lengths
    from generative_recommenders_b200 import _lib
    from generative_recommenders_b200.ops.hstu_attention import (cuda_hstu_attention_bwd, cuda_hstu_attention_fwd,
                                                                 delta_hstu_mha)

    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    ensure_built()
    dev = torch.device("cuda", 0)
    impls = {"wgmma": _lib.IMPL_AUTO, "generic": _lib.IMPL_GENERIC}
    res = {"heads": HEADS, "rounds": args.rounds, "window_s": args.window, "peak_tflops": PEAK_TFLOPS, "cells": [],
           "delta": []}

    def rate(flops, ms):
        return flops / (ms * 1e-3) / 1e12

    for (dqk, dv), lmax, batch in CELLS:
        lengths, nt, off = synth_lengths(batch, lmax, dev, 1001)
        L = int(off[-1])
        fl = attn_flops(lengths, HEADS, dqk, dv)
        g = torch.Generator(device=dev).manual_seed(7)
        x16 = torch.empty(L, HEADS, 2 * dqk + dv, device=dev).uniform_(-0.01, 0.01, generator=g).to(torch.bfloat16)
        do16 = torch.randn(L, HEADS, dv, device=dev, generator=g).to(torch.bfloat16)
        for dt in (torch.bfloat16, torch.float16):
            x, do = x16.to(dt), do16.to(dt)
            q, k, v = torch.split(x, [dqk, dqk, dv], dim=-1)
            outs = {n: torch.empty(L, HEADS, dv, device=dev, dtype=dt) for n in impls}
            grads = {n: (torch.empty(L, HEADS, dqk, device=dev, dtype=dt), torch.empty(L, HEADS, dqk, device=dev, dtype=dt),
                         torch.empty(L, HEADS, dv, device=dev, dtype=dt)) for n in impls}

            def fwd(n):
                return lambda: cuda_hstu_attention_fwd(lmax, 1.0 / dqk, q, k, v, off, num_targets=nt, impl=impls[n], out=outs[n])

            def bwd(n):
                return lambda: cuda_hstu_attention_bwd(lmax, 1.0 / dqk, do, q, k, v, *grads[n], off, num_targets=nt,
                                                       impl=impls[n], deterministic=False)

            row = {"dqk": dqk, "dv": dv, "lmax": lmax, "sequences": batch, "rows": L, "dtype": str(dt).replace("torch.", "")}
            for phase, mk, flops in (("fwd", fwd, fl["fwd"]), ("bwd", bwd, fl["bwd"])):
                iters, med, times = compare({n: mk(n) for n in impls}, args.rounds, args.window)
                torch.cuda.synchronize()
                if phase == "fwd":
                    err = {"out": rel_l2(outs["wgmma"], outs["generic"])}
                else:
                    err = {n: rel_l2(a, b) for n, a, b in zip(("dq", "dk", "dv"), grads["wgmma"], grads["generic"])}
                row[phase] = {"calls_per_window": iters, "ms_median": med, "ms_all": times,
                              "speedup_vs_generic": med["generic"] / med["wgmma"], "flops_per_call": flops,
                              "wgmma_tflops": rate(flops, med["wgmma"]),
                              "wgmma_frac_of_peak": rate(flops, med["wgmma"]) / PEAK_TFLOPS, "bound": "tensor-core FLOP/s",
                              "rel_l2_wgmma_vs_generic": err}
            res["cells"].append(row)
            print(json.dumps({"pair": [dqk, dv], "lmax": lmax, "dtype": row["dtype"],
                              **{ph: [row[ph]["ms_median"], row[ph]["speedup_vs_generic"]] for ph in ("fwd", "bwd")}}),
                  file=sys.stderr, flush=True)
            del outs, grads
        del x16, do16
        torch.cuda.empty_cache()

    dqk, dv = MAIN
    for B, delta in DELTA:
        lmax = 8192
        lengths, nt, off = synth_lengths(B, lmax, dev, 1001)
        L = int(off[-1])
        g = torch.Generator(device=dev).manual_seed(9)
        kv16 = torch.empty(L, HEADS, dqk + dv, device=dev).uniform_(-0.01, 0.01, generator=g).to(torch.bfloat16)
        q16 = torch.empty(B * delta, HEADS, dqk, device=dev).uniform_(-0.01, 0.01, generator=g).to(torch.bfloat16)
        ntd = torch.full((B,), delta, device=dev, dtype=torch.int64)
        # S and P V over each query row's keys (causal: the delta rows see about the whole sequence)
        flops = 2.0 * HEADS * delta * float(lengths.sum()) * (dqk + dv)
        kv_bytes = 2.0 * L * HEADS * (dqk + dv)
        for dt in (torch.bfloat16, torch.float16):
            kv, dq_ = kv16.to(dt), q16.to(dt)
            k, v = torch.split(kv, [dqk, dv], dim=-1)
            outs = {}

            def dcall(n):
                if n == "wgmma":
                    return lambda: outs.__setitem__(n, delta_hstu_mha(lmax, 1.0 / dqk, dq_, k, v, off, num_targets=ntd))
                return lambda: outs.__setitem__(n, cuda_hstu_attention_fwd(lmax, 1.0 / dqk, dq_, k, v, off, num_targets=ntd,
                                                                           impl=_lib.IMPL_GENERIC, delta_q_len=delta))

            iters, med, times = compare({n: dcall(n) for n in impls}, args.rounds, args.window)
            torch.cuda.synchronize()
            row = {"dqk": dqk, "dv": dv, "lmax": lmax, "sequences": B, "delta": delta, "dtype": str(dt).replace("torch.", ""),
                   "calls_per_window": iters, "ms_median": med, "ms_all": times,
                   "speedup_vs_generic": med["generic"] / med["wgmma"], "flops_per_call": flops,
                   "wgmma_tflops": rate(flops, med["wgmma"]), "wgmma_frac_of_peak": rate(flops, med["wgmma"]) / PEAK_TFLOPS,
                   "kv_bytes_per_call": kv_bytes, "wgmma_tbps": kv_bytes / (med["wgmma"] * 1e-3) / 1e12,
                   "wgmma_frac_of_hbm": kv_bytes / (med["wgmma"] * 1e-3) / 1e12 / PEAK_TBPS, "bound": "HBM bandwidth (K, V)",
                   "rel_l2_wgmma_vs_generic": rel_l2(outs["wgmma"], outs["generic"])}
            res["delta"].append(row)
            print(json.dumps({"delta": [B, delta], "dtype": row["dtype"], "ms": med, "x": row["speedup_vs_generic"]}),
                  file=sys.stderr, flush=True)
        del kv16, q16
        torch.cuda.empty_cache()
    res["card"] = card()  # read right after the timing, so the SM clock is the loaded one
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
