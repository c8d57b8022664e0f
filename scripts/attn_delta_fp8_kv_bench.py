"""Delta-q (KV-cached) attention forward over an fp8 (e4m3) K / V cache against the same attention over the bf16 cache.

    python scripts/attn_delta_fp8_kv_bench.py [--rounds 3] [--window 0.3] [--out FILE]

Cells (d, H, B, delta): those of scripts/attn_delta_bench.py (profiles/h100_attn_delta.json).  Inputs: B sequences with
cache lengths U[0.9, 1) * 8192 (seed 1001), whose last `delta` rows are the queries; q ~ N(0, 1) in bf16, k, v ~ N(0, 1)
quantised to e4m3 with per (sequence, head) descales amax / 448, alpha = 1/sqrt(d), num_targets = delta.

Arms, on the same values: "fp8_kv" (the e4m3 cache and its descales, attn_fwd_delta_e4m3kv_wgmma_kernel) and "bf16" (the
dequantised cache codes * descale, rounded to bf16, attn_fwd_delta_wgmma_kernel); rel_l2_fp8_kv_vs_bf16 includes that
rounding.  In every round the two arms run one
after the other with CUDA events, each over enough back-to-back calls to fill `--window` seconds; medians over rounds are
reported.  Kernel times come from `torch.profiler` over whole windows in a separate pass, alternated the same way.

Bytes are algorithmic: the K and V rows the delta rows attend (1 byte per element for fp8_kv, 2 for bf16), q and out, and
the fp32 partials of split key chunks (written once, read once).  The HBM share is those bytes over the kernel time, against
the 3.35 TB/s of the H100 SXM data sheet.  Prints one JSON line (also written to --out) with the card's name and power
limit, read in the same run.
"""
import argparse
import json
import math
import os
import statistics
import sys

import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from attn_delta_bench import CELLS, HBM_BYTES_PER_S, LMAX, profile_kernels, time_ms, workspace_bytes  # noqa: E402
from attn_fp8_bench import Sampler, card  # noqa: E402


def cell(d, H, B, delta, args, dev):
    from generative_recommenders_b200.ops.hstu_attention import cuda_hstu_attention_fwd

    g = torch.Generator(device=dev).manual_seed(1001)
    lengths = (LMAX * (0.9 + 0.1 * torch.rand(B, generator=g, device=dev))).long().clamp_max(LMAX)
    off = torch.zeros(B + 1, dtype=torch.int64, device=dev)
    off[1:] = torch.cumsum(lengths, 0)
    L = int(off[-1])
    rb = torch.repeat_interleave(torch.arange(B, device=dev), lengths)
    cache = {}
    for name in ("k", "v"):
        x = torch.randn(L, H, d, device=dev, generator=g)
        amax = torch.zeros(B, H, device=dev).index_reduce_(0, rb, x.abs().amax(-1), "amax")
        ds = torch.where(amax > 0, amax / 448.0, torch.ones_like(amax))
        codes = (x / ds[rb][:, :, None]).to(torch.float8_e4m3fn)
        cache[name] = (codes, ds, (codes.float() * ds[rb][:, :, None]).to(torch.bfloat16))
        del x
    dq = torch.randn(B * delta, H, d, device=dev, generator=g).to(torch.bfloat16)
    nt = torch.full((B,), delta, dtype=torch.int64, device=dev)
    alpha = 1.0 / math.sqrt(d)
    N = LMAX
    (k8, kd, k16), (v8, vd, v16) = cache["k"], cache["v"]
    outs = {}
    arms = {
        "fp8_kv": lambda: outs.__setitem__("fp8_kv", cuda_hstu_attention_fwd(N, alpha, dq, k8, v8, off, nt, delta_q_len=delta,
                                                                             descales=(None, kd, vd))),
        "bf16": lambda: outs.__setitem__("bf16", cuda_hstu_attention_fwd(N, alpha, dq, k16, v16, off, nt, delta_q_len=delta)),
    }
    iters = {}
    for name, fn in arms.items():
        fn()
        torch.cuda.synchronize()
        iters[name] = max(3, math.ceil(args.window * 1e3 / time_ms(fn, 3)))
    sampler = Sampler()
    times, clock, power = ({n: [] for n in arms} for _ in range(3))
    for _ in range(args.rounds):
        for name, fn in arms.items():
            with sampler:
                times[name].append(time_ms(fn, iters[name]))
            c, w = sampler.medians()
            clock[name].append(c)
            power[name].append(w)
    prof = {n: [] for n in arms}
    for _ in range(args.profile_rounds):
        for name, fn in arms.items():
            prof[name].append(profile_kernels(fn, iters[name], sampler))
    ws = workspace_bytes(N, alpha, dq, k16, v16, off, nt, delta)  # the same chunk rule for both arms
    qo_bytes = 2 * B * delta * H * d * 2
    byts = {"fp8_kv": 2 * L * H * d + qo_bytes + 2 * ws, "bf16": 2 * L * H * d * 2 + qo_bytes + 2 * ws}
    ms = {n: statistics.median(t) for n, t in times.items()}
    kernel_ms = {n: statistics.median(sum(r[1].values()) for r in rows) for n, rows in prof.items()}
    kernels = {n: {kk: statistics.median(r[1].get(kk, 0.0) for r in rows) for kk in rows[0][1]} for n, rows in prof.items()}
    ref = outs["bf16"].float()
    row = {
        "d": d, "heads": H, "batch": B, "delta": delta, "cached_rows": L, "calls_per_window": iters,
        "ms_per_call": ms, "ms_all": times, "kernel_ms_per_call": kernel_ms, "kernels_ms_per_call": kernels,
        "fp8_kv_speedup_vs_bf16_kernel_time": kernel_ms["bf16"] / kernel_ms["fp8_kv"],
        "fp8_kv_speedup_vs_bf16_call_time": ms["bf16"] / ms["fp8_kv"],
        "workspace_bytes": ws, "algorithmic_bytes": byts,
        "hbm_share_of_3.35TBps": {n: byts[n] / (kernel_ms[n] * 1e-3) / HBM_BYTES_PER_S for n in arms},
        "sm_clock_mhz_median": {n: statistics.median(c) if None not in c else None for n, c in clock.items()},
        "power_w_median": {n: statistics.median(w) if None not in w else None for n, w in power.items()},
        "rel_l2_fp8_kv_vs_bf16": float((outs["fp8_kv"].float() - ref).norm() / ref.norm().clamp_min(1e-30)),
    }
    del cache, dq, outs, k8, v8, k16, v16
    torch.cuda.empty_cache()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--window", type=float, default=0.3, help="seconds of back-to-back calls per timed window")
    ap.add_argument("--profile-rounds", type=int, default=2)
    ap.add_argument("--cells", default=None, help="comma-separated cell indices (default: all)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from bench import ensure_built

    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    ensure_built()
    dev = torch.device("cuda", 0)
    res = {"rounds": args.rounds, "window_s": args.window, "cells": []}
    pick = range(len(CELLS)) if args.cells is None else [int(i) for i in args.cells.split(",")]
    for i in pick:
        row = cell(*CELLS[i], args, dev)
        res["cells"].append(row)
        print(json.dumps({kk: row[kk] for kk in ("d", "heads", "batch", "delta", "ms_per_call", "kernel_ms_per_call",
                                                 "fp8_kv_speedup_vs_bf16_kernel_time", "hbm_share_of_3.35TBps",
                                                 "workspace_bytes", "sm_clock_mhz_median", "rel_l2_fp8_kv_vs_bf16")}),
              file=sys.stderr, flush=True)
    res["card"] = card()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
