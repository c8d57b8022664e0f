"""Non-causal (causal=False) attention on the wgmma kernels against the causal wgmma kernels and the generic kernels.

    python scripts/attn_bidir_bench.py [--rounds 3] [--window 0.3] [--cells 0,1] [--out FILE]

Cells (d, H, B, Lmax, dtype): B sequences of lengths U[0.9, 1) * Lmax (seed 1001), no targets or window; q, k ~ N(0, 1),
v, dout ~ N(0, 1), alpha = 1/sqrt(d).  Arms, on the same inputs, each timed for the forward and for the backward:
"bidir" (hstu_attn_fwd_bidir / _bwd_bidir on the attn_*_bidir_wgmma_kernel kernels), "causal" (hstu_attn_fwd / _bwd on
the causal wgmma kernels; the backward forced onto its deterministic split kernels where the fused one is the default,
so that both arms run the same kernel pair) and "generic_bidir" (the non-causal generic kernels, IMPL_GENERIC).  Times
are CUDA events over back-to-back calls filling `--window` seconds after a warm-up call, medians over rounds with the
arms alternated in every round; a call includes the pre-pass kernels of bf16 at d = 32 (DESIGN.md 3.0).

Score counts are computed here from the lengths: every (query, key) pair of a sequence for the non-causal mask, the
lower triangle with its diagonal for the causal one.  The tensor FLOPs are algorithmic: 4 d per score forward (S = Q K^T,
O += P V) and 10 d backward (S, dP, dV, dK, dQ), over the dense 989 TFLOP/s of the H100 SXM data sheet (bf16 / fp16).
`bidir_over_causal` is the measured time ratio; `score_ratio` is the ratio the score counts predict.  Prints one JSON line
(also written to --out) with the card's name and power limit, read in the same run.
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

from attn_delta_bench import time_ms  # noqa: E402
from attn_fp8_bench import Sampler, card  # noqa: E402

TENSOR_FLOPS = 989e12
BF, FP = torch.bfloat16, torch.float16
CELLS = [(32, 8, 64, 1024, BF), (32, 8, 64, 1024, FP), (32, 8, 32, 2048, BF), (32, 4, 16, 8192, BF), (32, 4, 16, 8192, FP),
         (64, 4, 32, 2048, BF), (64, 2, 16, 8192, FP), (128, 4, 32, 1024, BF), (128, 2, 16, 8192, BF)]


def cell(d, H, B, lmax, dtype, args, dev):
    from generative_recommenders_b200 import _lib
    from generative_recommenders_b200.ops.hstu_attention import cuda_hstu_attention_bwd, cuda_hstu_attention_fwd

    g = torch.Generator(device=dev).manual_seed(1001)
    lengths = (lmax * (0.9 + 0.1 * torch.rand(B, generator=g, device=dev))).long().clamp_max(lmax)
    off = torch.zeros(B + 1, dtype=torch.int64, device=dev)
    off[1:] = torch.cumsum(lengths, 0)
    L = int(off[-1])
    q, k, v, do = (torch.randn(L, H, d, device=dev, generator=g).to(dtype) for _ in range(4))
    grads = [torch.empty_like(q) for _ in range(3)]
    alpha = 1.0 / math.sqrt(d)
    outs = {}

    def fwd(name, causal, impl):
        return lambda: outs.__setitem__(name, cuda_hstu_attention_fwd(lmax, alpha, q, k, v, off, impl=impl, causal=causal))

    def bwd(causal, impl):
        return lambda: cuda_hstu_attention_bwd(lmax, alpha, do, q, k, v, *grads, off, impl=impl, causal=causal,
                                               deterministic=True)

    arms = {
        ("bidir", "fwd"): fwd("bidir", False, _lib.IMPL_UMMA), ("bidir", "bwd"): bwd(False, _lib.IMPL_UMMA),
        ("causal", "fwd"): fwd("causal", True, _lib.IMPL_UMMA), ("causal", "bwd"): bwd(True, _lib.IMPL_UMMA),
        ("generic_bidir", "fwd"): fwd("generic_bidir", False, _lib.IMPL_GENERIC),
        ("generic_bidir", "bwd"): bwd(False, _lib.IMPL_GENERIC),
    }
    iters = {}
    for key, fn in arms.items():
        fn()  # warm-up (module load, function attributes)
        torch.cuda.synchronize()
        iters[key] = max(2, math.ceil(args.window * 1e3 / time_ms(fn, 1)))
    sampler = Sampler()
    times = {key: [] for key in arms}
    clock = []
    for _ in range(args.rounds):
        for key, fn in arms.items():
            with sampler:
                times[key].append(time_ms(fn, iters[key]))
            clock.append(sampler.medians()[0])
    ms = {f"{a}_{p}": statistics.median(t) for (a, p), t in times.items()}
    lens = lengths.double()
    scores = {"bidir": float((lens * lens).sum()) * H, "causal": float((lens * (lens + 1) / 2).sum()) * H}
    flops = {"fwd": 4 * d, "bwd": 10 * d}
    share = {}
    for a, sc in (("bidir", scores["bidir"]), ("causal", scores["causal"]), ("generic_bidir", scores["bidir"])):
        for p in ("fwd", "bwd"):
            share[f"{a}_{p}"] = sc * flops[p] / (ms[f"{a}_{p}"] * 1e-3) / TENSOR_FLOPS
    ref = outs["generic_bidir"].float()
    row = {
        "d": d, "heads": H, "batch": B, "lmax": lmax, "dtype": str(dtype).split(".")[-1], "rows": L,
        "calls_per_window": {f"{a}_{p}": n for (a, p), n in iters.items()},
        "ms_per_call": ms, "ms_all": {f"{a}_{p}": t for (a, p), t in times.items()},
        "scores": scores, "score_ratio": scores["bidir"] / scores["causal"],
        "bidir_over_causal": {p: ms[f"bidir_{p}"] / ms[f"causal_{p}"] for p in ("fwd", "bwd")},
        "speedup_over_generic": {p: ms[f"generic_bidir_{p}"] / ms[f"bidir_{p}"] for p in ("fwd", "bwd")},
        "tensor_share_of_989TFLOPs": share,
        "sm_clock_mhz_median": statistics.median(clock) if None not in clock else None,
        "rel_l2_bidir_vs_generic_out": float((outs["bidir"].float() - ref).norm() / ref.norm().clamp_min(1e-30)),
    }
    del q, k, v, do, grads, outs
    torch.cuda.empty_cache()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--window", type=float, default=0.3, help="seconds of back-to-back calls per timed window")
    ap.add_argument("--cells", default=None, help="comma-separated cell indices (default: all)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from bench import ensure_built

    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    ensure_built()
    dev = torch.device("cuda", 0)
    res = {"rounds": args.rounds, "window_s": args.window, "card": card(), "cells": []}
    pick = range(len(CELLS)) if args.cells is None else [int(i) for i in args.cells.split(",")]
    for i in pick:
        row = cell(*CELLS[i], args, dev)
        res["cells"].append(row)
        print(json.dumps({kk: row[kk] for kk in ("d", "heads", "batch", "lmax", "dtype", "ms_per_call", "score_ratio",
                                                 "bidir_over_causal", "speedup_over_generic", "tensor_share_of_989TFLOPs",
                                                 "rel_l2_bidir_vs_generic_out")}), file=sys.stderr, flush=True)
    res["card_after"] = card()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
