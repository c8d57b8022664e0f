"""Delta-q (KV-cached) attention forward: the wgmma kernel against the generic kernel and the reference's Triton kernel.

    python scripts/attn_delta_bench.py [--rounds 3] [--window 0.3] [--out FILE]

Inputs: B sequences with cache lengths U[0.9, 1) * 8192 (seed 1001), whose last `delta` rows are the queries; q, k, v ~ N(0, 1)
in bf16, alpha = 1/sqrt(d), num_targets = delta.  Cells (d, H, B, delta): d = 32, H = 8 at B in {1, 16, 128} and delta in
{1, 16, 64, 256}; d = 64 and d = 128 at H = 4, B = 16, delta in {16, 256}; d = 256 at H = 4, B = 16, delta = 16.

Arms: "wgmma" (cuda_hstu_attention_fwd, which routes delta calls to attn_fwd_delta_wgmma_kernel), "generic" (impl=IMPL_GENERIC,
the CUDA-core kernel) and "triton" (the reference's triton_cached_hstu_mha from oracle/_ref, unmodified, when build() has
fetched it; reported as unavailable otherwise).  Every arm is warmed up (Triton autotunes there).  In every round the arms run
one after another with CUDA events, each over enough back-to-back calls to fill `--window` seconds; medians over rounds are
reported, with the median SM clock and power draw read through NVML during each window.  Kernel times come from
`torch.profiler` over whole sustained windows in a separate pass, alternated the same way.

Bytes are algorithmic: the K and V rows the delta rows attend (every row of the sequence: causal, no window), plus q and out,
plus for the wgmma arm the fp32 partials of split key chunks (written once, read once).  The share of bandwidth is those bytes
over the kernel time, against the 3.35 TB/s of the H100 SXM data sheet.  Finally, one line times STULayer.cached_forward at
the headline dims (D = 256, H = 8, d = 32, B = 16, delta = 16) and the share of it spent in the attention kernels.

Prints one JSON line (also written to --out) with the card's name and power limit, read in the same run.
"""
import argparse
import ctypes as C
import json
import math
import os
import statistics
import sys

import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from attn_fp8_bench import Sampler, card  # noqa: E402

CELLS = ([(32, 8, b, dl) for b in (1, 16, 128) for dl in (1, 16, 64, 256)] +
         [(d, 4, 16, dl) for d in (64, 128) for dl in (16, 256)] + [(256, 4, 16, 16)])
LMAX = 8192
HBM_BYTES_PER_S = 3.35e12


def triton_fn():
    ref_root = os.path.join(ROOT, "oracle", "_ref")
    if not os.path.isdir(os.path.join(ref_root, "generative_recommenders")):
        return None, "oracle/_ref is absent (oracle/fetch_reference_eager.py)"
    sys.path.insert(0, ref_root)
    try:
        import triton.language as tl

        for name in ("_experimental_descriptor_load", "_experimental_descriptor_store"):  # see bench.py run_triton
            if not hasattr(tl, name):
                setattr(tl, name, None)
        from generative_recommenders.ops.triton.triton_hstu_attention import triton_cached_hstu_mha
    except Exception as e:  # noqa: BLE001
        return None, f"import failed: {type(e).__name__}: {e}"[:300]
    return triton_cached_hstu_mha, None


def workspace_bytes(N, alpha, dq, k, v, off, nt, delta):
    """What the library asks for this call: the fp32 partials of its key chunks (0 with one chunk)."""
    from generative_recommenders_b200 import _lib
    from generative_recommenders_b200.ops.hstu_attention import _fill_common

    p = _lib.AttnParams()
    _fill_common(p, N, alpha, dq, k, v, off, nt, 0, 0, 0, _lib.IMPL_AUTO, delta)
    p.out, p.o_row_stride, p.o_head_stride = dq.data_ptr(), dq.stride(0), dq.stride(1)
    return int(_lib.lib().hstu_attn_workspace_bytes(C.byref(p), 0))


def time_ms(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def profile_kernels(fn, n, sampler):
    """(wall ms per call, kernel ms per call by kernel name, median SM clock) of one profiled sustained window."""
    from torch.profiler import ProfilerActivity, profile

    with sampler, profile(activities=[ProfilerActivity.CUDA]) as prof:
        wall = time_ms(fn, n)
    kern = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = getattr(ev, "cuda_time_total", 0.0)
        if t > 0 and "memcpy" not in ev.key.lower() and "memset" not in ev.key.lower():
            kern[ev.key[:120]] = kern.get(ev.key[:120], 0.0) + t / 1e3 / n
    return wall, kern, sampler.medians()[0]


def cell(d, H, B, delta, args, tri, dev):
    from generative_recommenders_b200 import _lib
    from generative_recommenders_b200.ops.hstu_attention import cuda_hstu_attention_fwd

    g = torch.Generator(device=dev).manual_seed(1001)
    lengths = (LMAX * (0.9 + 0.1 * torch.rand(B, generator=g, device=dev))).long().clamp_max(LMAX)
    off = torch.zeros(B + 1, dtype=torch.int64, device=dev)
    off[1:] = torch.cumsum(lengths, 0)
    L = int(off[-1])
    k, v = (torch.randn(L, H, d, device=dev, generator=g).to(torch.bfloat16) for _ in range(2))
    dq = torch.randn(B * delta, H, d, device=dev, generator=g).to(torch.bfloat16)
    nt = torch.full((B,), delta, dtype=torch.int64, device=dev)
    alpha = 1.0 / math.sqrt(d)
    N = LMAX
    outs = {}
    arms = {
        "wgmma": lambda: outs.__setitem__("wgmma", cuda_hstu_attention_fwd(N, alpha, dq, k, v, off, nt, delta_q_len=delta)),
        "generic": lambda: outs.__setitem__("generic", cuda_hstu_attention_fwd(N, alpha, dq, k, v, off, nt, delta_q_len=delta,
                                                                               impl=_lib.IMPL_GENERIC)),
    }
    if tri is not None:
        arms["triton"] = lambda: outs.__setitem__("triton", tri(N, alpha, dq, k, v, off, nt, 0, 0))
    iters, failed = {}, {}
    for name in list(arms):
        try:
            arms[name]()  # warm-up (Triton: autotuning)
            torch.cuda.synchronize()
            iters[name] = max(3, math.ceil(args.window * 1e3 / time_ms(arms[name], 3)))
        except Exception as e:  # noqa: BLE001  (the comparator only; our own arms must run)
            if name != "triton":
                raise
            failed[name] = f"{type(e).__name__}: {e}"[:300]
            del arms[name]
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
    ws = workspace_bytes(N, alpha, dq, k, v, off, nt, delta)
    kv_bytes = 2 * L * H * d * 2
    qo_bytes = 2 * B * delta * H * d * 2
    ms = {n: statistics.median(t) for n, t in times.items()}
    kernel_ms = {n: statistics.median(sum(r[1].values()) for r in rows) for n, rows in prof.items()}
    kernels = {n: {kk: statistics.median(r[1].get(kk, 0.0) for r in rows) for kk in rows[0][1]} for n, rows in prof.items()}
    byts = {n: kv_bytes + qo_bytes + (2 * ws if n == "wgmma" else 0) for n in arms}
    ref = outs["generic"].float()
    row = {
        "d": d, "heads": H, "batch": B, "delta": delta, "cached_rows": L, "calls_per_window": iters,
        "ms_per_call": ms, "ms_all": times, "kernel_ms_per_call": kernel_ms, "kernels_ms_per_call": kernels,
        "wgmma_speedup_vs_generic": ms["generic"] / ms["wgmma"],
        "wgmma_speedup_vs_triton": (ms["triton"] / ms["wgmma"]) if "triton" in ms else None,
        "workspace_bytes": ws, "algorithmic_bytes": byts,
        "hbm_share_of_3.35TBps": {n: byts[n] / (kernel_ms[n] * 1e-3) / HBM_BYTES_PER_S for n in arms},
        "sm_clock_mhz_median": {n: statistics.median(c) if None not in c else None for n, c in clock.items()},
        "power_w_median": {n: statistics.median(w) if None not in w else None for n, w in power.items()},
        "rel_l2_vs_generic": {n: float((o.float() - ref).norm() / ref.norm().clamp_min(1e-30)) for n, o in outs.items()},
        "unavailable": failed,
    }
    del k, v, dq, outs
    torch.cuda.empty_cache()
    return row


def layer_line(args, dev):
    """Per-layer STULayer.cached_forward at the headline dims, and the share of its device time in attention kernels."""
    from generative_recommenders_b200.modules.stu import STULayer, STULayerConfig, STUStack

    D, H, d, B, delta = 256, 8, 32, 16, 16
    torch.manual_seed(7)
    layer = STULayer(STULayerConfig(embedding_dim=D, num_heads=H, hidden_dim=d, attention_dim=d, output_dropout_ratio=0.0,
                                    target_aware=True))
    stack = STUStack([layer]).to(dev).to(torch.bfloat16).eval()
    g = torch.Generator(device=dev).manual_seed(1001)
    cache = (LMAX * (0.9 + 0.1 * torch.rand(B, generator=g, device=dev))).long().clamp_max(LMAX)
    full = cache + delta
    off = torch.zeros(B + 1, dtype=torch.int64, device=dev)
    off[1:] = torch.cumsum(full, 0)
    nt = torch.full((B,), delta, device=dev)
    x = torch.randn(int(off[-1]), D, device=dev).to(torch.bfloat16)
    rows = torch.cat([torch.arange(int(off[i + 1]) - delta, int(off[i + 1]), device=dev) for i in range(B)])
    with torch.no_grad():
        stack(x=x, x_lengths=full, x_offsets=off, max_seq_len=LMAX + delta, num_targets=nt, max_kv_caching_len=LMAX,
              kv_caching_lengths=cache)
        xd = x[rows].contiguous()
        fn = lambda: layer.cached_forward(delta_x=xd, num_targets=nt)  # noqa: E731
        fn()
        n = max(3, math.ceil(args.window * 1e3 / time_ms(fn, 3)))
        wall = statistics.median(time_ms(fn, n) for _ in range(args.rounds))
        _, kern, _ = profile_kernels(fn, n, Sampler())
    attn = sum(t for kk, t in kern.items() if "attn_fwd" in kk or "delta_reduce" in kk)
    return {"D": D, "heads": H, "d": d, "batch": B, "delta": delta, "ms_per_layer_call": wall,
            "kernel_ms_per_call": sum(kern.values()), "attention_kernel_ms_per_call": attn,
            "attention_share_of_layer_kernel_time": attn / max(sum(kern.values()), 1e-12),
            "attention_share_of_layer_wall_time": attn / wall, "kernels_ms_per_call": kern}


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
    tri, why = triton_fn()
    res = {"rounds": args.rounds, "window_s": args.window, "triton": why or "available", "cells": []}
    pick = range(len(CELLS)) if args.cells is None else [int(i) for i in args.cells.split(",")]
    for i in pick:
        row = cell(*CELLS[i], args, tri, dev)
        res["cells"].append(row)
        print(json.dumps({kk: row[kk] for kk in ("d", "heads", "batch", "delta", "ms_per_call", "kernel_ms_per_call",
                                                 "wgmma_speedup_vs_generic", "wgmma_speedup_vs_triton", "hbm_share_of_3.35TBps",
                                                 "workspace_bytes", "sm_clock_mhz_median", "rel_l2_vs_generic")}),
              file=sys.stderr, flush=True)
    res["cached_forward_layer"] = layer_line(args, dev)
    print(json.dumps(res["cached_forward_layer"]), file=sys.stderr, flush=True)
    res["card"] = card()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
