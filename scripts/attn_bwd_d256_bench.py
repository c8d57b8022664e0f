"""Attention backward at head dim 256: the split wgmma kernels against the generic CUDA-core kernels, timed on the same
inputs in one process.

    python scripts/attn_bwd_d256_bench.py [--rounds 5] [--window 0.5] [--out FILE]

Inputs: the `bench.py --workload attn` recipe (`synth_lengths`: lengths U[0.9, 1) Lmax with 1-20 targets, seed 1001;
`attn_inputs`: q, k, v as strided views of one [L, H, 3d] buffer, dO ~ N(0, 1)), alpha = 1/d, H = 4, d = 256, bf16 and fp16
(the fp16 inputs are the bf16 values converted).  Shapes: Lmax 512, 2048 and 8192.

Each (shape, dtype) is warmed up first.  Then, in every round, the two implementations of `cuda_hstu_attention_bwd` are
timed one after another with CUDA events, each over enough back-to-back calls to fill `--window` seconds (at least one):
  wgmma    AUTO, deterministic=False: attn_bwd_dkdv_wgmma_kernel + attn_bwd_dq_wgmma_kernel;
  generic  IMPL_GENERIC: the CUDA-core kernels, what AUTO ran at d = 256 before.
The medians over rounds are reported, with the achieved TFLOP/s of the wgmma path under bench.py's FLOP model (causal-halved
3 + 2 GEMMs) against the 989 TFLOP/s dense bf16 / fp16 data-sheet rate of the H100 SXM, and the rel-L2 distance between the
two results.  The reference's Triton kernel is timed (forward + backward, by bench.py --impl triton) only when oracle/_ref
is present.

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

D = 256
HEADS = 4
SHAPES = [(512, 512), (2048, 128), (8192, 16)]  # (Lmax, sequences)
PEAK_TFLOPS = 989.0  # H100 SXM data sheet, dense bf16 / fp16


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


def triton_row(lmax, batch):
    """bench.py's Triton arm (fwd + bwd of the reference kernel) at this shape, or why it was not run."""
    if not os.path.isdir(os.path.join(ROOT, "oracle", "_ref", "generative_recommenders")):
        return {"unavailable": "oracle/_ref is absent"}
    cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--impl", "triton", "--workload", "attn",
           "--attn-dim", str(D), "--attn-heads", str(HEADS), "--lmax", str(lmax), "--batch", str(batch), "--steps", "5",
           "--warmup", "2"]
    r = subprocess.run(cmd, capture_output=True, text=True, cwd=ROOT)
    lines = [x for x in r.stdout.splitlines() if x.startswith("{")]
    return json.loads(lines[-1]) if lines else {"unavailable": f"exit {r.returncode}: {r.stderr[-300:]}"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--window", type=float, default=0.5, help="seconds of back-to-back calls per timed window")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from bench import attn_flops, attn_inputs, ensure_built, synth_lengths
    from generative_recommenders_b200 import _lib
    from generative_recommenders_b200.ops.hstu_attention import cuda_hstu_attention_bwd

    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    ensure_built()
    dev = torch.device("cuda", 0)
    impls = {"wgmma": dict(), "generic": dict(impl=_lib.IMPL_GENERIC)}

    def time_ms(fn, n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n

    res = {"d": D, "heads": HEADS, "rounds": args.rounds, "window_s": args.window, "peak_tflops": PEAK_TFLOPS, "shapes": []}
    for lmax, batch in SHAPES:
        lengths, nt, off = synth_lengths(batch, lmax, dev, 1001)
        L = int(off[-1])
        flops = attn_flops(lengths, HEADS, D, D)["bwd"]
        x16, do16 = attn_inputs(L, HEADS, D, dev)
        for dt in (torch.bfloat16, torch.float16):
            x, do = x16.to(dt), do16.to(dt)
            q, k, v = torch.split(x, [D, D, D], dim=-1)
            grads = {name: tuple(torch.empty(L, HEADS, D, device=dev, dtype=dt) for _ in range(3)) for name in impls}

            def call(name):
                dq, dk, dv = grads[name]
                cuda_hstu_attention_bwd(lmax, 1.0 / D, do, q, k, v, dq, dk, dv, off, num_targets=nt, **impls[name])

            iters = {}
            for name in impls:  # warm-up, and the calls that fill one window
                call(name)
                iters[name] = max(1, math.ceil(args.window * 1e3 / time_ms(lambda: call(name), 1)))
            times = {name: [] for name in impls}
            for _ in range(args.rounds):
                for name in impls:
                    times[name].append(time_ms(lambda: call(name), iters[name]))
            med = {name: statistics.median(t) for name, t in times.items()}
            torch.cuda.synchronize()
            names = ("dq", "dk", "dv")
            row = {
                "lmax": lmax, "sequences": batch, "rows": L, "dtype": str(dt).replace("torch.", ""),
                "calls_per_window": iters, "ms_median": med, "ms_all": times,
                "speedup_vs_generic": med["generic"] / med["wgmma"],
                "bwd_flops_per_call": flops,
                "wgmma_tflops": flops / (med["wgmma"] * 1e-3) / 1e12,
                "wgmma_frac_of_peak": flops / (med["wgmma"] * 1e-3) / 1e12 / PEAK_TFLOPS,
                "rel_l2_wgmma_vs_generic": {n: rel_l2(a, b) for n, a, b in zip(names, grads["wgmma"], grads["generic"])},
                "finite": all(bool(torch.isfinite(a).all()) for a in grads["wgmma"]),
            }
            res["shapes"].append(row)
            print(json.dumps({k: row[k] for k in ("lmax", "dtype", "ms_median", "speedup_vs_generic", "wgmma_tflops")}),
                  file=sys.stderr, flush=True)
            del grads
        del x16, do16
        torch.cuda.empty_cache()
    res["card"] = card()  # read right after the timing, so the SM clock is the loaded one
    res["triton"] = {f"lmax{lmax}": triton_row(lmax, batch) for lmax, batch in SHAPES}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
