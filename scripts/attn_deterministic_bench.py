"""Cost of a bitwise-reproducible attention backward: the default, `deterministic=True` and the generic kernels, timed on the
same inputs in one process.

    python scripts/attn_deterministic_bench.py [--rounds 5] [--window 0.5] [--out FILE]

Inputs: the `bench.py --workload attn` recipe (`synth_lengths`: lengths U[0.9, 1) Lmax with 1-20 targets, seed 1001;
`attn_inputs`: q, k, v as strided views of one [L, H, 3d] buffer, dO ~ N(0, 1)), alpha = 1/d, H = 4, bf16 and fp16 (the
fp16 inputs are the bf16 values converted).  Shapes: d = 64 at Lmax 2048, d = 128 at Lmax 4096, d = 32 at Lmax 8192.

Each (shape, dtype) is warmed up first.  Then, in every round, the three implementations of `cuda_hstu_attention_bwd` are
timed one after another with CUDA events, each over enough back-to-back calls to fill `--window` seconds:
  default        AUTO, deterministic=False: the fused wgmma kernel + dQ convert at d = 64 / 128, the split kernels at d = 32;
  deterministic  AUTO, deterministic=True: the atomic-free dK / dV and dQ wgmma kernels;
  generic        IMPL_GENERIC: the CUDA-core kernels (reproducible too), what deterministic=True ran before.
The medians over rounds are reported.  On the same inputs it also reports the rel-L2 distance of the deterministic result
to the default and to the generic result, and whether two deterministic calls are bitwise equal.

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

SHAPES = [  # (d, Lmax, sequences): a call of a few milliseconds or more on the wgmma kernels
    (64, 2048, 128),
    (128, 4096, 32),
    (32, 8192, 16),
]
HEADS = 4


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--window", type=float, default=0.5, help="seconds of back-to-back calls per timed window")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from bench import attn_inputs, ensure_built, synth_lengths
    from generative_recommenders_b200 import _lib
    from generative_recommenders_b200.ops.hstu_attention import cuda_hstu_attention_bwd

    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    ensure_built()
    dev = torch.device("cuda", 0)
    impls = {"default": dict(deterministic=False), "deterministic": dict(deterministic=True),
             "generic": dict(impl=_lib.IMPL_GENERIC)}

    def time_ms(fn, n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n

    res = {"heads": HEADS, "rounds": args.rounds, "window_s": args.window, "shapes": []}
    for d, lmax, batch in SHAPES:
        lengths, nt, off = synth_lengths(batch, lmax, dev, 1001)
        L = int(off[-1])
        x16, do16 = attn_inputs(L, HEADS, d, dev)
        for dt in (torch.bfloat16, torch.float16):
            x, do = x16.to(dt), do16.to(dt)
            q, k, v = torch.split(x, [d, d, d], dim=-1)
            grads = {name: tuple(torch.empty(L, HEADS, d, device=dev, dtype=dt) for _ in range(3)) for name in impls}

            def call(name):
                dq, dk, dv = grads[name]
                cuda_hstu_attention_bwd(lmax, 1.0 / d, do, q, k, v, dq, dk, dv, off, num_targets=nt, **impls[name])

            iters = {}
            for name in impls:  # warm-up, and the calls that fill one window
                call(name)
                iters[name] = max(1, math.ceil(args.window * 1e3 / time_ms(lambda: call(name), 2)))
            times = {name: [] for name in impls}
            for _ in range(args.rounds):
                for name in impls:
                    times[name].append(time_ms(lambda: call(name), iters[name]))
            med = {name: statistics.median(t) for name, t in times.items()}
            # outputs on the same inputs: the buffers hold each implementation's last call
            torch.cuda.synchronize()
            det = [g.clone() for g in grads["deterministic"]]
            call("deterministic")
            torch.cuda.synchronize()
            again = grads["deterministic"]
            names = ("dq", "dk", "dv")
            row = {
                "d": d, "lmax": lmax, "sequences": batch, "rows": L, "dtype": str(dt).replace("torch.", ""),
                "calls_per_window": iters, "ms_median": med, "ms_all": times,
                "speedup_vs_generic": med["generic"] / med["deterministic"],
                "ratio_to_default": med["deterministic"] / med["default"],
                "rel_l2_det_vs_default": {n: rel_l2(a, b) for n, a, b in zip(names, det, grads["default"])},
                "rel_l2_det_vs_generic": {n: rel_l2(a, b) for n, a, b in zip(names, det, grads["generic"])},
                "det_bitwise_repeatable": all(torch.equal(a.view(torch.int16), b.view(torch.int16)) for a, b in zip(det, again)),
                "finite": all(bool(torch.isfinite(a).all()) for a in det),
            }
            res["shapes"].append(row)
            print(json.dumps({k: row[k] for k in ("d", "lmax", "dtype", "ms_median", "speedup_vs_generic", "ratio_to_default",
                                                   "det_bitwise_repeatable")}), file=sys.stderr, flush=True)
    res["card"] = card()  # read right after the timing, so the SM clock is the loaded one
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
