"""The d = 32 attention at the headline shape with bf16 inputs against the same values as fp16 inputs.

    python scripts/attn_fp16_operands_bench.py [--iters 20] [--rounds 5] [--profile DIR]

Headline attention call of `bench.py`: `synth_lengths(16, 8192, seed 1001)`, H = 8, d = 32, num_targets, alpha = 1/d,
`cuda_hstu_attention_fwd/bwd` (the kernels always schedule heavy tiles first, so `sort_by_length` is implied).  The fp16
tensors hold the bf16 values exactly (q, k, v, dO ~ N(0, 1/4) with magnitudes below 2^-10 raised to 2^-10).  The two dtypes are timed in alternating rounds with CUDA
events, `--iters` calls per round and direction, and the medians over rounds are reported.  With bf16 inputs a call runs
the pre-pass that makes exactly scaled fp16 copies and then the fp16 kernels (DESIGN.md section 3.0); with fp16 inputs it
runs the fp16 kernels alone, the ceiling of the bf16 path (before the pre-pass existed, the bf16 kernels multiplied P and dS
as bf16 hi / lo pairs).  `convert_*_ms` is the time of torch's bf16 -> fp16 conversion of the operands each direction
streams (q, k, v; and dO), for comparison with the pre-pass kernels.  `--profile DIR` instead runs a few calls of each dtype under torch.profiler and reports the median time of every
CUDA kernel, with the trace written to DIR.

Prints one JSON line with the card's name and power limit.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, plim, clk = (s.strip() for s in out.split(","))
        return {"name": name, "power_limit": plim, "sm_max_clock": clk}
    except Exception as e:  # the timing itself does not depend on nvidia-smi
        return {"name": torch.cuda.get_device_name(0), "power_limit": f"unknown ({e})"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--profile", default=None, metavar="DIR")
    args = ap.parse_args()
    from bench import ensure_built, synth_lengths
    from generative_recommenders_b200.ops.hstu_attention import cuda_hstu_attention_bwd, cuda_hstu_attention_fwd

    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    ensure_built()
    dev = torch.device("cuda", 0)
    lmax, H, d = 8192, 8, 32
    lengths, nt, off = synth_lengths(16, lmax, dev, 1001)
    L = int(off[-1])
    alpha = 1.0 / d
    torch.manual_seed(0)
    # |x| >= 2^-10 keeps every value a normal fp16 number, so the bf16 -> fp16 conversion is exact
    base = [0.5 * torch.randn(L, H, d, device=dev) for _ in range(4)]
    base = [(x.sign() * x.abs().clamp_min(2.0**-10)).to(torch.bfloat16) for x in base]
    ops = {}
    for dt in (torch.bfloat16, torch.float16):
        q, k, v, do = (t.to(dt) for t in base)
        assert all(torch.equal(a.float(), b.float()) for a, b in zip((q, k, v, do), base))
        dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
        ops[dt] = (
            lambda q=q, k=k, v=v: cuda_hstu_attention_fwd(lmax, alpha, q, k, v, off, num_targets=nt),
            lambda q=q, k=k, v=v, do=do, dq=dq, dk=dk, dv=dv: cuda_hstu_attention_bwd(
                lmax, alpha, do, q, k, v, dq, dk, dv, off, num_targets=nt),
        )
    conv = {"fwd": lambda: [t.to(torch.float16) for t in base[:3]], "bwd": lambda: [t.to(torch.float16) for t in base]}

    def time_ms(fn, n):
        fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n

    res = {"card": card(), "rows": L, "heads": H, "d": d, "iters": args.iters, "rounds": args.rounds}
    if args.profile:
        from torch.profiler import ProfilerActivity, profile

        os.makedirs(args.profile, exist_ok=True)
        for dt in ops:
            for fn in ops[dt]:
                fn()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.iters):
                for dt in ops:
                    ops[dt][0]()
                    ops[dt][1]()
            torch.cuda.synchronize()
        prof.export_chrome_trace(os.path.join(args.profile, "attn_fp16_operands.pt.trace.json"))
        per = {}
        for ev in prof.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA:
                per.setdefault(ev.name, []).append(ev.device_time / 1e3)
        res["kernels_ms"] = {name: {"median": statistics.median(t), "n": len(t)} for name, t in sorted(per.items())}
        print(json.dumps(res))
        return

    times = {k: [] for k in ("bf16_fwd", "bf16_bwd", "fp16_fwd", "fp16_bwd", "convert_fwd", "convert_bwd")}
    for dt in ops:  # warm-up
        for fn in ops[dt]:
            time_ms(fn, 2)
    for _ in range(args.rounds):
        for tag, dt in (("bf16", torch.bfloat16), ("fp16", torch.float16)):
            times[f"{tag}_fwd"].append(time_ms(ops[dt][0], args.iters))
            times[f"{tag}_bwd"].append(time_ms(ops[dt][1], args.iters))
        times["convert_fwd"].append(time_ms(conv["fwd"], args.iters))
        times["convert_bwd"].append(time_ms(conv["bwd"], args.iters))
    med = {k: statistics.median(v) for k, v in times.items()}
    res["ms_median"] = med
    res["ms_all"] = times
    bf, fp = med["bf16_fwd"] + med["bf16_bwd"], med["fp16_fwd"] + med["fp16_bwd"]
    res["saving_fraction"] = (bf - fp) / bf
    res["saving_fraction_after_convert"] = (bf - fp - med["convert_fwd"] - med["convert_bwd"]) / bf
    print(json.dumps(res))


if __name__ == "__main__":
    main()
