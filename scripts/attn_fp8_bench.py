"""Forward attention on fp8 (e4m3) inputs against bf16 and fp16 on the same values, in one process.

    python scripts/attn_fp8_bench.py [--rounds 5] [--window 0.5] [--mixed-dims] [--out FILE]

Inputs: `bench.py`'s length recipe (`synth_lengths`: lengths U[0.9, 1) Lmax with 1-20 targets, seed 1001); q, k ~ N(0, 1)
and v ~ N(0, 1), alpha = 1/sqrt(d) (rms(alpha S) = 1).  q, k, v are quantised per (sequence, head) with descale = amax / 448;
the bf16 and fp16 arms run on the dequantised values (x8 * descale) rounded to their dtype.  Shapes (d, Lmax, sequences,
heads): the headline attention d = 32 at 8192 / 16 / 8, and d = 64 at 2048 / 128, d = 128 at 4096 / 32, d = 256 at
1024 / 128, all with 4 heads.  `--mixed-dims` runs the dqk < dv cells instead, with the batches of attn_mixed_dims_bench.py:
(128, 256) at Lmax 512 / 2048 / 8192 with 512 / 128 / 16 sequences, and (32, 64), (32, 128), (32, 256), (64, 128),
(64, 256) at Lmax 2048 with 128 sequences, all with 4 heads; q, k have dqk columns, v has dv, and alpha = 1/sqrt(dqk).

Each arm is warmed up.  Then, in every round, the three arms run one after another with CUDA events, each over enough
back-to-back calls to fill `--window` seconds; medians over rounds are reported (wall-clock ms per call; the fp8 arm includes
its pre-pass, the fp16 copy of v).  The card runs under a power limit, so its SM clock depends on what it runs: during every
window a thread reads the SM clock and the power draw through NVML (read-only queries), and each arm's medians are reported
beside its time.  Kernel-level times come from `torch.profiler` over whole sustained windows, alternated the same way
(`--profile-rounds`): the device time of each arm's kernels per call, the idle time of the device inside the window (wall
minus kernel time), and the kernel time in SM clock cycles (kernel time x the window's median SM clock), which does not
depend on the clock the power limit allowed.  Each arm's rel-L2 against an fp64 evaluation of the same (dequantised)
values is taken on two sampled sequences.

Prints one JSON line (also written to --out) with the card's name, power limit and SM clock, read in the same run.
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys
import threading

import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)

SHAPES = [(32, 32, 8192, 16, 8), (64, 64, 2048, 128, 4), (128, 128, 4096, 32, 4), (256, 256, 1024, 128, 4)]  # (dqk, dv, ...)
MIXED_SHAPES = [(128, 256, 512, 512, 4), (128, 256, 2048, 128, 4), (128, 256, 8192, 16, 4)] + [
    (dqk, dv, 2048, 128, 4) for dqk, dv in [(32, 64), (32, 128), (32, 256), (64, 128), (64, 256)]]
FP8 = torch.float8_e4m3fn


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), (s.strip() for s in out.split(","))))
    except Exception as e:  # the timing itself does not depend on nvidia-smi
        return {"name": torch.cuda.get_device_name(0), "error": str(e)}


class Sampler:
    """Median SM clock (MHz) and power draw (W) of GPU 0 while the `with` block runs, read through NVML every 10 ms."""

    def __init__(self):
        try:
            import pynvml

            pynvml.nvmlInit()
            self.nv, self.h = pynvml, pynvml.nvmlDeviceGetHandleByIndex(torch.cuda.current_device())
        except Exception:  # the timing does not depend on NVML; the clock and power fields are then None
            self.nv = None

    def __enter__(self):
        self.clk, self.pw, self.stop = [], [], threading.Event()
        if self.nv is not None:
            self.t = threading.Thread(target=self._run, daemon=True)
            self.t.start()
        return self

    def _run(self):
        while not self.stop.wait(0.01):
            self.clk.append(self.nv.nvmlDeviceGetClockInfo(self.h, self.nv.NVML_CLOCK_SM))
            self.pw.append(self.nv.nvmlDeviceGetPowerUsage(self.h) / 1e3)

    def __exit__(self, *exc):
        self.stop.set()
        if self.nv is not None:
            self.t.join()
        return False

    def medians(self):
        med = lambda x: statistics.median(x) if x else None  # noqa: E731
        return med(self.clk), med(self.pw)


def quantize(x, off):
    """Per (sequence, head): descale = amax / 448, x8 = e4m3(x / descale); returns x8 and the descales [B, H]."""
    o = off.tolist()
    ds = torch.ones(len(o) - 1, x.shape[1], device=x.device)
    x8 = torch.empty(x.shape, dtype=FP8, device=x.device)
    for b in range(len(o) - 1):
        s, e = o[b], o[b + 1]
        if e > s:
            amax = x[s:e].float().abs().amax(dim=(0, 2))
            ds[b] = torch.where(amax > 0, amax / 448.0, torch.ones_like(amax))
            x8[s:e] = (x[s:e].float() / ds[b][None, :, None]).clamp(-448, 448).to(FP8)
    return x8, ds


def ref_fp64(N, alpha, q, k, v, s, e, nt, O):
    """fp64 attention of rows [s, e) (one sequence, all heads) on the GPU; q, k, v already dequantised (fp64)."""
    n = min(e - s, N)
    m = torch.from_numpy(O.attn_valid_mask(n, nt, 0, 0, 0)).to(q.device, torch.float64)
    qb, kb, vb = (t[s:s + n].transpose(0, 1) for t in (q, k, v))
    p = torch.nn.functional.silu(torch.matmul(qb, kb.transpose(1, 2)) * alpha) / N * m
    return torch.matmul(p, vb).transpose(0, 1)


def rel_l2(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--window", type=float, default=0.5, help="seconds of back-to-back calls per timed window")
    ap.add_argument("--profile-rounds", type=int, default=2, help="alternated rounds of profiled sustained windows")
    ap.add_argument("--mixed-dims", action="store_true", help="the dqk < dv cells (MIXED_SHAPES) instead of SHAPES")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from bench import ensure_built, synth_lengths
    from generative_recommenders_b200.ops.hstu_attention import cuda_hstu_attention_fwd
    from oracle import hstu_oracle as O

    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    ensure_built()
    dev = torch.device("cuda", 0)

    def time_ms(fn, n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n

    res = {"rounds": args.rounds, "window_s": args.window, "shapes": []}
    for dqk, dv, lmax, batch, heads in (MIXED_SHAPES if args.mixed_dims else SHAPES):
        lengths, nt, off = synth_lengths(batch, lmax, dev, 1001)
        L = int(off[-1])
        g = torch.Generator(device=dev).manual_seed(3003)
        q8, k8, v8 = (quantize(torch.randn(L, heads, w, device=dev, generator=g), off) for w in (dqk, dqk, dv))
        ds = (q8[1], k8[1], v8[1])
        q8, k8, v8 = q8[0], k8[0], v8[0]
        o = off.tolist()
        rows = torch.repeat_interleave(torch.arange(batch, device=dev), torch.tensor([o[i + 1] - o[i] for i in range(batch)], device=dev))
        deq = [x.double() * dd.double()[rows][:, :, None] for x, dd in zip((q8, k8, v8), ds)]
        arms = {"fp8": (q8, k8, v8), "bf16": tuple(x.to(torch.bfloat16) for x in deq), "fp16": tuple(x.to(torch.float16) for x in deq)}
        alpha = 1.0 / math.sqrt(dqk)
        outs = {}

        def call(name):
            q, k, v = arms[name]
            kw = dict(descales=ds) if name == "fp8" else {}
            outs[name] = cuda_hstu_attention_fwd(lmax, alpha, q, k, v, off, num_targets=nt, **kw)

        iters = {}
        for name in arms:
            call(name)
            iters[name] = max(1, math.ceil(args.window * 1e3 / time_ms(lambda: call(name), 2)))
        sampler = Sampler()
        times, clock, power = ({name: [] for name in arms} for _ in range(3))
        for _ in range(args.rounds):
            for name in arms:
                with sampler:
                    times[name].append(time_ms(lambda: call(name), iters[name]))
                c, w = sampler.medians()
                clock[name].append(c)
                power[name].append(w)
        med = {name: statistics.median(t) for name, t in times.items()}
        med_or_none = lambda x: statistics.median(x) if None not in x else None  # noqa: E731
        clock_med = {name: med_or_none(c) for name, c in clock.items()}
        power_med = {name: med_or_none(w) for name, w in power.items()}
        # accuracy on two sampled sequences (the outputs of each arm's last call)
        torch.cuda.synchronize()
        errs = {name: [] for name in arms}
        for b in (0, batch // 2):
            ref = ref_fp64(lmax, alpha, *deq, o[b], o[b + 1], int(nt[b]), O)
            n = ref.shape[0]
            for name in arms:
                errs[name].append(rel_l2(outs[name][o[b]:o[b] + n], ref))
        # kernel-level: profiled sustained windows, arms alternated as above.  Per arm and window: device time of its kernels per
        # call (by kernel), wall time per call of the same window, and the window's median SM clock
        from torch.profiler import ProfilerActivity, profile

        prof_rows = {name: [] for name in arms}
        for _ in range(args.profile_rounds):
            for name in arms:
                with sampler, profile(activities=[ProfilerActivity.CUDA]) as prof:
                    wall = time_ms(lambda: call(name), iters[name])
                kern = {}
                for ev in prof.key_averages():
                    t = getattr(ev, "device_time_total", None)
                    if t is None:
                        t = getattr(ev, "cuda_time_total", 0.0)
                    if t > 0 and "kernel" in ev.key.lower():
                        kern[ev.key[:120]] = kern.get(ev.key[:120], 0.0) + t / 1e3 / iters[name]
                prof_rows[name].append((wall, sum(kern.values()), sampler.medians()[0], kern))
        kernel_ms, kernels, idle_ms, kcycles = {}, {}, {}, {}
        for name, rows_ in prof_rows.items():
            kernel_ms[name] = statistics.median(r[1] for r in rows_)
            idle_ms[name] = statistics.median(r[0] - r[1] for r in rows_)
            kcycles[name] = statistics.median(r[1] * r[2] for r in rows_) if None not in (r[2] for r in rows_) else None
            kernels[name] = {k: statistics.median(r[3].get(k, 0.0) for r in rows_) for k in rows_[0][3]}
        prepass = sum(t for k, t in kernels["fp8"].items() if "convert_kernel" in k)
        attn = sum(t for k, t in kernels["fp8"].items() if "e4m3_wgmma_kernel" in k or "e4m3_mixed_wgmma_kernel" in k)
        row = {
            **({"d": dqk} if dqk == dv else {"dqk": dqk, "dv": dv}), "lmax": lmax, "sequences": batch, "heads": heads, "rows": L, "calls_per_window": iters,
            "ms_median": med, "ms_all": times, "fp8_over_bf16": med["fp8"] / med["bf16"], "fp8_over_fp16": med["fp8"] / med["fp16"],
            "sm_clock_mhz_median": clock_med, "power_w_median": power_med,
            "kernel_ms_per_call": kernel_ms, "kernel_fp8_over_bf16": kernel_ms["fp8"] / kernel_ms["bf16"],
            "kernel_fp8_over_fp16": kernel_ms["fp8"] / kernel_ms["fp16"], "device_idle_ms_per_call": idle_ms,
            "kernel_kilocycles_per_call": kcycles,
            "profile_fp8_ms_per_call": {"prepass_v_to_fp16": prepass, "attention_kernel": attn,
                                        **({} if dqk == dv else {"prepass_share": prepass / (prepass + attn)})},
            "profile_kernels_ms_per_call": kernels,
            "rel_l2_vs_fp64_sampled": {name: max(e) for name, e in errs.items()},
            "finite": all(bool(torch.isfinite(x).all()) for x in outs.values()),
        }
        res["shapes"].append(row)
        print(json.dumps({k: row[k] for k in ("d", "dqk", "dv", "lmax", "ms_median", "fp8_over_bf16", "fp8_over_fp16", "sm_clock_mhz_median",
                                               "power_w_median", "kernel_ms_per_call", "kernel_fp8_over_bf16",
                                               "kernel_fp8_over_fp16", "device_idle_ms_per_call", "kernel_kilocycles_per_call",
                                               "profile_fp8_ms_per_call", "rel_l2_vs_fp64_sampled") if k in row}), file=sys.stderr,
              flush=True)
        del arms, outs, deq
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
