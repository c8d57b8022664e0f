"""Peak memory and per-kernel device time of the headline training step of `bench.py`.

    python scripts/stu_step_profile.py [--steps 2] [--warmup 3] [--out FILE]

The stack, inputs and step of `bench.py --workload hstu_large` (16 STU layers, D = 256, H = 8, dqk = dv = 32, bf16,
Lmax 8192, 16 sequences of seed 1001, dropout 0.2, recompute_uvqk / normed_x / y, AdamW), without the timing windows.  After
`--warmup` steps it reports `torch.cuda.max_memory_allocated()` over one step, then runs `--steps` steps under torch.profiler
and reports, per step, the device time of the attention pre-pass kernels (`fp16_operands_*`), the attention kernels, and
every `aten::addmm` by input shapes (the uvqk GEMM of the forward and the one the backward recomputes, the output GEMM).
Prints one JSON line with the card's name and power limit; `--out` also writes it to FILE.
"""
import argparse
import json
import os
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
    except Exception as e:  # the measurement itself does not depend on nvidia-smi
        return {"name": torch.cuda.get_device_name(0), "power_limit": f"unknown ({e})"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from bench import ensure_built, synth_lengths
    from generative_recommenders_b200.modules.stu import STULayer, STULayerConfig, STUStack

    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    ensure_built()
    dev = torch.device("cuda", 0)
    D, H, dh, layers, lmax = 256, 8, 32, 16, 8192
    lengths, nt, off = synth_lengths(16, lmax, dev, 1001)
    torch.cuda.manual_seed(4321)
    torch.manual_seed(7)
    stack = STUStack([STULayer(STULayerConfig(embedding_dim=D, num_heads=H, hidden_dim=dh, attention_dim=dh,
                                              output_dropout_ratio=0.2, target_aware=True, recompute_normed_x=True,
                                              recompute_uvqk=True, recompute_y=True, sort_by_length=True))
                      for _ in range(layers)]).to(dev).to(torch.bfloat16)
    opt = torch.optim.AdamW(list(stack.parameters()), lr=1e-4, fused=True)
    torch.manual_seed(100)
    x = torch.randn(int(off[-1]), D, device=dev, dtype=torch.bfloat16)

    def step():
        opt.zero_grad(set_to_none=False)
        y = stack(x=x, x_lengths=lengths, x_offsets=off, max_seq_len=lmax, num_targets=nt)
        y.float().square().mean().backward()
        opt.step()

    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(dev)
    step()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated(dev)

    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU], record_shapes=True) as prof:
        for _ in range(args.steps):
            step()
        torch.cuda.synchronize()
    kernels, addmm = {}, {}
    for e in prof.key_averages():
        t = e.device_time_total / 1e3 / args.steps  # ms per step
        if "fp16_operands" in e.key or "wgmma_kernel" in e.key:
            kernels[e.key] = {"ms_per_step": round(t, 4), "calls_per_step": e.count / args.steps}
    for e in prof.key_averages(group_by_input_shape=True):
        if e.key == "aten::addmm":
            addmm[str(e.input_shapes)] = {"ms_per_step": round(e.device_time_total / 1e3 / args.steps, 4),
                                          "calls_per_step": e.count / args.steps}
    out = {"card": card(), "rows": int(off[-1]), "peak_memory_allocated_bytes": peak,
           "kernels": kernels, "addmm_by_input_shapes": addmm}
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
