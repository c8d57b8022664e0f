"""Registers, spills and tanh schedule of the wgmma attention kernels, read from the compiler's output (no GPU needed).

    python scripts/sass_report.py [--kernel SUBSTRING]

Compiles the wgmma attention units (UNITS) to sm_90a cubins with the flags of build.py plus `-Xptxas -v`, and prints
one JSON line per wgmma attention kernel: its registers, spill stores / loads (bytes), the ptxas notes and warnings it got
(C7510 / C7512 / C7515: wgmma serialisation; C7519: a warpgroup.arrive ptxas inserted), and `tanh_per_block`, the most
MUFU.TANH instructions in one basic block of its SASS (`cuobjdump -sass`).  A block ends at a branch and starts at a branch
target.  The elementwise stage of these kernels issues one tanh per score; when a per-score branch splits the stage into
one block per score, tanh_per_block is 1 and every warp waits out the full MUFU latency once per score, since nothing
independent is left in the block to issue in between.  `iter_instrs` is what one thread issues in one steady-state tile
iteration on the full-tile path, spin loops counted once (iter_instrs below): the tanh block plus the ring, descriptor and
branch bookkeeping around the MMAs.
"""
import argparse
import concurrent.futures
import importlib.util
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
CSRC = os.path.join(ROOT, "generative_recommenders_b200", "csrc")
UNITS = ("attn_wgmma_fwd.cu", "attn_wgmma_bwd.cu", "attn_wgmma_fwd_e4m3.cu", "attn_wgmma_mixed_fwd.cu", "attn_wgmma_mixed_bwd.cu",
         "attn_wgmma_mixed_fwd_e4m3.cu", "attn_wgmma_delta_fp8kv.cu",
         "attn_wgmma_bidir.cu")
_CTRL = ("BRA", "BRX", "JMP", "JMX", "CALL", "RET", "EXIT", "BSSY")  # instructions that end a block or name a branch target


def tools():
    """(nvcc, cuobjdump, cu++filt) or None when the CUDA toolkit is not installed."""
    nvcc = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        return None
    bindir = os.path.dirname(os.path.realpath(nvcc))
    found = [shutil.which(t) or os.path.join(bindir, t) for t in ("cuobjdump", "cu++filt")]
    return (nvcc, *found) if all(os.path.exists(t) for t in found) else None


def _load_build():
    spec = importlib.util.spec_from_file_location("hstu_build", os.path.join(ROOT, "generative_recommenders_b200", "build.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def parse_ptxas(log):
    """ptxas -v output -> {mangled kernel: {"registers", "spill_stores", "spill_loads", "notes": ["C7519", ...]}}"""
    out, cur = {}, None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", line)
        if m:
            cur = out.setdefault(m.group(1), {"notes": []})
            continue
        m = re.search(r"\((C\d+)\).*in function '([^']+)'", line)
        if m:
            out.setdefault(m.group(2), {"notes": []})["notes"].append(m.group(1))
            continue
        if cur is None:
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m:
            cur["spill_stores"], cur["spill_loads"] = int(m.group(1)), int(m.group(2))
        m = re.search(r"Used (\d+) registers", line)
        if m:
            cur["registers"] = int(m.group(1))
    return out


def max_tanh_per_block(sass):
    """The most MUFU.TANH in one basic block of one function's `cuobjdump -sass` listing."""
    ins = []  # (address, instruction text)
    for line in sass.splitlines():
        m = re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;", line)
        if m:
            ins.append((int(m.group(1), 16), m.group(2)))
    starts = set()
    for i, (addr, text) in enumerate(ins):
        op = re.sub(r"^@!?U?P[T0-9]+\s+", "", text).split()[0].split(".")[0]
        if op in _CTRL:
            starts.update(int(t, 16) for t in re.findall(r"0x([0-9a-f]+)", text))
            if op != "BSSY" and i + 1 < len(ins):
                starts.add(ins[i + 1][0])
    best = run = 0
    for addr, text in ins:
        if addr in starts:
            run = 0
        if "MUFU.TANH" in text:
            run += 1
            best = max(best, run)
    return best


def _blocks(sass):
    """Basic blocks of one function's listing: [(first address, [instruction text]), ...] in address order, and the successor
    addresses of each block (taken branch targets and, unless the block ends in an unpredicated branch or exit, the next
    block)."""
    ins = []
    for line in sass.splitlines():
        m = re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;", line)
        if m and not m.group(2).startswith("NOP"):
            ins.append((int(m.group(1), 16), m.group(2)))
    starts, ends = {ins[0][0]} if ins else set(), set()
    for i, (addr, text) in enumerate(ins):
        op = re.sub(r"^@!?U?P[T0-9]+\s+", "", text).split()[0].split(".")[0]
        if op in _CTRL and op != "BSSY":
            starts.update(int(t, 16) for t in re.findall(r"0x([0-9a-f]+)", text) if op != "CALL")
            ends.add(addr)
    blocks = []
    for addr, text in ins:
        if addr in starts or not blocks or blocks[-1][1][-1][0] in ends:
            blocks.append((addr, []))
        blocks[-1][1].append((addr, text))
    succ = {}
    for i, (first, body) in enumerate(blocks):
        text = body[-1][1]
        op = re.sub(r"^@!?U?P[T0-9]+\s+", "", text).split()[0].split(".")[0]
        s = []
        if op in ("BRA", "BRX", "JMP", "JMX"):
            s = [int(t, 16) for t in re.findall(r"0x([0-9a-f]+)", text)]
        falls = text.startswith("@") or op not in ("BRA", "BRX", "JMP", "JMX", "EXIT", "RET")
        if falls and i + 1 < len(blocks):
            s.append(blocks[i + 1][0])
        succ[first] = s
    return [(first, [t for _, t in body]) for first, body in blocks], succ


def iter_instrs(sass):
    """Instructions one thread issues in one steady-state iteration of the tile loop, on the path through the elementwise
    block of the most MUFU.TANH (the full-tile path, where no score is masked).  The tile loop is the smallest loop that holds
    that block.  Inside it every back edge is dropped, so that a spin loop (an mbarrier wait) counts once, and the iteration
    is the path from the loop head through that block to the back edge with the most HGMMA (every MMA of a tile: not the
    last tile, which issues no MMA for the next one), and of those the one of the fewest instructions: branches taken only
    by some warps or on some tiles (the refill, the mask cases, the zeroing of rows past the sequence end) are not on it.
    None when there is no such loop."""
    blocks, succ = _blocks(sass)
    tanh = {a: sum("MUFU.TANH" in t for t in body) for a, body in blocks}
    if not tanh or max(tanh.values()) == 0:
        return None
    best_t = max(tanh.values())
    targets = [a for a in tanh if tanh[a] == best_t]
    pred = {a: [] for a, _ in blocks}
    for a, s in succ.items():
        for b in s:
            if b in pred:
                pred[b].append(a)
    loops = []  # (nodes, head, tail) of each back edge tail -> head
    for a, s in succ.items():
        for head in s:
            if head <= a and head in pred:
                nodes, stack = {head, a}, [a]
                while stack:
                    for p in pred[stack.pop()]:
                        if p not in nodes:
                            nodes.add(p)
                            stack.append(p)
                if any(t in nodes for t in targets):
                    loops.append((nodes, head, a))
    if not loops:
        return None
    nodes, head, tail = min(loops, key=lambda x: len(x[0]))

    # a path's cost is (-HGMMA, instructions), least first; both ends counted
    cost = {a: (-sum(t.startswith("HGMMA") for t in body), len(body)) for a, body in blocks}

    def add(x, y, sign=1):
        return (x[0] + sign * y[0], x[1] + sign * y[1])

    def dist_from(src, forward):  # least cost of a forward (address-increasing) path inside the loop from / to src
        d = {src: cost[src]}
        for a in sorted(nodes, reverse=not forward):
            if a not in d:
                continue
            nxt = [b for b in succ[a] if b in nodes and b > a] if forward else [p for p in pred[a] if p in nodes and p < a]
            for b in nxt:
                c = add(d[a], cost[b])
                if b not in d or c < d[b]:
                    d[b] = c
        return d

    down, up = dist_from(head, True), dist_from(tail, False)
    paths = [add(add(down[t], up[t]), cost[t], -1) for t in targets if t in down and t in up]
    return min(paths)[1] if paths else None


def _sass_by_function(text):
    funcs, name, buf = {}, None, []
    for line in text.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            if name:
                funcs[name] = "\n".join(buf)
            name, buf = m.group(1), []
        elif name:
            buf.append(line)
    if name:
        funcs[name] = "\n".join(buf)
    return funcs


def report(kernel_filter="wgmma_kernel"):
    """{demangled kernel name: {"registers", "spill_stores", "spill_loads", "notes", "tanh_per_block"}} of the attention
    kernels whose name contains `kernel_filter`."""
    tl = tools()
    if tl is None:
        raise RuntimeError("nvcc / cuobjdump / cu++filt not found")
    nvcc, cuobjdump, cufilt = tl
    build = _load_build()
    res = {}
    with tempfile.TemporaryDirectory(prefix="hstu_sass_") as tmp:
        gen = os.path.join(tmp, "gen")
        spec = importlib.util.spec_from_file_location("gen_wgmma_ops", os.path.join(ROOT, "scripts", "gen_wgmma_ops.py"))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        mod.main(gen)

        def one(unit):
            cubin = os.path.join(tmp, unit.replace(".cu", ".cubin"))
            r = subprocess.run([nvcc] + build.NVCC_FLAGS + ["-I", gen, "-Xptxas", "-v", "-cubin", os.path.join(CSRC, unit), "-o", cubin],
                               capture_output=True, text=True)
            if r.returncode != 0:
                raise RuntimeError(f"nvcc failed for {unit}:\n{r.stderr}")
            sass = subprocess.run([cuobjdump, "-sass", cubin], capture_output=True, text=True, check=True).stdout
            return parse_ptxas(r.stdout + r.stderr), _sass_by_function(sass)

        with concurrent.futures.ThreadPoolExecutor(len(UNITS)) as ex:
            parts = list(ex.map(one, UNITS))
    for info, funcs in parts:
        for mangled, sass in funcs.items():
            name = subprocess.run([cufilt, mangled], capture_output=True, text=True, check=True).stdout.strip()
            if kernel_filter not in name:
                continue
            res[name] = {**info.get(mangled, {"notes": []}), "tanh_per_block": max_tanh_per_block(sass),
                         "iter_instrs": iter_instrs(sass)}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--kernel", default="wgmma_kernel", help="report kernels whose demangled name contains this")
    args = ap.parse_args()
    for name, r in sorted(report(args.kernel).items()):
        print(json.dumps({"kernel": name, **r}))


if __name__ == "__main__":
    sys.exit(main())
