"""In-tree build of libhstu_b200.so (sm_90a only).

    python -m generative_recommenders_b200.build [--force]

Each translation unit under csrc/ is compiled with
    nvcc -std=c++20 -gencode arch=compute_90a,code=sm_90a -lineinfo -O3
and linked into generative_recommenders_b200/lib/libhstu_b200.so (+ the test-only libhstu_b200_selftest.so; git-ignored).  nvcc cross-compiles without a GPU, so this is also the "does it build" check of __graft_entry__.build().
"""
import concurrent.futures
import importlib.util
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(ROOT, "build", "hstu_b200")
LIB = os.path.join(HERE, "lib", "libhstu_b200.so")
SELFTEST_LIB = os.path.join(HERE, "lib", "libhstu_b200_selftest.so")  # test infrastructure: wgmma / TMA self test
GEN = os.path.join(OBJ, "gen")  # generated headers (wgmma_ops.cuh, scripts/gen_wgmma_ops.py)
SELFTEST_SOURCES = ["wgmma_selftest.cu", "tmap.cu"]
SOURCES = ["api.cu", "attn_generic.cu", "attn_wgmma_fwd.cu", "attn_wgmma_bwd.cu", "attn_wgmma_fwd_e4m3.cu", "attn_wgmma_mixed_fwd.cu", "attn_wgmma_mixed_fwd_e4m3.cu", "attn_wgmma_mixed_bwd.cu", "attn_wgmma_delta_fp8kv.cu", "attn_wgmma_bidir.cu", "attn_fp16_operands.cu", "tmap.cu", "norm.cu", "norm_fast.cu", "jagged.cu", "position.cu", "sampled_softmax.cu", "jagged_bmm.cu"]
NVCC_FLAGS = [
    "-std=c++20", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-Wall", "-Xcudafe", "--diag_suppress=177",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def _deps_mtime() -> float:
    paths = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(ROOT, "include", "hstu_b200.h"), __file__,
                                                                  os.path.join(ROOT, "scripts", "gen_wgmma_ops.py")]
    return max(os.path.getmtime(p) for p in paths)


def is_fresh() -> bool:
    return all(os.path.exists(p) and os.path.getmtime(p) >= _deps_mtime() for p in (LIB, SELFTEST_LIB))


def _compile(src: str, extra, reuse: bool = False) -> str:
    obj = os.path.join(OBJ, src.replace(".cu", ".o"))
    if reuse and os.path.exists(obj):
        return obj
    hdrs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))]
    hdrs += [os.path.join(ROOT, "include", "hstu_b200.h"), os.path.join(GEN, "wgmma_ops.cuh")]
    newest = max(os.path.getmtime(p) for p in hdrs + [os.path.join(CSRC, src), __file__])
    if os.path.exists(obj) and os.path.getmtime(obj) >= newest:
        return obj
    cmd = [_nvcc()] + NVCC_FLAGS + ["-I", GEN] + list(extra) + ["-c", os.path.join(CSRC, src), "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
    if r.stderr.strip():
        sys.stderr.write(r.stderr)
    return obj


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and is_fresh():
        return LIB
    os.makedirs(OBJ, exist_ok=True)
    os.makedirs(os.path.dirname(LIB), exist_ok=True)
    if force and not os.environ.get("HSTU_EXP_SRC"):
        for f in os.listdir(OBJ):
            if os.path.isfile(os.path.join(OBJ, f)):  # objects only: GEN is a directory, regenerated below
                os.remove(os.path.join(OBJ, f))
    spec = importlib.util.spec_from_file_location("gen_wgmma_ops", os.path.join(ROOT, "scripts", "gen_wgmma_ops.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    gen.main(GEN)
    extra = ["-Xptxas", "-v"] if verbose else []
    if os.environ.get("HSTU_DEBUG_SPIN"):
        extra.append("-DHSTU_DEBUG_SPIN")
    for flag in os.environ.get("HSTU_EXP", "").split():
        extra.append("-D" + flag)
    all_src = list(dict.fromkeys(SOURCES + SELFTEST_SOURCES))
    # HSTU_EXP_SRC="norm.cu,...": an experiment that touches only these units -- recompile them with the HSTU_EXP defines and
    # link against the existing objects of everything else (A/B runs on the GPU box without a two-minute full rebuild)
    only = [t for t in os.environ.get("HSTU_EXP_SRC", "").split(",") if t]
    for t in only:
        o = os.path.join(OBJ, t.replace(".cu", ".o"))
        if os.path.exists(o):
            os.remove(o)
    with concurrent.futures.ThreadPoolExecutor(max_workers=min(8, len(all_src))) as ex:
        objs = dict(zip(all_src, ex.map(lambda s: _compile(s, extra if (not only or s in only) else [], reuse=bool(only) and s not in only),
                                        all_src)))
    for lib, srcs in ((LIB, SOURCES), (SELFTEST_LIB, SELFTEST_SOURCES)):
        cmd = [_nvcc(), "-shared", "-o", lib] + [objs[s] for s in srcs] + ["-gencode", "arch=compute_90a,code=sm_90a"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
