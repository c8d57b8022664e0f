#!/usr/bin/env python3
"""CPU-baseline recipe: copy the original project's OWN PyTorch-eager HSTU block (unmodified Python, from a checkout of
facebookresearch/generative-recommenders) into the git-ignored oracle/_ref/, so that `bench.py` can time the real eager
reference (cpu_baseline.kind = "reference") and the reference's Triton attention on machines that have no such checkout.
`__graft_entry__.build()` runs it.  The three fbgemm_gpu jagged ops it calls
are supplied by oracle/fbgemm_shim.py.  Nothing under oracle/_ref/ is committed or imported by the product package.

    python oracle/fetch_reference_eager.py      # checkout at /root/reference, or HSTU_REFERENCE_ROOT=<checkout>

Copied (relative to <checkout>/generative_recommenders/): common.py, modules/stu.py, ops/*.py, ops/pytorch/*.py,
ops/triton/*.py (imported by the facades at module import time; never called on the CPU path).  Without a checkout nothing
is copied (the message says so) and bench.py times the oracle port instead.
"""
import glob
import os
import shutil
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEFAULT_ROOT = "/root/reference"  # where the build environment keeps the checkout of the original project
DST = os.path.join(ROOT, "oracle", "_ref", "generative_recommenders")
PATTERNS = ["common.py", "modules/stu.py", "ops/*.py", "ops/pytorch/*.py", "ops/triton/*.py"]


def main() -> int:
    src_root = os.environ.get("HSTU_REFERENCE_ROOT") or DEFAULT_ROOT
    src = os.path.join(src_root, "generative_recommenders")
    if not os.path.isdir(src):
        print(f"oracle/_ref: no checkout of generative-recommenders at {src_root} (set HSTU_REFERENCE_ROOT): nothing copied; "
              "bench.py will time the oracle port and report the Triton comparator as unavailable", file=sys.stderr)
        return 1
    n = 0
    for pat in PATTERNS:
        for f in sorted(glob.glob(os.path.join(src, pat))):
            dst = os.path.join(DST, os.path.relpath(f, src))
            os.makedirs(os.path.dirname(dst), exist_ok=True)
            shutil.copyfile(f, dst)
            n += 1
    print(f"copied {n} files to {DST}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
