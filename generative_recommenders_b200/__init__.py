"""generative_recommenders_b200 -- H100 (sm_90a) backend of the HSTU hot path.

Python host layer mirroring the reference operator surface (`generative_recommenders.ops.*`,
`generative_recommenders.modules.stu`) on top of the C-ABI library libhstu_b200.so (include/hstu_b200.h).
Only `HammerKernel.CUDA` is implemented here; there is no eager / CPU fallback.
"""
from .common import HammerKernel, HammerModule  # noqa: F401

__version__ = "0.1.0"
