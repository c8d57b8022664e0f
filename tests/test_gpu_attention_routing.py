"""The routing table of the attention C ABI on an sm_90 device: for every (dtype, dqk, dv) the wgmma kernels take, and a few
they refuse, what hstu_attn_select_impl, hstu_attn_workspace_bytes, hstu_attn_fp16_operands_bytes,
hstu_attn_bwd_fp16_operands_workspace_bytes and the non-causal hstu_attn_bidir_select_impl and
hstu_attn_bidir_workspace_bytes return, forward and backward, with delta-q (one key chunk and several), the
deterministic flag, a relative bias, each impl request, and one misaligned view per tensor.  Nothing is launched: the
pointers are placeholders.  `_want` is the table; a routing change edits it on purpose."""
import ctypes as C

import pytest
import torch

from test_attention_deterministic_cpu import HSTU_ERR_UNSUPPORTED, _params

pytestmark = pytest.mark.gpu

SQUARE = [(32, 32), (64, 64), (128, 128), (256, 256)]
MIXED = [(32, 64), (32, 128), (32, 256), (64, 128), (64, 256), (128, 256)]
REFUSED = [(64, 32), (256, 128), (40, 40)]
TENSORS = ["q", "k", "v", "out", "dout", "dq", "dk", "dv_out"]
READS = {False: {"q", "k", "v", "out"}, True: set(TENSORS)}  # the backward does not read out, but refuses a misaligned base
H, ROWS, DELTA = 2, 4096, 16


def _align256(n):
    return (n + 255) // 256 * 256


def _case(dtype, dqk, dv, bwd, det=0, bias=False, batch=2, delta=0, mis=None, impl=0):
    p = _params(dtype, dqk, dv, deterministic=det, impl=impl, rows=ROWS, bias=bias)
    p.batch, p.delta_q_len = batch, delta
    if mis == "q_stride":  # a row stride of 8 elements more: a whole 16-byte unit for 16-bit data, half of one for e4m3
        p.q_row_stride += 8
    elif mis is not None:  # a base 2 bytes past a 16-byte boundary
        setattr(p, mis, getattr(p, mis) + 2)
    return p


def _variants(bwd):
    yield {}
    yield {"det": 1}
    yield {"bias": True}
    yield {"bias": True, "det": 1}
    if not bwd:
        yield {"delta": DELTA, "batch": 2}  # 2 x 2 x 1 query-tile CTAs: the 2048 keys split into 4 chunks
        yield {"delta": DELTA, "batch": 132}  # 264 CTAs: one chunk
    yield {"mis": "q_stride"}
    for t in TENSORS:
        yield {"mis": t}


def _select(dtype, dqk, dv, bwd, det=0, bias=False, batch=2, delta=0, mis=None, impl=0):
    """hstu_attn_select_impl as the table has it."""
    from generative_recommenders_b200 import _lib

    pairs = (dqk, dv) in SQUARE + MIXED
    if dtype == _lib.E4M3:  # forward only, wgmma only, 16-element strides of q, k, v
        ok = pairs and not delta and not bias and mis not in READS[False] and mis != "q_stride"
        return _lib.IMPL_UMMA if not bwd and impl != _lib.IMPL_GENERIC and ok else HSTU_ERR_UNSUPPORTED
    if bwd and det and bias:  # the bias-table gradients are added with atomics
        return HSTU_ERR_UNSUPPORTED
    can = dtype in (_lib.BF16, _lib.F16) and pairs and not bias and mis not in READS[bwd]
    if bwd and det and (dqk == 256 or dqk != dv):  # the split kernels there have no deterministic route
        can = False
    if impl == _lib.IMPL_GENERIC:
        return _lib.IMPL_GENERIC
    if impl == _lib.IMPL_UMMA:
        return _lib.IMPL_UMMA if can else HSTU_ERR_UNSUPPORTED
    return _lib.IMPL_UMMA if can else _lib.IMPL_GENERIC


def _select_bidir(dtype, dqk, dv, bwd, det=0, bias=False, batch=2, delta=0, mis=None, impl=0):
    """hstu_attn_bidir_select_impl as the table has it: the non-causal wgmma kernels take bf16 / fp16 at dqk == dv in
    {32, 64, 128} without delta-q, and the wgmma views of the causal ones."""
    from generative_recommenders_b200 import _lib

    if delta or bias or dtype == _lib.E4M3:  # refused whatever impl asks
        return HSTU_ERR_UNSUPPORTED
    can = dtype in (_lib.BF16, _lib.F16) and dqk == dv and dqk in (32, 64, 128) and mis not in READS[bwd]
    if impl == _lib.IMPL_GENERIC:
        return _lib.IMPL_GENERIC
    if impl == _lib.IMPL_UMMA:
        return _lib.IMPL_UMMA if can else HSTU_ERR_UNSUPPORTED
    return _lib.IMPL_UMMA if can else _lib.IMPL_GENERIC


def _want(dtype, dqk, dv, bwd, **v):
    """(select_impl, workspace_bytes, fp16_operands_bytes, bwd_fp16_operands_workspace_bytes, bidir_select_impl,
    bidir_workspace_bytes)"""
    from generative_recommenders_b200 import _lib

    batch, delta, det = v.get("batch", 2), v.get("delta", 0), v.get("det", 0)
    amax = _align256(batch * H * 4 * 4)
    copy = _align256(ROWS * H * 32 * 2)  # one fp16 [L, H, 32] copy
    sel = _select(dtype, dqk, dv, bwd, **v)
    if sel != _lib.IMPL_UMMA:
        ws = 0
    elif dtype == _lib.E4M3:
        ws = _align256(ROWS * H * dv * 2)  # the fp16 copy of v
    elif delta:
        ws = 4 * batch * delta * H * dv * 4 if batch == 2 else 0  # the fp32 partials of 4 key chunks
    elif dtype == _lib.BF16 and dqk == dv == 32:
        ws = amax + (4 if bwd else 3) * copy  # the scaled fp16 copies of q, k, v (and dO)
    elif not bwd or dqk in (32, 256) or dqk != dv or det:
        ws = 0  # the split backward
    else:
        ws = ROWS * H * dqk * 4  # the fused backward's fp32 dQ accumulator
    fwd_sel = _select(dtype, dqk, dv, False, **v)
    kept = amax + 3 * copy if dtype == _lib.BF16 and dqk == dv == 32 and not delta and fwd_sel == _lib.IMPL_UMMA else 0
    bidir_sel = _select_bidir(dtype, dqk, dv, bwd, **v)
    # the non-causal backward is always split: its only workspace is the scaled fp16 operands of bf16 at d = 32
    bidir_ws = amax + (4 if bwd else 3) * copy if bidir_sel == _lib.IMPL_UMMA and dtype == _lib.BF16 and dqk == 32 else 0
    return sel, ws, kept, amax + copy, bidir_sel, bidir_ws


def _dtypes():
    from generative_recommenders_b200 import _lib

    return {"bf16": _lib.BF16, "fp16": _lib.F16, "e4m3": _lib.E4M3, "fp32": _lib.F32}


@pytest.fixture(scope="module")
def lib():
    from generative_recommenders_b200 import _lib
    from generative_recommenders_b200.build import build

    build()
    return _lib.lib()


@pytest.mark.parametrize("dtype,dqk,dv", [(t, *d) for t in ("bf16", "fp16", "e4m3") for d in SQUARE + MIXED + REFUSED]
                         + [("fp32", 32, 32), ("fp32", 64, 64)])
def test_attention_routing_table(lib, dtype, dqk, dv):
    from generative_recommenders_b200 import _lib

    assert torch.cuda.get_device_capability() == (9, 0)
    code = _dtypes()[dtype]
    n = 0
    for bwd in (False, True):
        for v in _variants(bwd):
            for impl in (_lib.IMPL_AUTO, _lib.IMPL_GENERIC, _lib.IMPL_UMMA):
                p = C.byref(_case(code, dqk, dv, bwd, impl=impl, **v))
                got = (lib.hstu_attn_select_impl(p, int(bwd)), lib.hstu_attn_workspace_bytes(p, int(bwd)),
                       lib.hstu_attn_fp16_operands_bytes(p), lib.hstu_attn_bwd_fp16_operands_workspace_bytes(p),
                       lib.hstu_attn_bidir_select_impl(p, int(bwd)), lib.hstu_attn_bidir_workspace_bytes(p, int(bwd)))
                assert got == _want(code, dqk, dv, bwd, impl=impl, **v), (dtype, dqk, dv, "bwd" if bwd else "fwd", impl, v)
                n += 1
    assert n == 3 * (15 + 13)
