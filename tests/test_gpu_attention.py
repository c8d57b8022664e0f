"""GPU parity of the jagged HSTU attention (through the C-ABI) against the golden vectors of the reference eager
path and against the CPU oracle on seeded inputs that follow the reference's own test recipe
(ops/tests/hstu_attention_test.py:35-163,256-290)."""
import glob
import itertools
import os
import random

import pytest
import torch

from conftest import GOLDEN, golden
from oracle import hstu_oracle as O
from util import assert_rel, offsets_from

pytestmark = pytest.mark.gpu


def _mods():
    from generative_recommenders_b200 import _lib
    from generative_recommenders_b200.common import HammerKernel
    from generative_recommenders_b200.ops.hstu_attention import delta_hstu_mha, hstu_mha, hstu_rel_bias_attention

    return _lib, HammerKernel, hstu_mha, delta_hstu_mha, hstu_rel_bias_attention


def _run(g, impl, dtype=None):
    _lib, HK, hstu_mha, _, _ = _mods()
    dev = torch.device("cuda")
    dt = dtype or g["q"].dtype
    q, k, v = (g[n].to(dev, dt).requires_grad_() for n in ("q", "k", "v"))
    nt = None if g["num_targets"] is None else g["num_targets"].to(dev)
    out = hstu_mha(max_seq_len=g["max_seq_len"], alpha=g["alpha"], q=q, k=k, v=v, seq_offsets=g["seq_offsets"].to(dev),
                   num_targets=nt, max_attn_len=g["max_attn_len"], contextual_seq_len=g["contextual_seq_len"],
                   min_full_attn_seq_len=g["min_full_attn_seq_len"], kernel=HK.CUDA, impl=impl)
    out.backward(g["dout"].to(dev, dt))
    return out.detach(), q.grad, k.grad, v.grad


@pytest.mark.parametrize("fname", sorted(os.path.basename(p) for p in glob.glob(os.path.join(GOLDEN, "attn_*.pt"))))
def test_attention_golden(fname):
    _lib = _mods()[0]
    g = golden(fname)
    ref = g["ref_f32"]
    impls = [_lib.IMPL_GENERIC]
    if g["q"].dtype != torch.float32:
        impls.append(_lib.IMPL_AUTO)
    for impl in impls:
        out, dq, dk, dv = _run(g, impl)
        for name, a in (("out", out), ("dq", dq), ("dk", dk), ("dv", dv)):
            assert_rel(a, ref[name], f"{fname}:{name}:impl{impl}")
        # the reference's own criterion (hstu_attention_test.py:152-163): assert_close (default tolerances of the dtype)
        # of out, dv, dk, dq against the eager path evaluated in the native dtype
        nat = g["ref_native"]
        for name, a in (("out", out), ("dv", dv), ("dk", dk), ("dq", dq)):
            torch.testing.assert_close(a.cpu(), nat[name], msg=lambda m, n=name: f"{fname}:{n}:impl{impl}: {m}")


def _random_case(seed, dtype, B, H, max_uih, max_tgt, dqk, dv, targets, window, ctx, min_full=0, i32=False):
    g = torch.Generator().manual_seed(seed)
    lengths = torch.randint(max_uih + 1, (B,), generator=g)
    nt = torch.randint(1, max_tgt + 1, (B,), generator=g)
    lengths = lengths + nt + ctx
    N = max_uih + max_tgt + ctx
    off = offsets_from(lengths.tolist())
    L = int(off[-1])
    mk = lambda d: torch.empty(L, H, d).uniform_(-0.1, 0.1, generator=g).to(dtype)  # noqa: E731
    case = dict(max_seq_len=N, alpha=1.0 / dqk**0.5, q=mk(dqk), k=mk(dqk), v=mk(dv),
                dout=torch.randn(L, H, dv, generator=g).to(dtype), seq_offsets=off.to(torch.int32) if i32 else off,
                num_targets=(nt.to(torch.int32) if i32 else nt) if targets else None,
                max_attn_len=(random.Random(seed).randint(1, max(1, max_uih // 5)) if window else 0),
                contextual_seq_len=ctx, min_full_attn_seq_len=min_full)
    return case


def _check_vs_oracle(case, impl, tag):
    kw = dict(num_targets=case["num_targets"], max_attn_len=case["max_attn_len"],
              contextual_seq_len=case["contextual_seq_len"], min_full_attn_seq_len=case["min_full_attn_seq_len"])
    ref_out = O.hstu_mha_fwd(case["max_seq_len"], case["alpha"], case["q"], case["k"], case["v"], case["seq_offsets"], **kw)
    rdq, rdk, rdv = O.hstu_mha_bwd(case["max_seq_len"], case["alpha"], case["dout"], case["q"], case["k"], case["v"],
                                   case["seq_offsets"], **kw)
    out, dq, dk, dv = _run(case, impl)
    for name, a, r in (("out", out, ref_out), ("dq", dq, rdq), ("dk", dk, rdk), ("dv", dv, rdv)):
        assert_rel(a, r, f"{tag}:{name}")


def _selected(case, _lib):
    """Which implementation AUTO dispatches to for this case (forward)."""
    import ctypes as C

    from generative_recommenders_b200.ops.hstu_attention import _fill_common

    dev = torch.device("cuda")
    q, k, v = (case[n].to(dev) for n in ("q", "k", "v"))
    p = _lib.AttnParams()
    nt = None if case["num_targets"] is None else case["num_targets"].to(dev)
    _fill_common(p, case["max_seq_len"], case["alpha"], q, k, v, case["seq_offsets"].to(dev), nt, case["max_attn_len"],
                 case["contextual_seq_len"], case["min_full_attn_seq_len"], _lib.IMPL_AUTO)
    out = torch.empty(q.shape[0], q.shape[1], v.shape[2], device=dev, dtype=q.dtype)
    p.out = out.data_ptr()
    p.o_row_stride, p.o_head_stride = out.stride(0), out.stride(1)
    return _lib.lib().hstu_attn_select_impl(C.byref(p), 0)


GRID = list(itertools.product([torch.float32, torch.bfloat16], [(20, 20), (100, 20), (128, 512), (256, 20)],
                              [(16, 16), (32, 64), (64, 32), (128, 128)], [False, True], [False, True], [0, 10]))


@pytest.mark.parametrize("idx", range(0, len(GRID), 3))
def test_attention_random_grid_generic(idx):
    """Seeded sweep over the reference's hypothesis space (dtype, lengths, head dims, targets, window, contextual)."""
    _lib = _mods()[0]
    dtype, (uih, tgt), (dqk, dv), targets, window, ctx = GRID[idx]
    case = _random_case(1000 + idx, dtype, 4 + idx % 5, 1 + idx % 4, uih, tgt, dqk, dv, targets, window, ctx,
                        i32=bool(idx % 2))
    _check_vs_oracle(case, _lib.IMPL_GENERIC, f"grid{idx}")


@pytest.mark.parametrize("d", [32, 64, 128])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("opts", [(False, False, 0, 0), (True, False, 0, 0), (True, True, 0, 0), (True, True, 7, 0),
                                  (True, True, 5, 33), (False, False, 4, 0)])
def test_attention_umma_vs_oracle(d, dtype, opts):
    """wgmma/TMA forward (+ backward of whichever implementation AUTO selects) against the fp32 oracle."""
    _lib = _mods()[0]
    targets, window, ctx, min_full = opts
    case = _random_case(7000 + d + ctx, dtype, 5, 3, 300, 24, d, d, targets, window, ctx, min_full)
    assert _selected(case, _lib) == _lib.IMPL_UMMA
    _check_vs_oracle(case, _lib.IMPL_UMMA, f"umma-d{d}-{dtype}-{opts}")


def test_attention_strided_views_and_empty():
    """q/k/v as non-contiguous views of one buffer (hstu_attention_bench.py:228-233), empty sequences, L == 0."""
    _lib, HK, hstu_mha, _, _ = _mods()
    dev = torch.device("cuda")
    torch.manual_seed(5)
    lengths = [0, 130, 0, 257, 1, 128]
    off = offsets_from(lengths, dev)
    L, H, d = sum(lengths), 2, 64
    x = torch.empty(L, H, 3 * d, device=dev, dtype=torch.bfloat16).uniform_(-0.1, 0.1)
    q, k, v = torch.split(x, [d, d, d], dim=-1)
    for impl in (_lib.IMPL_GENERIC, _lib.IMPL_AUTO):
        out = hstu_mha(300, 1.0 / d, q, k, v, off, kernel=HK.CUDA, impl=impl)
        ref = O.hstu_mha_fwd(300, 1.0 / d, q.cpu(), k.cpu(), v.cpu(), off.cpu())
        assert_rel(out, ref, f"strided impl{impl}")
    e = torch.empty(0, H, d, device=dev, dtype=torch.bfloat16)
    out = hstu_mha(16, 0.1, e, e, e, torch.zeros(3, dtype=torch.int64, device=dev), kernel=HK.CUDA)
    assert out.shape == (0, H, d)


@pytest.mark.parametrize("d,dtype", [(32, torch.bfloat16), (64, torch.float16), (24, torch.float32)])
def test_rows_beyond_max_seq_len_are_ignored_and_zero(d, dtype):
    """A sequence longer than max_seq_len: the reference drops the rows >= N on the way in (jagged_to_padded_dense truncates)
    and returns zeros for them (pt_hstu_attention.py:97-167).  out / dq / dk / dv of those rows must be written as zeros, not
    left as uninitialised memory (they flow into the weight-gradient GEMMs of the fused block)."""
    _lib, HK, hstu_mha, _, _ = _mods()
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(31)
    lengths, N, H = [300, 77, 260, 256], 256, 2
    off = offsets_from(lengths)
    L = int(off[-1])
    q, k, v = (torch.empty(L, H, d).uniform_(-0.3, 0.3, generator=g).to(dtype) for _ in range(3))
    do = torch.randn(L, H, d, generator=g).to(dtype)
    nt = torch.tensor([4, 2, 0, 9])
    ref = O.hstu_mha_fwd(N, 0.2, q, k, v, off, nt)
    rdq, rdk, rdv = O.hstu_mha_bwd(N, 0.2, do, q, k, v, off, nt)
    tail = torch.cat([torch.arange(int(off[i]) + N, int(off[i + 1])) for i in range(len(lengths)) if lengths[i] > N])
    assert float(ref[tail].abs().max()) == 0.0
    impls = [_lib.IMPL_GENERIC] + ([_lib.IMPL_UMMA] if dtype != torch.float32 else [])
    for impl in impls:
        junk = torch.full((8 * L * H * d,), float("nan"), device=dev, dtype=dtype)  # poison what the allocator hands out next
        del junk
        qd, kd, vd = (t.to(dev).requires_grad_() for t in (q, k, v))
        out = hstu_mha(N, 0.2, qd, kd, vd, off.to(dev), num_targets=nt.to(dev), kernel=HK.CUDA, impl=impl)
        out.backward(do.to(dev))
        for name, a, r in (("out", out, ref), ("dq", qd.grad, rdq), ("dk", kd.grad, rdk), ("dv", vd.grad, rdv)):
            assert torch.isfinite(a).all(), f"{name} impl {impl}: non-finite rows"
            assert float(a[tail.to(dev)].abs().max()) == 0.0, f"{name} impl {impl}: rows >= max_seq_len are not zero"
            assert_rel(a, r, f"len > N: {name} impl {impl}")


@pytest.mark.parametrize("fname", ["delta_plain.pt", "delta_ctx.pt"])
def test_delta_attention_golden(fname):
    _lib, HK, _, delta_hstu_mha, _ = _mods()
    g = golden(fname)
    dev = torch.device("cuda")
    out = delta_hstu_mha(max_seq_len=g["max_seq_len"], alpha=g["alpha"], delta_q=g["delta_q"].to(dev), k=g["k"].to(dev),
                         v=g["v"].to(dev), seq_offsets=g["seq_offsets"].to(dev), num_targets=g["num_targets"].to(dev),
                         max_attn_len=g["max_attn_len"], contextual_seq_len=g["contextual_seq_len"], kernel=HK.CUDA)
    assert_rel(out, g["out"], fname)


def test_research_rel_bias_attention_golden():
    _lib, HK, _, _, rel_attn = _mods()
    g = golden("research_attn.pt")
    dev = torch.device("cuda")
    H, dqk, dv = g["H"], g["dqk"], g["dv"]
    q = g["q"].view(-1, H, dqk).to(dev).requires_grad_()
    k = g["k"].view(-1, H, dqk).to(dev).requires_grad_()
    v = g["v"].view(-1, H, dv).to(dev).requires_grad_()
    pos_w = g["pos_w"].to(dev).requires_grad_()
    ts_w = g["ts_w"].to(dev).requires_grad_()
    out = rel_attn(g["n"], q, k, v, g["seq_offsets"].to(dev), pos_w, ts_w, g["timestamps"].to(dev))
    out.backward(g["dout"].view(-1, H, dv).to(dev))
    assert_rel(out.reshape(-1, H * dv), g["out"], "research out")
    assert_rel(q.grad.reshape(-1, H * dqk), g["dq"], "research dq")
    assert_rel(k.grad.reshape(-1, H * dqk), g["dk"], "research dk")
    assert_rel(v.grad.reshape(-1, H * dv), g["dv_"], "research dv")
    assert_rel(pos_w.grad, g["dpos_w"], "research dpos_w", tol=1e-4)
    assert_rel(ts_w.grad, g["dts_w"], "research dts_w", tol=1e-4)


def test_target_invariance_metamorphic():
    """Swapping two target rows of the inputs permutes the outputs identically (modules/tests/stu_test.py:174-325):
    targets attend to the history and to themselves, never to each other."""
    _lib, HK, hstu_mha, _, _ = _mods()
    dev = torch.device("cuda")
    torch.manual_seed(11)
    lengths, nts = [150, 200], [6, 9]
    off = offsets_from(lengths, dev)
    H, d = 2, 32
    L = sum(lengths)
    q, k, v = (torch.empty(L, H, d, device=dev, dtype=torch.bfloat16).uniform_(-0.3, 0.3) for _ in range(3))
    nt = torch.tensor(nts, device=dev)
    perm = torch.arange(L, device=dev)
    a, bb = lengths[0] - 2, lengths[0] - 5  # two target rows of sequence 0
    perm[a], perm[bb] = bb, a
    for impl in (_lib.IMPL_GENERIC, _lib.IMPL_AUTO):
        o1 = hstu_mha(256, 0.2, q, k, v, off, num_targets=nt, kernel=HK.CUDA, impl=impl)
        o2 = hstu_mha(256, 0.2, q[perm], k[perm], v[perm], off, num_targets=nt, kernel=HK.CUDA, impl=impl)
        assert_rel(o2, o1[perm].float(), f"target invariance impl {impl}", tol=2e-3)
