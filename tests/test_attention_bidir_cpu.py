"""CPU: the non-causal (causal=False) attention where no GPU is needed.

- The library's mask (hstu_mask_valid_bidir) is the eager reference's causal=False mask (tests/bidir_oracle.py).
- Its key / query ranges cover that mask at tiles of 32, 64 and 128 rows, and are exactly [0, len) without a window.
- The test oracle matches the goldens made by the unmodified reference's pytorch_hstu_mha(causal=False).
- The new d = 32 wgmma kernels keep the register budget of the causal ones: <= 128 registers, no spills, tanh stages
  without per-score branches (scripts/sass_report.py).
- The Python layer refuses what the non-causal path does not take before it touches a device.
"""
import ctypes as C
import glob
import importlib.util
import os

import numpy as np
import pytest
import torch

from bidir_oracle import attn_valid_mask_bidir, hstu_mha_bwd_bidir, hstu_mha_fwd_bidir
from conftest import GOLDEN, ROOT, golden
from oracle import hstu_oracle as O
from test_abi_cpu import CASES

F32_TOL = 2e-6
# lengths around the 64- and 128-row tiles, with targets, a window and a contextual prefix
TILE_CASES = CASES + [(63, 3, 0, 0, 0), (64, -1, 0, 0, 0), (65, 2, 0, 0, 4), (127, 9, 20, 0, 0), (128, 1, 7, 16, 2),
                      (129, 5, 0, 0, 0), (191, 64, 30, 0, 0), (256, 130, 0, 0, 0), (257, 0, 64, 0, 70)]


@pytest.fixture(scope="module")
def lib():
    from generative_recommenders_b200 import _lib
    from generative_recommenders_b200.build import build

    build()
    return _lib.lib()


def _ref(case):
    n, nt, win, mf, ctx = case
    return attn_valid_mask_bidir(n, None if nt < 0 else nt, win, ctx, mf)


@pytest.mark.parametrize("case", TILE_CASES)
def test_mask_matches_the_eager_reference(lib, case):
    n, nt, win, mf, ctx = case
    ref = _ref(case)
    got = np.array([[lib.hstu_mask_valid_bidir(n, nt, win, mf, ctx, i, j) for j in range(n)] for i in range(n)], dtype=bool)
    assert np.array_equal(got, ref)


def test_mask_semantics():
    """History rows see the target keys; a target row sees every history key and of the targets only its own key."""
    n, nt = 12, 3
    m = attn_valid_mask_bidir(n, nt)
    hist, tgt = slice(0, n - nt), slice(n - nt, n)
    assert m[hist, tgt].all() and m[tgt, hist].all() and m[hist, hist].all()
    assert np.array_equal(m[tgt, tgt], np.eye(nt, dtype=bool))
    # the causal mask is the lower triangle of the same rule
    causal = O.attn_valid_mask(n, nt)
    assert not (causal & ~m).any()
    # a window bounds |id_i - id_j| on both sides
    w = attn_valid_mask_bidir(20, None, max_attn_len=3)
    i, j = np.indices(w.shape)
    assert np.array_equal(w, np.abs(i - j) <= 3)


@pytest.mark.parametrize("case", TILE_CASES)
@pytest.mark.parametrize("tile", [32, 64, 128])
def test_tile_ranges_cover_the_mask(lib, case, tile):
    n, nt, win, mf, ctx = case
    ref = _ref(case)
    lo, hi, chi = C.c_int32(), C.c_int32(), C.c_int32()
    for m0 in range(0, n, tile):
        m1 = min(n, m0 + tile)
        assert lib.hstu_kv_range_for_q_rows_bidir(n, nt, win, mf, ctx, m0, m1, C.byref(lo), C.byref(hi)) == 0
        cols = np.nonzero(ref[m0:m1].any(axis=0))[0]
        assert cols.min() >= lo.value and cols.max() < hi.value, (case, m0, lo.value, hi.value, cols.min(), cols.max())
        if win == 0:
            assert (lo.value, hi.value) == (0, n)
        assert lib.hstu_q_range_for_kv_rows_bidir(n, nt, win, mf, ctx, m0, m1, C.byref(lo), C.byref(hi), C.byref(chi)) == 0
        rows = np.nonzero(ref[:, m0:m1].any(axis=1))[0]
        for r in rows:
            assert (lo.value <= r < hi.value) or r < chi.value, (case, m0, r, lo.value, hi.value, chi.value)
        if win == 0:
            assert (lo.value, hi.value, chi.value) == (0, n, 0)


def test_window_ranges_skip_tiles(lib):
    """With a window the ranges are bounded on both sides, so the kernels skip the tiles outside them."""
    lo, hi, chi = C.c_int32(), C.c_int32(), C.c_int32()
    assert lib.hstu_kv_range_for_q_rows_bidir(1024, -1, 100, 0, 0, 512, 576, C.byref(lo), C.byref(hi)) == 0
    assert (lo.value, hi.value) == (412, 676)
    assert lib.hstu_q_range_for_kv_rows_bidir(1024, -1, 100, 0, 0, 512, 640, C.byref(lo), C.byref(hi), C.byref(chi)) == 0
    assert (lo.value, hi.value, chi.value) == (412, 740, 0)


def _bidir_files():
    return sorted(os.path.basename(p) for p in glob.glob(os.path.join(GOLDEN, "bidir_attn_*.pt")))


def test_bidir_goldens_exist():
    assert len(_bidir_files()) >= 5


@pytest.mark.parametrize("fname", _bidir_files())
def test_oracle_matches_the_reference_goldens(fname):
    g = golden(fname)
    kw = dict(num_targets=g["num_targets"], max_attn_len=g["max_attn_len"], contextual_seq_len=g["contextual_seq_len"],
              min_full_attn_seq_len=g["min_full_attn_seq_len"])
    out = hstu_mha_fwd_bidir(g["max_seq_len"], g["alpha"], g["q"], g["k"], g["v"], g["seq_offsets"], **kw)
    dq, dk, dv = hstu_mha_bwd_bidir(g["max_seq_len"], g["alpha"], g["dout"], g["q"], g["k"], g["v"], g["seq_offsets"], **kw)
    ref = g["ref_f32"]
    for name, a in (("out", out), ("dq", dq), ("dk", dk), ("dv", dv)):
        assert O.rel_l2(a, ref[name]) <= F32_TOL, (fname, name, O.rel_l2(a, ref[name]))
    # and they are not the causal answer
    causal = O.hstu_mha_fwd(g["max_seq_len"], g["alpha"], g["q"], g["k"], g["v"], g["seq_offsets"], dtype=torch.float64, **kw)
    assert O.rel_l2(causal, ref["out"]) > 0.1


def test_oracle_matches_the_causal_oracle_on_a_symmetric_problem():
    """With q == k the scores are symmetric, so the non-causal output is the causal one plus the strictly upper triangle."""
    torch.manual_seed(3)
    off = torch.tensor([0, 7, 20])
    q = torch.randn(20, 1, 8, dtype=torch.float64)
    v = torch.randn(20, 1, 8, dtype=torch.float64)
    full = hstu_mha_fwd_bidir(20, 0.5, q, q, v, off)
    causal = O.hstu_mha_fwd(20, 0.5, q, q, v, off, dtype=torch.float64)
    for s, e in ((0, 7), (7, 20)):
        S = torch.nn.functional.silu(0.5 * q[s:e, 0] @ q[s:e, 0].T) / 20
        upper = torch.triu(S, 1) @ v[s:e, 0]
        torch.testing.assert_close(full[s:e, 0], causal[s:e, 0] + upper)


_spec = importlib.util.spec_from_file_location("sass_report", os.path.join(ROOT, "scripts", "sass_report.py"))
sass_report = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(sass_report)

D32_BIDIR = ("attn_fwd_bidir_wgmma_kernel<(int)32,", "attn_bwd_dkdv_bidir_wgmma_kernel<(int)32,",
             "attn_bwd_dq_bidir_wgmma_kernel<(int)32,")


@pytest.fixture(scope="module")
def report():
    if sass_report.tools() is None:
        pytest.skip("nvcc / cuobjdump not installed")
    return sass_report.report("bidir_wgmma_kernel")


@pytest.mark.parametrize("kernel", D32_BIDIR)
def test_d32_bidir_kernels_keep_the_causal_budget(report, kernel):
    found = [r for name, r in report.items() if kernel in name]
    assert len(found) == 1, (kernel, sorted(report))
    r = found[0]
    assert r["registers"] <= 128, r
    assert r["spill_stores"] == 0 and r["spill_loads"] == 0, r
    assert r["tanh_per_block"] >= 8, r
    assert not set(r["notes"]) & {"C7510", "C7512", "C7515"}, r


def test_every_bidir_wgmma_kernel_is_spill_free(report):
    """d = 32 / 64 / 128, bf16 and fp16 (no bf16 kernel at d = 32: it runs on scaled fp16 operands)."""
    names = sorted(report)
    assert len(names) == 15, names
    for name in names:
        assert report[name]["spill_stores"] == 0 and report[name]["spill_loads"] == 0, (name, report[name])


def test_host_layer_refuses_what_the_non_causal_path_does_not_take():
    from generative_recommenders_b200.ops.hstu_attention import cuda_hstu_attention_bwd, cuda_hstu_attention_fwd

    q = torch.zeros(4, 1, 32)
    off = torch.tensor([0, 4])
    with pytest.raises(RuntimeError, match="delta_q"):
        cuda_hstu_attention_fwd(8, 0.25, q, q, q, off, delta_q_len=2, causal=False)
    with pytest.raises(RuntimeError, match="fp8"):
        f8 = q.to(torch.float8_e4m3fn)
        cuda_hstu_attention_fwd(8, 0.25, f8, f8, f8, off, causal=False)
    with pytest.raises(RuntimeError, match="relative bias"):
        cuda_hstu_attention_fwd(8, 0.25, q, q, q, off, bias=(torch.zeros(15), None, None), causal=False)
    with pytest.raises(RuntimeError, match="relative bias"):
        cuda_hstu_attention_bwd(8, 0.25, q, q, q, q, q, q, q, off, bias=(torch.zeros(15), None, None), causal=False)


def test_c_abi_refusals_and_routing(lib):
    """No device is needed to route: delta-q, a relative bias and e4m3 are refused; fp32, d = 256 and dqk != dv take the
    generic kernels, and forcing the wgmma kernels on them is refused."""
    from generative_recommenders_b200 import _lib

    def params(**kw):
        p = _lib.AttnParams()
        p.abi_version, p.dtype, p.batch, p.heads, p.dqk, p.dv, p.max_seq_len, p.total_rows = 1, _lib.BF16, 2, 2, 32, 32, 64, 0
        for k, v in kw.items():
            setattr(p, k, v)
        return p

    for kw, what in ((dict(delta_q_len=4), b"delta_q"), (dict(pos_w=16), b"relative bias"), (dict(dtype=_lib.E4M3), b"fp8")):
        for bwd in (0, 1):
            if bwd and "delta_q_len" in kw:
                continue  # a backward of delta-q is refused by the argument checks already
            assert lib.hstu_attn_bidir_select_impl(C.byref(params(**kw)), bwd) == -2
            assert what in lib.hstu_last_error()
    for kw in (dict(dtype=_lib.F32), dict(dqk=256, dv=256), dict(dqk=32, dv=64), dict(dqk=48, dv=48)):
        assert lib.hstu_attn_bidir_select_impl(C.byref(params(**kw)), 0) == _lib.IMPL_GENERIC
        assert lib.hstu_attn_bidir_select_impl(C.byref(params(impl=_lib.IMPL_UMMA, **kw)), 0) == -2
        assert b"generic" in lib.hstu_last_error()
    assert lib.hstu_attn_bidir_workspace_bytes(C.byref(params()), 1) == 0  # empty problem


DEVICE_PTR = b"expected a CUDA device pointer"
# (case, backward, expected return of hstu_attn_{fwd|bwd}, hstu_attn_{fwd|bwd}_bidir, hstu_attn_select_impl,
# hstu_attn_bidir_select_impl, hstu_attn_workspace_bytes, hstu_attn_bidir_workspace_bytes); a refusal is (code, message part).
# The entries differ where the table says so: the causal ones refuse e4m3 themselves, return 0 on an empty problem and bind
# the device of q before routing; the non-causal ones route first.
ENTRY_TABLE = [
    (dict(rows=0), False, 0, 0, 1, 1, 0, 0),
    (dict(rows=0), True, 0, 0, 1, 1, 0, 0),
    (dict(rows=0, dtype="e4m3"), False, (-1, b"go through hstu_attn_fwd_fp8"), (-2, b"fp8 (e4m3) inputs are not supported"),
     (-2, b"the generic kernels take no fp8 input"), (-2, b"fp8 (e4m3) inputs are not supported"), 0, 0),
    (dict(rows=0, dtype="e4m3"), True, (-2, b"hstu_attn_bwd: fp8 (e4m3) attention has no backward"),
     (-2, b"fp8 (e4m3) inputs are not supported"), (-2, b"fp8 (e4m3) attention has no backward: hstu_attn_fwd_fp8"),
     (-2, b"fp8 (e4m3) inputs are not supported"), 0, 0),
    (dict(rows=0, delta=4), False, 0, (-2, b"delta_q (the KV-cached forward) is causal only"), 1,
     (-2, b"delta_q (the KV-cached forward) is causal only"), 0, 0),
    (dict(rows=0, bias=True), True, 0, (-2, b"the relative bias is not supported"),
     (-2, b"deterministic backward with a relative bias"), (-2, b"the relative bias is not supported"), 0, 0),
    (dict(dqk=48, impl=2), False, (-1, DEVICE_PTR), (-2, b"it takes bf16 / fp16 at dqk == dv in {32, 64, 128}"),
     (-2, b"delta=0 bias=0"), (-2, b"non-causal wgmma path does not support this problem (dtype=1 dqk=48 dv=48)"), 0, 0),
    (dict(dqk=48, impl=2), True, (-1, DEVICE_PTR), (-2, b"non-causal wgmma path"), (-2, b"delta=0 bias=0"),
     (-2, b"non-causal wgmma path"), 0, 0),
    (dict(), True, (-1, DEVICE_PTR), (-1, DEVICE_PTR), 1, 1, 0, 0),
    (dict(dtype="e4m3", impl=0), False, (-1, b"go through hstu_attn_fwd_fp8"), (-2, b"fp8 (e4m3) inputs are not supported"),
     2, (-2, b"fp8 (e4m3) inputs are not supported"), 4096 * 2 * 32 * 2, 0),
    (dict(delta=4), True, *[(-1, b"backward of delta-q attention is not defined")] * 4, 0, 0),
    (None, False, *[(-1, b"params is NULL")] * 4, 0, 0),
]


@pytest.mark.parametrize("case,bwd,want", [(c, b, tuple(w)) for c, b, *w in ENTRY_TABLE])
def test_c_abi_attention_entries_at_both_masks(lib, case, bwd, want):
    """Return code and message of every attention entry, causal and non-causal, for refused and empty problems, with
    placeholder pointers: nothing here needs a device.  Problems the argument checks pass reach the device binding of the
    run entries, which refuses a placeholder q on any machine.  Default impl: generic, which routes without a device query."""
    from generative_recommenders_b200 import _lib
    from test_attention_deterministic_cpu import _params

    p = None
    if case is not None:
        kw = dict(case)
        dtype = {"bf16": _lib.BF16, "e4m3": _lib.E4M3}[kw.pop("dtype", "bf16")]
        dqk = kw.pop("dqk", 32)
        p = _params(dtype, dqk, deterministic=1, impl=kw.pop("impl", _lib.IMPL_GENERIC), rows=kw.pop("rows", 4096),
                    bias=kw.pop("bias", False))
        p.delta_q_len = kw.pop("delta", 0)
        assert not kw, kw
        p = C.byref(p)
    d = "bwd" if bwd else "fwd"
    calls = ((f"hstu_attn_{d}", None), (f"hstu_attn_{d}_bidir", None), ("hstu_attn_select_impl", int(bwd)),
             ("hstu_attn_bidir_select_impl", int(bwd)), ("hstu_attn_workspace_bytes", int(bwd)),
             ("hstu_attn_bidir_workspace_bytes", int(bwd)))
    for (name, arg), w in zip(calls, want):
        rc = getattr(lib, name)(p, arg)
        if isinstance(w, tuple):
            assert (rc, w[1] in lib.hstu_last_error()) == (w[0], True), (name, rc, lib.hstu_last_error(), w)
        else:
            assert rc == w, (name, rc, lib.hstu_last_error(), w)
