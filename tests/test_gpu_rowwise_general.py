"""The general row-wise kernels of csrc/norm.cu against the fp64 oracle, through the cuda_* entry points, at the shapes and layouts
that reach each of their specialisations: 16-bit and fp32 elements, the vector (16-byte) and scalar (VEC = 1) paths -- the
latter taken by odd lengths, misaligned pointers and row strides that are not a multiple of the vector -- the per-lane
capacities PL = 8 / 16 / 32, LayerNorm / SwishLayerNorm / RMSNorm, the output stage with layer or group norm, three concat modes
and silu(u), dropout, more rows than the grid (so every warp loops and the backward's register accumulators take several rows),
and SiLU on the strided u columns of uvqk.  Length-256 16-bit layer norms belong to the fast kernels (test_gpu_norm_fast.py)
and are left out.  Inputs are rounded to the kernel's dtype first; the oracle runs in fp64 on those values.
"""
import pytest
import torch

from oracle import hstu_oracle as O
from util import TOL, _assert_ulp, assert_rel, assert_same_zeros

pytestmark = pytest.mark.gpu
DEV = "cuda"
DTYPES16 = [torch.bfloat16, torch.float16]
IDS = {torch.float32: "fp32", torch.bfloat16: "bf16", torch.float16: "fp16"}
EPS = 1e-6
F32 = TOL[torch.float32]  # statistics and parameter gradients are fp32 outputs: the fp32 bound


def _ops():
    from generative_recommenders_b200.ops import hstu_compute as hc
    from generative_recommenders_b200.ops import layer_norm as ln
    return hc, ln


def _place(t, layout):
    """t [n, D] on the GPU in one of three layouts: contiguous; a contiguous view at storage offset 1 (pointer misaligned, so
    the scalar path even when D % 8 == 0); rows of stride D + 3 (not a multiple of 8)."""
    n, D = t.shape
    if layout == "contig":
        return t.to(DEV).contiguous()
    if layout == "offset1":
        buf = torch.zeros(n * D + 1, dtype=t.dtype, device=DEV)
        v = buf[1:].view(n, D)
    else:
        v = torch.zeros(n, D + 3, dtype=t.dtype, device=DEV)[:, :D]
    v.copy_(t.to(DEV))
    return v


# ------------------------------------------------------------------------------------------------------------------
# LayerNorm / SwishLayerNorm / RMSNorm
# ------------------------------------------------------------------------------------------------------------------
def _norm_reference(kind, x, w, b, dy):
    x64, w64, b64 = (t.double().requires_grad_() for t in (x, w, b))
    if kind == "rms":
        rstd = torch.rsqrt(x64.detach().square().mean(-1) + EPS)
        y, mean = O.rms_norm_fwd(x64, w64, EPS, dtype=torch.float64), None
    else:
        _, mean, rstd = O.layer_norm_fwd(x64.detach(), w64.detach(), b64.detach(), EPS, dtype=torch.float64)
        f = O.swish_layer_norm_fwd if kind == "swish" else lambda *a, **k: O.layer_norm_fwd(*a, **k)[0]
        y = f(x64, w64, b64, EPS, dtype=torch.float64)
    y.backward(dy.double())
    return y.detach(), mean, rstd, x64.grad, w64.grad, b64.grad


def _norm_kernel(kind, x, w, b, dy):
    hc, ln = _ops()
    if kind != "rms":
        y, mean, rstd = ln.cuda_layer_norm_fwd(x, w, b, EPS, kind == "swish")
        dx, dw, db = ln.cuda_layer_norm_bwd(dy, x, w, b, mean, rstd, kind == "swish")
        return y, mean, rstd, dx, dw, db
    # RMSNorm has no cuda_* entry point of its own: its autograd function is the thin host layer over the C ABI
    xl, wl = x.detach().requires_grad_(), w.detach().float().requires_grad_()
    y = ln.rms_norm(xl, wl, EPS)
    y.backward(dy)
    return y, None, None, xl.grad, wl.grad, None


def _norm_case(kind, dtype, D, rows, layout, seed):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(rows, D, generator=g) * 1.7 + 0.3).to(dtype)
    w = (1 + 0.5 * torch.randn(D, generator=g)).to(dtype)  # far from ones: a backward that drops w cannot pass
    b = (0.2 * torch.randn(D, generator=g)).to(dtype)
    dy = torch.randn(rows, D, generator=g).to(dtype)
    got = _norm_kernel(kind, _place(x, layout), w.to(DEV), b.to(DEV), _place(dy, layout))
    ref = _norm_reference(kind, x, w, b, dy)
    y, mean, rstd, dx, dw, db = got
    assert_rel(y, ref[0], f"{kind} y")
    if mean is not None:
        assert_rel(mean, ref[1], f"{kind} mean", tol=F32)
        assert_rel(rstd, ref[2], f"{kind} rstd", tol=F32)
    assert_rel(dx, ref[3], f"{kind} dx")
    assert_rel(dw, ref[4], f"{kind} dw", tol=F32)
    if db is not None:
        assert_rel(db, ref[5], f"{kind} db", tol=F32)


@pytest.mark.parametrize("rows", [1, 4300, 17000])  # 4300 > 528 x 8: the backward loops; 17000 > 2112 x 8: so does the forward
@pytest.mark.parametrize("D", [50, 64, 200, 384, 1000, 1024])
@pytest.mark.parametrize("kind", ["ln", "swish", "rms"])
@pytest.mark.parametrize("dtype", DTYPES16, ids=IDS.get)
def test_norm_general(dtype, kind, D, rows):
    _norm_case(kind, dtype, D, rows, "contig", seed=D * 7 + rows)


# the RMSNorm C ABI takes dense rows: no strided case for it
@pytest.mark.parametrize("kind,layout", [("ln", "offset1"), ("ln", "stride"), ("swish", "offset1"), ("swish", "stride"),
                                         ("rms", "offset1")])
@pytest.mark.parametrize("D", [64, 200, 384, 1024])
@pytest.mark.parametrize("dtype", DTYPES16, ids=IDS.get)
def test_norm_general_scalar_layouts(dtype, D, kind, layout):
    _norm_case(kind, dtype, D, 4300, layout, seed=D * 11 + len(layout))


# ------------------------------------------------------------------------------------------------------------------
# output stage  y = u' * Norm(attn)  [+ concat], u' = silu(u) or u
# ------------------------------------------------------------------------------------------------------------------
def _nmd_reference(attn, u, w, b, dout, silu_u, concat, gn, H, dv):
    a64, u64, w64, b64 = (t.double().requires_grad_() for t in (attn, u, w, b))
    uf = torch.nn.functional.silu(u64) if silu_u else u64
    if gn:
        ah = a64.view(-1, H, dv)
        m = ah.mean(-1, keepdim=True)
        nrm = ((ah - m) * torch.rsqrt((ah - m).square().mean(-1, keepdim=True) + EPS) * w64.view(1, H, 1)
               + b64.view(1, H, 1)).reshape(-1, H * dv)
    else:
        nrm = O.layer_norm_fwd(a64, w64, b64, EPS, dtype=torch.float64)[0]
    y = uf * nrm
    if concat == 1:
        y = torch.cat([uf, a64, y], dim=1)   # concat_ux (pt_hstu_linear.py:57-58)
    elif concat == 2:
        y = torch.cat([uf, nrm, y], dim=1)   # concat_ua of the research block (hstu.py:427-437)
    y.backward(dout.double())
    return y.detach(), a64.grad, u64.grad, w64.grad, b64.grad


def _columns(t, W):
    """attn / u as column views of one wider buffer (row stride 2 W + 24, both starting at a 16-byte boundary)."""
    n = t[0].shape[0]
    buf = torch.zeros(n, 2 * W + 24, dtype=t[0].dtype, device=DEV)
    a, u = buf[:, 8:8 + W], buf[:, W + 16:2 * W + 16]
    a.copy_(t[0].to(DEV))
    u.copy_(t[1].to(DEV))
    return a, u


def _nmd_case(dtype, H, dv, gn, concat, silu_u, seed):
    hc, _ = _ops()
    g = torch.Generator().manual_seed(seed)
    W = H * dv
    G = H if gn else 1
    # more than 528 x 8 vectors: every backward warp loops.  At the two widest rows the fp64 oracle of that many rows costs
    # seconds per case, so only bf16 (the benchmarked dtype; the loop is the same code for every dtype) runs them
    n = 4300 // G + 13 if W < 512 or dtype == torch.bfloat16 else 1100
    np_ = H if gn else W
    attn = (torch.randn(n, W, generator=g) * 0.8 + 0.1).to(dtype)
    u = torch.randn(n, W, generator=g).to(dtype)
    w = (1 + 0.5 * torch.randn(np_, generator=g)).to(dtype)
    b = (0.2 * torch.randn(np_, generator=g)).to(dtype)
    dout = torch.randn(n, W * (3 if concat else 1), generator=g).to(dtype)
    a_d, u_d = _columns((attn, u), W)
    out, mean, rstd = hc.cuda_norm_mul_dropout_fwd(a_d, u_d, w.to(DEV), b.to(DEV), EPS, 0.0, 0, silu_u, concat, gn, H, dv)
    dattn, du, dw, db = hc.cuda_norm_mul_dropout_bwd(dout.to(DEV), a_d, u_d, w.to(DEV), b.to(DEV), mean, rstd, 0.0, 0, silu_u,
                                                     concat, gn, H, dv)
    ref = _nmd_reference(attn, u, w, b, dout, silu_u, concat, gn, H, dv)
    assert_rel(out, ref[0], "out")
    assert_rel(dattn, ref[1], "dattn")
    assert_rel(du, ref[2], "du")
    assert dw.shape == db.shape == (np_,)
    assert_rel(dw, ref[3], "dw", tol=F32)
    assert_rel(db, ref[4], "db", tol=F32)


@pytest.mark.parametrize("silu_u", [False, True])
@pytest.mark.parametrize("concat", [0, 1, 2])
@pytest.mark.parametrize("H,dv", [(8, 8), (8, 12), (8, 64), (8, 128)])  # H dv = 64 (amzn_books), 96, 512, 1024
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32], ids=IDS.get)
def test_output_stage_layer_norm(dtype, H, dv, concat, silu_u):
    _nmd_case(dtype, H, dv, False, concat, silu_u, seed=H * dv + 10 * concat + int(silu_u))


@pytest.mark.parametrize("silu_u", [False, True])
@pytest.mark.parametrize("concat", [0, 1, 2])
@pytest.mark.parametrize("dv", [8, 12, 32, 128])  # dv = 12 takes the scalar path
@pytest.mark.parametrize("H", [2, 8])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32], ids=IDS.get)
def test_output_stage_group_norm(dtype, H, dv, concat, silu_u):
    _nmd_case(dtype, H, dv, True, concat, silu_u, seed=1000 + H * dv + 10 * concat + int(silu_u))


# ------------------------------------------------------------------------------------------------------------------
# dropout on the general kernels
# ------------------------------------------------------------------------------------------------------------------
def _positive_inputs(n, W, dtype, seed):
    """attn, u, and LN parameters for which u * Norm(attn) is bounded away from zero: a zero output is a dropped one."""
    g = torch.Generator().manual_seed(seed)
    attn = (torch.randn(n, W, generator=g) + 3.0).to(dtype).to(DEV)
    u = (torch.rand(n, W, generator=g) + 0.5).to(dtype).to(DEV)
    return attn, u


def _misaligned(t):
    buf = torch.zeros(t.numel() + 1, dtype=t.dtype, device=DEV)
    v = buf[1:].view(t.shape)
    v.copy_(t)
    return v


@pytest.mark.parametrize("p", [0.2, 0.5])
@pytest.mark.parametrize("concat", [0, 1])
@pytest.mark.parametrize("dtype", DTYPES16, ids=IDS.get)
def test_dropout_vector_and_scalar_paths_agree(dtype, concat, p):
    """amzn_books' output stage (H dv = 64): the aligned tensors take the vector path, a misaligned copy of them the scalar one
    (dropout_keep per element); the masks depend only on (seed, flat index), so both zero patterns must be identical, the
    keep rate must be 1 - p, and the backward must zero exactly the gradient elements that the forward dropped."""
    hc, _ = _ops()
    n, H, dv, seed = 4400, 8, 8, 1234567 + concat
    W = H * dv
    attn, u = _positive_inputs(n, W, dtype, seed=int(p * 10) + concat)
    w = torch.ones(W, device=DEV, dtype=dtype)
    b = torch.full((W,), 4.0, device=DEV, dtype=dtype)  # LN(attn) + 4 > 0
    out_v, mean, rstd = hc.cuda_norm_mul_dropout_fwd(attn, u, w, b, EPS, p, seed, False, concat, False, H, dv)
    am, um = _misaligned(attn), _misaligned(u)
    out_s, _, _ = hc.cuda_norm_mul_dropout_fwd(am, um, _misaligned(w), _misaligned(b), EPS, p, seed, False, concat, False, H, dv)
    assert_same_zeros(out_v, out_s, "vector vs scalar dropout path")
    keep = (out_v != 0).float().mean().item()
    assert abs(keep - (1 - p)) < 0.01, keep
    dout = torch.ones_like(out_v)
    for a_, u_, what in ((attn, u, "vector"), (am, um, "scalar")):
        _, du, _, _ = hc.cuda_norm_mul_dropout_bwd(dout, a_, u_, w, b, mean, rstd, p, seed, False, concat, False, H, dv)
        if concat:  # du = dropout(dout_u) + dropout(dout_y) * LN(attn): zero iff both parts were dropped
            dropped = (out_v[:, :W] == 0) & (out_v[:, 2 * W:] == 0)
        else:
            dropped = out_v == 0
        assert torch.equal(du == 0, dropped), f"{what} backward: the zeroed du elements are not the dropped ones"


def test_dropout_group_norm_scalar_path_matches_layer_norm_view():
    """Group norm at dv = 12 (scalar path) and a layer-norm view of the same [n, 96] tensors (vector path): the dropout mask
    is a function of the flat output index only, so the zero patterns must coincide."""
    hc, _ = _ops()
    n, H, dv, p, seed = 3001, 8, 12, 0.2, 42424242
    W = H * dv
    attn, u = _positive_inputs(n, W, torch.bfloat16, seed=3)
    for concat in (0, 1):
        out_ln, _, _ = hc.cuda_norm_mul_dropout_fwd(attn, u, torch.ones(W, device=DEV, dtype=torch.bfloat16),
                                                    torch.full((W,), 4.0, device=DEV, dtype=torch.bfloat16), EPS, p, seed,
                                                    False, concat, False, H, dv)
        out_gn, _, _ = hc.cuda_norm_mul_dropout_fwd(attn, u, torch.ones(H, device=DEV, dtype=torch.bfloat16),
                                                    torch.full((H,), 4.0, device=DEV, dtype=torch.bfloat16), EPS, p, seed,
                                                    False, concat, True, H, dv)
        assert_same_zeros(out_ln, out_gn, f"group norm dv = 12 vs layer-norm view (concat {concat})")
        keep = (out_gn != 0).float().mean().item()
        assert abs(keep - (1 - p)) < 0.01, keep


# ------------------------------------------------------------------------------------------------------------------
# SiLU on a strided column block
# ------------------------------------------------------------------------------------------------------------------
def _silu_refs(x, dy):
    x64, dy64 = x.double().cpu(), dy.double().cpu()
    sg = torch.sigmoid(x64)
    fwd = x64 * sg
    bwd = dy64 * sg * (1 + x64 * (1 - sg))
    mag_b = dy64.abs() * sg * (1 + x64.abs() * (1 - sg))
    return fwd, bwd, (fwd.abs(), x64.abs()), (mag_b, x64.abs())


@pytest.mark.parametrize("shape", ["block", "uvqk8", "uvqk_odd", "large"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16], ids=IDS.get)
def test_silu_fwd_bwd(dtype, shape):
    """block: contiguous [1001, 200] (vector count not a multiple of 4 x 256); uvqk8: the u columns of uvqk at ml20m's layout
    (H = 8, dv = dqk = 32: row stride 2 H (dv + dqk) = 1024); uvqk_odd: H = 3, dv = 5, dqk = 6 -> stride 66 (not a multiple of
    8) and 15 u columns; large: [45000, 256], more vectors than the 1056-CTA forward and 2112-CTA backward grids cover in one
    pass.  The backward writes d_u in place into a NaN-poisoned duvqk: every other column must stay bit-identical."""
    hc, _ = _ops()
    g = torch.Generator().manual_seed(len(shape))
    if shape in ("block", "large"):
        n, c = (1001, 200) if shape == "block" else (45000, 256)
        stride = c
    else:
        H, dv, dqk = (8, 32, 32) if shape == "uvqk8" else (3, 5, 6)
        n, c, stride = 2053, H * dv, 2 * H * (dv + dqk)
    buf = (3 * torch.randn(n, stride, generator=g)).to(dtype)
    dy = torch.randn(n, c, generator=g).to(dtype)
    bufd = buf.to(DEV)
    x = bufd[:, :c]
    y = hc.cuda_silu_fwd(x)
    fwd, bwd, mag_f, mag_b = _silu_refs(buf[:, :c], dy)
    _assert_ulp(y, fwd, mag_f, dtype, "silu forward")
    poison = torch.full((n, stride), float("nan"), dtype=dtype, device=DEV)
    before = poison.clone()
    hc.cuda_silu_bwd(dy.to(DEV), x, poison[:, :c])
    _assert_ulp(poison[:, :c], bwd, mag_b, dtype, "silu backward")
    ibits = {torch.float32: torch.int32, torch.bfloat16: torch.int16, torch.float16: torch.int16}[dtype]
    assert torch.equal(poison[:, c:].view(ibits), before[:, c:].view(ibits)), "silu backward wrote outside d_u"
    assert torch.equal(bufd.cpu().view(ibits), buf.view(ibits)), "silu forward modified its input"
