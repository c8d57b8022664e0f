"""The bf16 d = 32 attention backward on the fp16 operands its forward kept (hstu_attn_fwd_keep_fp16_operands /
hstu_attn_bwd_on_fp16_operands, DESIGN.md 3.0): bitwise the backward that converts q, k, v again, NaN / Inf included, and
calls that do not run on such operands leave the handle empty and work as before."""
import pytest
import torch

from util import offsets_from

pytestmark = pytest.mark.gpu

D, H, N = 32, 2, 1024
LENGTHS = [1024, 700, 1100, 333]  # the third sequence runs past max_seq_len
TARGETS = [4, 1, 9, 2]


def _inputs(seed=5, dtype=torch.bfloat16, d=D):
    g = torch.Generator().manual_seed(seed)
    L = sum(LENGTHS)
    q, k, v = ((0.4 * torch.randn(L, H, d, generator=g)).to(dtype) for _ in range(3))
    do = torch.randn(L, H, d, generator=g).to(dtype)
    return [t.cuda() for t in (q, k, v, do)]


def _fwd_bwd(q, k, v, do, kept, **mask):
    """(out, dq, dk, dv, handle); kept: the forward keeps its operands and the backward reads no q, k, v."""
    from generative_recommenders_b200.ops.hstu_attention import Fp16Operands, cuda_hstu_attention_bwd, cuda_hstu_attention_fwd

    off = offsets_from(LENGTHS, "cuda")
    nt = torch.tensor(TARGETS, device="cuda")
    ops = Fp16Operands() if kept else None
    out = cuda_hstu_attention_fwd(N, 1.0 / D**0.5, q, k, v, off, num_targets=nt, fp16_operands=ops, **mask)
    dq, dk, dv = (torch.empty_like(t) for t in (q, k, v))
    has = ops is not None and ops.buf is not None
    cuda_hstu_attention_bwd(N, 1.0 / D**0.5, do, None if has else q, None if has else k, None if has else v, dq, dk, dv,
                            off, num_targets=nt, fp16_operands=ops, **mask)
    torch.cuda.synchronize()
    return out, dq, dk, dv, ops


def _bits(t):
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


@pytest.mark.parametrize("mask", [{}, {"max_attn_len": 200, "contextual_seq_len": 6}])
def test_kept_operands_bitwise(mask):
    q, k, v, do = _inputs()
    ref = _fwd_bwd(q, k, v, do, False, **mask)
    got = _fwd_bwd(q, k, v, do, True, **mask)
    assert got[4].buf is not None
    for name, a, b in zip(("out", "dq", "dk", "dv"), got[:4], ref[:4]):
        assert torch.equal(_bits(a), _bits(b)), name


def test_kept_operands_bitwise_with_nonfinite_inputs():
    q, k, v, do = _inputs(seed=6)
    off = offsets_from(LENGTHS, "cpu").tolist()
    # one (sequence, head) of each: Inf in q, NaN in v and dO; every other (sequence, head) keeps finite results
    q[off[1] + 17, 1, 3] = float("inf")
    v[off[1] + 40, 1, 0] = float("nan")
    do[off[3] + 2, 0, 5] = float("nan")
    ref = _fwd_bwd(q, k, v, do, False)
    got = _fwd_bwd(q, k, v, do, True)
    for name, a, b in zip(("out", "dq", "dk", "dv"), got[:4], ref[:4]):
        assert torch.equal(_bits(a), _bits(b)), name
    for t in got[1:4]:
        assert torch.isfinite(t[off[0]:off[1]]).all()  # sequence 0 shares no scale with the poisoned ones
        assert torch.isfinite(t[off[1]:off[2], 0]).all() and torch.isfinite(t[off[2]:off[3]]).all()
    assert not torch.isfinite(got[1][off[1]:off[2], 1]).all()  # ... and the poisoned head does see its NaN / Inf


def test_kept_operands_backward_twice():
    """The backward leaves the handle as the forward wrote it (retain_graph-style second backward)."""
    from generative_recommenders_b200.ops.hstu_attention import cuda_hstu_attention_bwd

    q, k, v, do = _inputs(seed=7)
    _, dq, dk, dv, ops = _fwd_bwd(q, k, v, do, True)
    again = [torch.empty_like(t) for t in (dq, dk, dv)]
    off = offsets_from(LENGTHS, "cuda")
    cuda_hstu_attention_bwd(N, 1.0 / D**0.5, do, None, None, None, *again, off,
                            num_targets=torch.tensor(TARGETS, device="cuda"), fp16_operands=ops)
    torch.cuda.synchronize()
    for a, b in zip(again, (dq, dk, dv)):
        assert torch.equal(_bits(a), _bits(b))


@pytest.mark.parametrize("dtype,d", [(torch.float16, 32), (torch.bfloat16, 64)])
def test_handle_stays_empty_off_the_bf16_d32_path(dtype, d):
    q, k, v, do = _inputs(seed=8, dtype=dtype, d=d)
    ref = _fwd_bwd(q, k, v, do, False)
    got = _fwd_bwd(q, k, v, do, True)
    assert got[4].buf is None
    for name, a, b in zip(("out", "dq", "dk", "dv"), got[:4], ref[:4]):
        assert torch.equal(_bits(a), _bits(b)), name


def test_kept_operands_take_misaligned_views():
    """The kept backward has no generic fallback: a dout, dq, dk or dv view the wgmma kernels cannot take (row stride not a
    whole number of 16-byte units) goes through a contiguous copy, with the same bits."""
    from generative_recommenders_b200.ops.hstu_attention import cuda_hstu_attention_bwd

    q, k, v, do = _inputs(seed=12)
    ref = _fwd_bwd(q, k, v, do, False)
    _, _, _, _, ops = _fwd_bwd(q, k, v, do, True)
    L = q.shape[0]
    wide = torch.zeros(L, H * D + 3, dtype=do.dtype, device="cuda")  # e.g. cat([dout, extra], 1) with 3 extra columns
    wide[:, :H * D] = do.view(L, H * D)
    bufs = [torch.zeros(L, H * D + 5, dtype=do.dtype, device="cuda") for _ in range(3)]
    grads = [b[:, :H * D].view(L, H, D) for b in bufs]
    cuda_hstu_attention_bwd(N, 1.0 / D**0.5, wide[:, :H * D].view(L, H, D), None, None, None, *grads,
                            offsets_from(LENGTHS, "cuda"), num_targets=torch.tensor(TARGETS, device="cuda"), fp16_operands=ops)
    torch.cuda.synchronize()
    for name, a, b in zip(("dq", "dk", "dv"), grads, ref[1:4]):
        assert torch.equal(_bits(a), _bits(b)), name


def test_hstu_mha_with_misaligned_dout():
    """hstu_mha at bf16 d = 32 with a dout whose row stride is no whole number of 16-byte units: the backward runs (on the
    generic kernels, which take any strides) and gives the gradients of the wgmma backward on a contiguous dout."""
    from generative_recommenders_b200.ops.hstu_attention import hstu_mha

    q, k, v, do = _inputs(seed=9)
    ref = _fwd_bwd(q, k, v, do, False)
    qg, kg, vg = (t.clone().requires_grad_() for t in (q, k, v))
    off = offsets_from(LENGTHS, "cuda")
    out = hstu_mha(N, 1.0 / D**0.5, qg, kg, vg, off, num_targets=torch.tensor(TARGETS, device="cuda"))
    L = q.shape[0]
    extra = torch.ones(L, 3, dtype=out.dtype, device="cuda", requires_grad=True)
    y = torch.cat([out.view(L, H * D), extra], dim=1)
    y.backward(torch.cat([do.view(L, H * D), torch.zeros(L, 3, dtype=do.dtype, device="cuda")], dim=1))
    assert torch.equal(_bits(out), _bits(ref[0]))
    for name, a, b in zip(("dq", "dk", "dv"), (qg.grad, kg.grad, vg.grad), ref[1:4]):
        a, b = a.float(), b.float()
        assert float((a - b).norm() / b.norm()) < 1e-2, name  # two implementations, each within bf16 storage of the oracle


def test_kept_operands_of_other_sizes_are_rejected():
    from generative_recommenders_b200.ops.hstu_attention import cuda_hstu_attention_bwd

    q, k, v, do = _inputs(seed=13)
    _, dq, dk, dv, ops = _fwd_bwd(q, k, v, do, True)
    ops.nbytes -= 256  # as if kept by a forward over fewer rows
    with pytest.raises(RuntimeError, match="operands buffer"):
        cuda_hstu_attention_bwd(N, 1.0 / D**0.5, do, None, None, None, dq, dk, dv, offsets_from(LENGTHS, "cuda"),
                                num_targets=torch.tensor(TARGETS, device="cuda"), fp16_operands=ops)


def test_stu_layer_recompute_uvqk_bitwise():
    """The layer's backward recomputes only the u columns of the uvqk GEMM under recompute_uvqk; its gradients are those of
    the backward that keeps the whole uvqk.  That the narrower GEMM gives the bits of the u columns of the full one is
    cuBLAS's choice of kernels for the two widths (it holds on H100 with CUDA 12.8 / 12.9), not something this project's
    code guarantees: a failure after a cuBLAS update means the two GEMMs now round differently, not that the handoff broke."""
    from generative_recommenders_b200.modules.stu import STULayer, STULayerConfig, STUStack

    off = offsets_from(LENGTHS, "cuda")
    L = sum(LENGTHS)
    x = torch.randn(L, 64, generator=torch.Generator().manual_seed(10)).to(torch.bfloat16).cuda()
    grads = []
    for recompute in (True, False):
        torch.manual_seed(11)
        stack = STUStack([STULayer(STULayerConfig(embedding_dim=64, num_heads=H, hidden_dim=D, attention_dim=D,
                                                  output_dropout_ratio=0.0, recompute_uvqk=recompute))])
        stack = stack.cuda().to(torch.bfloat16)
        xi = x.clone().requires_grad_()
        y = stack(x=xi, x_lengths=torch.tensor(LENGTHS, device="cuda"), x_offsets=off, max_seq_len=max(LENGTHS),
                  num_targets=torch.tensor(TARGETS, device="cuda"))
        y.float().square().mean().backward()
        grads.append([xi.grad] + [p.grad for p in stack.parameters()])
    for a, b in zip(*grads):
        assert torch.equal(_bits(a), _bits(b))
