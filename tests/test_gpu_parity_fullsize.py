"""GPU parity of the wgmma/TMA attention kernels against the CPU oracle AT THE SHAPES THAT ARE BENCHMARKED
(BASELINE.json: d = 32 at Lmax = 8192 is the HSTU-large headline; d = 64 / 128 / 256 are the microbench grid), and of the
bf16 STU stack (forward, dx and every parameter gradient) in the configuration bench.py times.

The oracle evaluates one [n, n] score matrix per (sequence, head) in fp32: 8192 rows x 2 heads is a few seconds of CPU.
Tolerance: tests/util.py (sqrt((1e-3)^2 + q^2), q = storage rounding of the 16-bit output) -- no further allowance -- on the
whole tensor and on every 64-row segment of every (sequence, head).
"""
import pytest
import torch

from oracle import hstu_oracle as O
from util import assert_rel, assert_rel_segments, offsets_from

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda")


def _case(d, lmax, lengths, targets, H, dtype, seed, scale=0.5):
    g = torch.Generator().manual_seed(seed)
    off = offsets_from(lengths)
    L = int(off[-1])
    x = torch.empty(L, H, 3 * d).uniform_(-scale, scale, generator=g).to(dtype)
    q, k, v = torch.split(x, [d, d, d], dim=-1)  # strided views of one buffer, as the fused block passes them
    dout = torch.randn(L, H, d, generator=g).to(dtype)
    return q, k, v, dout, off, torch.tensor(targets)


@pytest.mark.parametrize("d,lmax,lengths,targets,H", [
    (32, 8192, [8192, 7411], [20, 3], 2),       # the headline head dim at the headline length (one full-length sequence)
    (64, 2048, [2048, 1850, 1], [11, 0, 1], 2),   # a 1-row sequence next to two long ones
    (64, 4224, [517, 300, 129, 0, 64], [11, 0, 1, 0, 3], 2),   # max_seq_len far above every length: most CTAs return at once
    (32, 1024, [1024, 77, 0, 640, 1, 255, 256, 257], [3, 0, 0, 20, 1, 0, 9, 2], 3),   # empty / 1-row sequences, lengths around a tile edge
    (128, 4096, [4096, 3700], [7, 20], 2),
    (256, 1024, [1024, 921, 130], [5, 20, 0], 2),
])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_umma_fwd_bwd_vs_oracle_at_bench_shapes(d, lmax, lengths, targets, H, dtype):
    from generative_recommenders_b200 import _lib
    from generative_recommenders_b200.common import HammerKernel
    from generative_recommenders_b200.ops.hstu_attention import hstu_mha

    if dtype == torch.float16 and lmax == 8192:
        pytest.skip("one dtype is enough at the largest size (CPU oracle time)")
    q, k, v, dout, off, nt = _case(d, lmax, lengths, targets, H, dtype, 4242 + d)
    alpha = 1.0 / d**0.5
    qd, kd, vd = (t.to(DEV).requires_grad_() for t in (q, k, v))
    # d = 256: wgmma forward, generic backward (dK + dV alone fill the registers) -> AUTO; otherwise wgmma is forced
    impl = _lib.IMPL_AUTO if d == 256 else _lib.IMPL_UMMA
    if d == 256:
        import ctypes as C

        from generative_recommenders_b200.ops.hstu_attention import _fill_common

        p = _lib.AttnParams()
        _fill_common(p, lmax, alpha, qd, kd, vd, off.to(DEV), nt.to(DEV), 0, 0, 0, _lib.IMPL_AUTO)
        o_ = torch.empty(qd.shape, device=DEV, dtype=dtype)
        p.out, p.o_row_stride, p.o_head_stride = o_.data_ptr(), o_.stride(0), o_.stride(1)
        assert _lib.lib().hstu_attn_select_impl(C.byref(p), 0) == _lib.IMPL_UMMA, "d = 256 forward must run on wgmma"
    out = hstu_mha(lmax, alpha, qd, kd, vd, off.to(DEV), num_targets=nt.to(DEV), kernel=HammerKernel.CUDA, impl=impl)
    out.backward(dout.to(DEV))
    ref = O.hstu_mha_fwd(lmax, alpha, q, k, v, off, nt)
    rdq, rdk, rdv = O.hstu_mha_bwd(lmax, alpha, dout, q, k, v, off, nt)
    for name, a, r in (("out", out, ref), ("dq", qd.grad, rdq), ("dk", kd.grad, rdk), ("dv", vd.grad, rdv)):
        assert_rel(a, r, f"wgmma d={d} lmax={lmax} {dtype} {name}")
        assert_rel_segments(a, r, off, lmax, f"wgmma d={d} lmax={lmax} {dtype} {name}")


@pytest.mark.parametrize("dout_scale", [1.0, 3e-8, 2e4])
def test_umma_bwd_is_invariant_to_the_scale_of_dout(dout_scale):
    """dS is a 16-bit tensor-core operand: gradients as small as a mean-over-1e7-elements loss produces, or large ones, must
    come out with the same relative accuracy."""
    from generative_recommenders_b200 import _lib
    from generative_recommenders_b200.common import HammerKernel
    from generative_recommenders_b200.ops.hstu_attention import hstu_mha

    d, lmax, H = 32, 700, 3
    q, k, v, dout, off, nt = _case(d, lmax, [700, 513, 64], [3, 9, 1], H, torch.bfloat16, 99)
    dout = (dout.float() * dout_scale).to(torch.bfloat16)
    alpha = 1.0 / d**0.5
    qd, kd, vd = (t.to(DEV).requires_grad_() for t in (q, k, v))
    hstu_mha(lmax, alpha, qd, kd, vd, off.to(DEV), num_targets=nt.to(DEV), kernel=HammerKernel.CUDA,
             impl=_lib.IMPL_UMMA).backward(dout.to(DEV))
    rdq, rdk, rdv = O.hstu_mha_bwd(lmax, alpha, dout, q, k, v, off, nt)
    for name, a, r in (("dq", qd.grad, rdq), ("dk", kd.grad, rdk), ("dv", vd.grad, rdv)):
        assert_rel(a, r, f"dout x {dout_scale:g}: {name}")


def test_stu_stack_bf16_gradients_vs_oracle():
    """The configuration bench.py times -- D=256, H=8, dqk=dv=32, bf16, recompute on, wgmma attention writing dq/dk/dv in
    place into the strided `duvqk` -- forward, dx and EVERY parameter gradient against the fp32 oracle evaluated on the
    bf16-valued parameters.  Between the ops of a layer the GPU path stores bf16 activations (LN output, uvqk, attention
    output, y: ~8 roundings per layer and direction), which the fp32 oracle does not: the budget for this end-to-end
    comparison is therefore stated separately (1e-2), it is not the per-op tolerance of tests/util.py."""
    from generative_recommenders_b200 import _lib
    from generative_recommenders_b200.modules.stu import STULayer, STULayerConfig, STUStack

    torch.manual_seed(17)
    D, H, dh, layers, N = 256, 8, 32, 2, 1536
    lengths = [1536, 1200, 333]
    nts = [12, 3, 1]
    off = offsets_from(lengths)
    L = int(off[-1])
    stack = STUStack([STULayer(STULayerConfig(embedding_dim=D, num_heads=H, hidden_dim=dh, attention_dim=dh,
                                              output_dropout_ratio=0.0, target_aware=True, recompute_normed_x=True,
                                              recompute_uvqk=True, recompute_y=True, sort_by_length=True))
                      for _ in range(layers)])
    # non-trivial norm parameters (the default initialisation is weight 1 / bias 0)
    with torch.no_grad():
        for n, p in stack.named_parameters():
            if "norm_weight" in n:
                p.add_(0.1 * torch.randn_like(p))
            if "norm_bias" in n or "beta" in n:
                p.add_(0.05 * torch.randn_like(p))
    stack = stack.to(DEV).to(torch.bfloat16)
    x = torch.randn(L, D).to(torch.bfloat16)
    dout = torch.randn(L, D).to(torch.bfloat16)
    xd = x.to(DEV).requires_grad_()
    launches0 = _lib.LAUNCHES
    y = stack(x=xd, x_lengths=torch.tensor(lengths, device=DEV), x_offsets=off.to(DEV), max_seq_len=N,
              num_targets=torch.tensor(nts, device=DEV))
    y.backward(dout.to(DEV))
    assert _lib.LAUNCHES > launches0
    sd = {k: v.detach().float().cpu() for k, v in stack.state_dict().items()}
    layer_params = [{k.split(".")[-1]: v for k, v in sd.items() if k.startswith(f"_stu_layers.{i}.")} for i in range(layers)]
    ry, rdx, rgrads = O.stu_stack_fwd_bwd(x.float(), off, N, torch.tensor(nts), layer_params, H, dh, dh, dout.float())
    assert_rel(y, ry, "stack bf16 y", tol=1e-2)
    assert_rel(xd.grad, rdx, "stack bf16 dx", tol=1e-2)
    for n, p in stack.named_parameters():
        i, name = int(n.split(".")[1]), n.split(".")[-1]
        assert_rel(p.grad, rgrads[i][name], f"stack bf16 grad {n}", tol=1e-2)
