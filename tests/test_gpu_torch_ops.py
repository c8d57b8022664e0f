"""torch.ops.hstu.hstu_mha / hstu_mha_fwd / hstu_mha_bwd (the reference's native schema, flash_api.cpp:275-365) on H100."""
import pytest
import torch

from oracle import hstu_oracle as O
from util import assert_rel, offsets_from

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")


def _inputs(d=64, H=2):
    g = torch.Generator().manual_seed(21)
    lengths = [300, 0, 129, 511]
    off = offsets_from(lengths)
    L = int(off[-1])
    q, k, v = (torch.empty(L, H, d).uniform_(-0.4, 0.4, generator=g).to(torch.bfloat16) for _ in range(3))
    do = torch.randn(L, H, d, generator=g).to(torch.bfloat16)
    return q, k, v, do, off, torch.tensor([3, 0, 7, 20])


def test_registered_ops_match_the_oracle_and_deterministic_is_bitwise_reproducible():
    from generative_recommenders_b200 import torch_ops

    torch_ops.register()
    q, k, v, do, off, nt = _inputs()
    N, alpha = 512, 0.125
    ref = O.hstu_mha_fwd(N, alpha, q, k, v, off, nt)
    rdq, rdk, rdv = O.hstu_mha_bwd(N, alpha, do, q, k, v, off, nt)
    off32, nt32 = off.to(DEV, torch.int32), nt.to(DEV, torch.int32)  # the reference op takes int32 offsets (flash_common.cpp)
    grads = []
    for deterministic in (False, True, True):
        qd, kd, vd = (t.to(DEV).requires_grad_() for t in (q, k, v))
        out = torch.ops.hstu.hstu_mha(N, alpha, qd, kd, vd, off32, True, nt32, None, 0, 0, 0, None, None, None, True,
                                      deterministic, 0)
        out.backward(do.to(DEV))
        for name, a, r in (("out", out, ref), ("dq", qd.grad, rdq), ("dk", kd.grad, rdk), ("dv", vd.grad, rdv)):
            assert_rel(a, r, f"torch.ops.hstu.hstu_mha deterministic={deterministic} {name}")
        grads.append((qd.grad.clone(), kd.grad.clone(), vd.grad.clone()))
    for a, b in zip(grads[1], grads[2]):
        assert torch.equal(a, b), "deterministic=True must be bitwise reproducible"
    # raw forward / backward operators: caller-allocated gradients, written in place
    qd, kd, vd = (t.to(DEV) for t in (q, k, v))
    out = torch.ops.hstu.hstu_mha_fwd(N, alpha, qd, kd, vd, off32, True, nt32, None, 0, 0, 0, None, None, None, 0)
    dq, dk, dv = torch.empty_like(qd), torch.empty_like(kd), torch.empty_like(vd)
    res = torch.ops.hstu.hstu_mha_bwd(N, alpha, do.to(DEV), qd, kd, vd, dq, dk, dv, off32, True, nt32, None, 0, 0, 0, True, False, 0)
    assert len(res) == 3 and res[0].data_ptr() == dq.data_ptr()
    assert_rel(out, ref, "hstu_mha_fwd")
    assert_rel(dq, rdq, "hstu_mha_bwd dq")
    with pytest.raises(RuntimeError):
        torch.ops.hstu.hstu_mha_fwd(N, alpha, qd, kd, vd, off32, True, nt32, torch.ones(N, device=DEV), 0, 0, 0, None, None, None, 0)
