"""The d = 32 wgmma attention backward reduces dQ without atomics, so two calls on the same inputs give bitwise identical
dq / dk / dv."""
import pytest
import torch

from util import offsets_from

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_d32_wgmma_backward_is_bitwise_repeatable(dtype):
    from generative_recommenders_b200 import _lib
    from generative_recommenders_b200.ops.hstu_attention import cuda_hstu_attention_bwd

    dev = torch.device("cuda")
    g = torch.Generator(device="cpu").manual_seed(11)
    lengths, N, H, d = [8192, 7700, 8100, 6000], 8192, 4, 32  # long rows: each dq element sums up to 64 key tiles
    off = offsets_from(lengths, dev)
    L = sum(lengths)
    q, k, v = (torch.empty(L, H, d).uniform_(-0.3, 0.3, generator=g).to(dev, dtype) for _ in range(3))
    do = torch.randn(L, H, d, generator=g).to(dev, dtype)
    nt = torch.tensor([3, 17, 1, 9], device=dev)
    runs = []
    for _ in range(2):
        dq, dk, dv = (torch.full((L, H, d), float("nan"), device=dev, dtype=dtype) for _ in range(3))
        cuda_hstu_attention_bwd(N, 1.0 / d**0.5, do, q, k, v, dq, dk, dv, off, num_targets=nt, impl=_lib.IMPL_UMMA)
        runs.append((dq, dk, dv))
    torch.cuda.synchronize()
    for name, a, b in zip(("dq", "dk", "dv"), *runs):
        assert torch.isfinite(a).all(), f"{name}: non-finite values"
        assert torch.equal(a.view(torch.int16), b.view(torch.int16)), f"{name}: two calls differ"
