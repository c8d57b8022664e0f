"""The bf16 d = 32 wgmma attention on exactly scaled fp16 copies (DESIGN.md 3.0): the copies are exact, rows past
max_seq_len do not change the scales, and power-of-two changes of the inputs act bitwise on the outputs."""
import ctypes as C

import pytest
import torch

from test_attention_fp16_operands_cpu import operand_exps
from util import offsets_from

pytestmark = pytest.mark.gpu

D, H, N = 32, 2, 1024
LENGTHS = [1024, 700, 1100, 333]  # the third sequence runs past max_seq_len


def _inputs(seed=3):
    g = torch.Generator().manual_seed(seed)
    L = sum(LENGTHS)
    q, k, v = ((0.4 * torch.randn(L, H, D, generator=g)).to(torch.bfloat16) for _ in range(3))
    do = torch.randn(L, H, D, generator=g).to(torch.bfloat16)
    return [t.cuda() for t in (q, k, v, do)]


def _run(q, k, v, do, alpha=1.0 / D**0.5):
    from generative_recommenders_b200 import _lib
    from generative_recommenders_b200.ops.hstu_attention import cuda_hstu_attention_bwd, cuda_hstu_attention_fwd

    off = offsets_from(LENGTHS, "cuda")
    nt = torch.tensor([4, 1, 9, 2], device="cuda")
    out = cuda_hstu_attention_fwd(N, alpha, q, k, v, off, num_targets=nt, impl=_lib.IMPL_UMMA)
    dq, dk, dv = (torch.empty_like(t) for t in (q, k, v))
    cuda_hstu_attention_bwd(N, alpha, do, q, k, v, dq, dk, dv, off, num_targets=nt, impl=_lib.IMPL_UMMA)
    torch.cuda.synchronize()
    return out, dq, dk, dv


def _prepass(q, k, v, do, alpha=0.25):
    """Runs the backward through the C ABI with a workspace owned here: (amax bits [B, H, 4], fp16 copies [4][L, H, D])."""
    from generative_recommenders_b200 import _lib
    from generative_recommenders_b200.ops import hstu_attention as ha

    off = offsets_from(LENGTHS, "cuda")
    p = _lib.AttnParams()
    ha._fill_common(p, N, alpha, q, k, v, off, None, 0, 0, 0, _lib.IMPL_UMMA)
    dq, dk, dv = (torch.empty_like(t) for t in (q, k, v))
    p.dout, p.dq, p.dk, p.dv_out = do.data_ptr(), dq.data_ptr(), dk.data_ptr(), dv.data_ptr()
    p.do_row_stride, p.do_head_stride = do.stride(0), do.stride(1)
    p.dq_row_stride, p.dq_head_stride = dq.stride(0), dq.stride(1)
    p.dk_row_stride, p.dk_head_stride = dk.stride(0), dk.stride(1)
    p.dv_row_stride, p.dv_head_stride = dv.stride(0), dv.stride(1)
    ws = ha._workspace(p, True, q.device)
    _lib.check(_lib.lib().hstu_attn_bwd(C.byref(p), _lib.stream_ptr(q.device)), "hstu_attn_bwd")
    torch.cuda.synchronize()
    base = p.workspace - ws.data_ptr()
    B, L = len(LENGTHS), q.shape[0]
    amax_bytes = (B * H * 4 * 4 + 255) // 256 * 256
    copy_bytes = (L * H * D * 2 + 255) // 256 * 256
    raw = ws[base:]
    amax = raw[: B * H * 16].view(torch.int32).view(B, H, 4).clone()
    copies = [raw[amax_bytes + i * copy_bytes: amax_bytes + i * copy_bytes + L * H * D * 2].view(torch.float16).view(L, H, D).clone()
              for i in range(4)]
    return amax, copies


def test_fp16_copies_are_the_bf16_inputs_times_a_power_of_two():
    q, k, v, do = _inputs()
    amax, copies = _prepass(q, k, v, do)
    off = [0]
    for n in LENGTHS:
        off.append(off[-1] + n)
    for b in range(len(LENGTHS)):
        rows = slice(off[b], off[b] + min(LENGTHS[b], N))
        for h in range(H):
            bits = amax[b, h].cpu().tolist()
            vals = [torch.tensor([x], dtype=torch.int32).view(torch.float32).item() for x in bits]
            ref = [float(t[rows, h].float().abs().max()) for t in (q, k, v, do)]
            assert vals == ref, (b, h, vals, ref)
            ex = operand_exps(vals, 0.25)
            for i, (t, e) in enumerate(zip((q, k, v, do), (ex["q"], ex["k"], ex["v"], ex["o"]))):
                back = torch.ldexp(copies[i][rows, h].float(), torch.tensor(float(-e), device="cuda")).to(torch.bfloat16)
                assert torch.equal(back.view(torch.int16), t[rows, h].view(torch.int16)), (b, h, i)


def test_rows_past_max_seq_len_do_not_change_the_scales():
    q, k, v, do = _inputs()
    amax0, _ = _prepass(q, k, v, do)
    start = LENGTHS[0] + LENGTHS[1] + N  # rows >= max_seq_len of the third sequence
    end = start + LENGTHS[2] - N
    for t, val in zip((q, k, v, do), (1e4, float("inf"), float("nan"), -3e5)):
        t[start:end] = val
    amax1, _ = _prepass(q, k, v, do)
    assert torch.equal(amax0, amax1)


def _bits(ts):
    return [t.view(torch.int16) for t in ts]


@pytest.mark.parametrize("e", [3, -5])
def test_power_of_two_changes_of_the_inputs_act_bitwise(e):
    q, k, v, do = _inputs()
    out, dq, dk, dv = _run(q, k, v, do)
    s = 2.0**e
    # q 2^e with k 2^-e: out and dv unchanged, dq scaled by 2^-e, dk by 2^e
    o1, dq1, dk1, dv1 = _run(q * s, k / s, v, do)
    assert torch.equal(o1.view(torch.int16), out.view(torch.int16))
    assert torch.equal(dv1.view(torch.int16), dv.view(torch.int16))
    assert torch.equal(dq1.view(torch.int16), (dq / s).view(torch.int16))
    assert torch.equal(dk1.view(torch.int16), (dk * s).view(torch.int16))
    # v 2^e: out, dq and dk scaled by 2^e
    o2, dq2, dk2, dv2 = _run(q, k, v * s, do)
    for a, b_ in ((o2, out * s), (dq2, dq * s), (dk2, dk * s), (dv2, dv)):
        assert torch.equal(a.view(torch.int16), b_.view(torch.int16))
    # dO 2^e: dq, dk and dv scaled by 2^e
    _, dq3, dk3, dv3 = _run(q, k, v, do * s)
    for a, b_ in ((dq3, dq * s), (dk3, dk * s), (dv3, dv * s)):
        assert torch.equal(a.view(torch.int16), b_.view(torch.int16))
