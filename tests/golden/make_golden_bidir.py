"""Generate the non-causal attention golden vectors from the UNMODIFIED reference eager path.

    python tests/golden/make_golden_bidir.py   # checkout at /root/reference, or HSTU_REFERENCE_ROOT=<checkout>

Writes tests/golden/bidir_attn_*.pt: outputs and gradients of the reference's own
ops/pytorch/pt_hstu_attention.py::pytorch_hstu_mha(causal=False) (its facade hstu_mha asserts causal=True, so the eager
function is called directly) on the CPU, on seeded inputs made by the recipe of make_golden.py's attn_case, with the
fbgemm_gpu jagged ops of oracle/fbgemm_shim.py.  They pin tests/bidir_oracle.py (tests/test_attention_bidir_cpu.py).
The files are named bidir_attn_* so that the causal checks over attn_*.pt do not pick them up.
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
REF_ROOT = os.environ.get("HSTU_REFERENCE_ROOT") or "/root/reference"
if not os.path.isdir(os.path.join(REF_ROOT, "generative_recommenders")):
    sys.exit(f"make_golden_bidir.py: no checkout of generative-recommenders at {REF_ROOT} (set HSTU_REFERENCE_ROOT)")
sys.path.insert(0, REF_ROOT)

from oracle import fbgemm_shim  # noqa: E402

fbgemm_shim.install()

import torch  # noqa: E402
from generative_recommenders.ops.pytorch.pt_hstu_attention import pytorch_hstu_mha  # noqa: E402


def offsets_from(lengths):
    off = torch.zeros(len(lengths) + 1, dtype=torch.int64)
    off[1:] = torch.cumsum(torch.as_tensor(lengths, dtype=torch.int64), 0)
    return off


def bidir_case(name, seed, B, H, max_uih, max_tgt, dqk, dv, targets, max_attn_len, ctx, min_full):
    g = torch.Generator().manual_seed(seed)
    lengths = torch.randint(max_uih + 1, (B,), generator=g)
    lengths[0] = 0 if B > 2 else lengths[0]  # an empty-history sequence
    nt = torch.randint(1, max_tgt + 1, (B,), generator=g)
    lengths = lengths + nt + ctx
    N = max_uih + max_tgt + ctx
    off = offsets_from(lengths.tolist())
    L = int(off[-1])
    mk = lambda d: torch.empty(L, H, d).uniform_(-0.1, 0.1, generator=g)  # noqa: E731
    q, k, v = mk(dqk), mk(dqk), mk(dv)
    dout = torch.randn(L, H, dv, generator=g)
    alpha = 1.0 / dqk**0.5
    qq, kk, vv = (t.clone().requires_grad_() for t in (q, k, v))
    out = pytorch_hstu_mha(max_seq_len=N, alpha=alpha, q=qq, k=kk, v=vv, seq_offsets=off, causal=False,
                           num_targets=nt if targets else None, max_attn_len=max_attn_len, contextual_seq_len=ctx,
                           min_full_attn_seq_len=min_full)
    out.backward(dout)
    torch.save(dict(name=name, max_seq_len=N, alpha=alpha, q=q, k=k, v=v, dout=dout, seq_offsets=off,
                    num_targets=nt if targets else None, max_attn_len=max_attn_len, contextual_seq_len=ctx,
                    min_full_attn_seq_len=min_full,
                    ref_f32=dict(out=out.detach(), dq=qq.grad, dk=kk.grad, dv=vv.grad)),
               os.path.join(HERE, f"bidir_attn_{name}.pt"))


def main():
    torch.manual_seed(0)
    bidir_case("plain", 11, 4, 2, 40, 6, 16, 16, False, 0, 0, 0)
    bidir_case("targets", 12, 5, 2, 50, 9, 16, 16, True, 0, 0, 0)
    bidir_case("context", 13, 4, 2, 40, 5, 16, 16, True, 0, 6, 0)
    bidir_case("window", 15, 4, 2, 60, 6, 16, 16, True, 7, 0, 0)
    bidir_case("window_full", 14, 4, 1, 70, 8, 16, 16, True, 9, 4, 13)


if __name__ == "__main__":
    main()
