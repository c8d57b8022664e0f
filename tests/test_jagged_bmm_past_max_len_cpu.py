"""The contract of jagged_dense_bmm_broadcast_add for sequences longer than max_seq_len, on the CPU: rows at positions
>= max_seq_len are exact zeros in the output and in d_jagged, and add nothing to d_dense / d_bias.  It is what the
reference's eager path computes (ops/pytorch/pt_jagged.py:77-98: truncate at max_seq_len with jagged_to_padded_dense, come
back through dense_to_jagged, which pads the rows past the dense length with 0), pinned here by the fixture
jagged_bmm_past_max_len_bf16.pt generated from that path, and by the fbgemm stand-in's dense_to_jagged that it relies on."""
import torch

from conftest import golden
from oracle import fbgemm_shim
from oracle import hstu_oracle as O
from util import offsets_from

FIXTURE = "jagged_bmm_past_max_len_bf16.pt"


def test_fixture_reaches_past_max_seq_len():
    """The fixture has sequences shorter than, equal to and longer than max_seq_len (not a multiple of 64), one past the
    second 64-row tile; their rows past max_seq_len are zeros in out and d_jagged and the others are not."""
    g = golden(FIXTURE)
    m = g["max_seq_len"]
    off = g["seq_offsets"].tolist()
    lengths = [e - s for s, e in zip(off[:-1], off[1:])]
    assert m % 64 != 0 and 0 in lengths and m in lengths and m + 1 in lengths and max(lengths) > 64 * ((m + 63) // 64)
    for s, e in zip(off[:-1], off[1:]):
        n = min(e - s, m)
        for name in ("out", "d_jagged"):
            assert bool((g[name][s + n:e] == 0).all()), f"{name}: rows past max_seq_len must be zero"
            assert bool((g[name][s:s + n] != 0).any(-1).all()), f"{name}: rows below max_seq_len must carry values"


def test_oracle_matches_fixture_past_max_seq_len():
    """The oracle in the fixture's dtype reproduces the reference, and in fp64 it keeps the rows past max_seq_len at exact
    zeros with no gradient through them."""
    g = golden(FIXTURE)
    m = g["max_seq_len"]
    j, d, b = (g[n].clone().requires_grad_() for n in ("jagged", "dense", "bias"))
    out = O.jagged_dense_bmm_broadcast_add(m, g["seq_offsets"], j, d, b)
    out.backward(g["dout"])
    torch.testing.assert_close(out, g["out"])
    for a, r in ((j.grad, g["d_jagged"]), (d.grad, g["d_dense"]), (b.grad, g["d_bias"])):
        torch.testing.assert_close(a, r)

    j64, d64, b64 = (g[n].double().requires_grad_() for n in ("jagged", "dense", "bias"))
    out64 = O.jagged_dense_bmm_broadcast_add(m, g["seq_offsets"], j64, d64, b64)
    assert out64.dtype == torch.float64
    out64.backward(g["dout"].double())
    off = g["seq_offsets"].tolist()
    ref_dd = torch.zeros_like(d64)
    for bi, (s, e) in enumerate(zip(off[:-1], off[1:])):
        n = min(e - s, m)
        assert bool((out64[s + n:e] == 0).all()) and bool((j64.grad[s + n:e] == 0).all())
        ref_dd[bi] = j64[s:s + n].detach().T @ g["dout"][s:s + n].double()
    torch.testing.assert_close(d64.grad, ref_dd, rtol=1e-12, atol=1e-12)


def test_shim_dense_to_jagged_pads_rows_past_dense_length():
    """dense_to_jagged returns one row per jagged row: rows past the dense length are 0 (fbgemm's padding value), and the
    gradient reaches only the dense rows that were read."""
    lengths = [0, 2, 5, 3]
    off = offsets_from(lengths)
    N, D = 3, 4
    dense = torch.randn(len(lengths), N, D, dtype=torch.float64, requires_grad=True)
    vals, offs = fbgemm_shim._dense_to_jagged(dense, [off], total_L=int(off[-1]))
    assert vals.shape == (sum(lengths), D) and offs[0] is off
    expect = torch.cat([torch.cat([dense[b, :min(n, N)], dense.new_zeros(max(n - N, 0), D)]) for b, n in enumerate(lengths)])
    assert torch.equal(vals, expect)
    vals.backward(torch.ones_like(vals))
    mask = (torch.arange(N).view(1, N) < torch.tensor(lengths).view(-1, 1)).double().unsqueeze(-1).expand_as(dense)
    assert torch.equal(dense.grad, mask)
    # lengths within the dense length: the rows as before, nothing padded
    short = offsets_from([1, 3, 0, 2])
    v2, _ = fbgemm_shim._dense_to_jagged(dense.detach(), [short])
    assert torch.equal(v2, torch.cat([dense.detach()[0, :1], dense.detach()[1, :3], dense.detach()[3, :2]]))
