"""The bf16 d = 32 attention on exactly scaled fp16 operands (DESIGN.md 3.0), emulated on the CPU.

`operand_exps` restates the exponents of csrc/attn_fp16_operands.cuh; `emulate` quantises every MMA operand as the kernels
do (fp16 copies of q, k, v, dO; fp16 P and dS after their scales; fp32 accumulation; bf16 outputs) and is held to the
parity bound of the GPU tests against the fp64 oracle."""
import math

import numpy as np
import pytest
import torch

from oracle import hstu_oracle as O
from util import TOL

D = 32


def _log2(bits):
    """floor(log2 x) of a non-negative float given by its fp32 bits, or None for 0, Inf and NaN."""
    e, m = bits >> 23, bits & 0x7FFFFF
    if bits == 0 or e >= 255:
        return None
    return e - 127 if e else m.bit_length() - 1 - 149


def _bits(x):
    return int(np.array(abs(x), dtype=np.float32).view(np.uint32))


def _clamp(e):
    return max(-126, min(127, e))


def operand_exps(amax, alpha, d=D):
    """amax: the four amax values (q, k, v, dO) of one (sequence, head) -> dict of exponents q, k, v, o, p, s."""
    lq, lk, lv, lo = (_log2(_bits(a)) for a in amax)
    la = _log2(_bits(alpha))
    ld = int(math.log2(d))
    x = {n: 0 if l is None else 14 - l for n, l in zip("qkvo", (lq, lk, lv, lo))}
    if la is not None:
        r = x["q"] + x["k"] - (la - 1 + 126)
        if r > 0:
            x["q"] -= (r + 1) // 2
            x["k"] -= r // 2
    x["p"] = 0 if None in (lq, lk, la) else _clamp(15 - (la + ld + lq + lk + 4))
    x["s"] = 0 if None in (lv, lo) else _clamp(15 - (ld + lo + lv + 5))
    return x


def _f32(x):
    return x.to(torch.float32)


def _pow2(e):
    return math.ldexp(1.0, _clamp(e))


def emulate(q, k, v, do, alpha, n_max, scale_pd=True):
    """One sequence, one head, causal mask: out, dq, dk, dv (bf16) as the scaled fp16 kernels compute them."""
    amax = [float(t.float().abs().max()) for t in (q, k, v, do)]
    ex = operand_exps(amax, alpha)
    if not scale_pd:
        ex["p"] = ex["s"] = 0
    qc, kc, vc, oc = (_f32(torch.ldexp(t.double(), torch.tensor(float(e))).to(torch.float16))
                      for t, e in zip((q, k, v, do), (ex["q"], ex["k"], ex["v"], ex["o"])))
    n = q.shape[0]
    mask = torch.ones(n, n).tril().bool()
    c_s = np.float32(np.ldexp(np.float32(alpha / 2), -(ex["q"] + ex["k"])))
    s = qc @ kc.T  # fp32 accumulators: 2^(e_q + e_k) S
    x = s * float(c_s)
    t = torch.tanh(x)
    p = torch.where(mask, (x * _pow2(ex["p"])) * (1 + t), 0.0).to(torch.float16).float()
    dp = oc @ vc.T  # 2^(e_v + e_o) dP
    g2 = t + x * (1 - t * t)
    ds = torch.where(mask, dp * (1 + g2) * _pow2(ex["s"] - ex["v"] - ex["o"]), 0.0).to(torch.float16).float()
    out = torch.ldexp((p @ vc) * (1.0 / n_max), torch.tensor(float(-(ex["p"] + ex["v"]))))
    dv = torch.ldexp((p.T @ oc) * (1.0 / n_max), torch.tensor(float(-(ex["p"] + ex["o"]))))
    dk_scale = 0.5 * alpha / n_max
    dk = torch.ldexp((ds.T @ qc) * dk_scale, torch.tensor(float(-(ex["s"] + ex["q"]))))
    dq = torch.ldexp((ds @ kc) * dk_scale, torch.tensor(float(-(ex["s"] + ex["k"]))))
    return [t.to(torch.bfloat16) for t in (out, dq, dk, dv)]


def _case(n, sigma, seed, tiny=False):
    g = torch.Generator().manual_seed(seed)
    if tiny:  # the `attn` bench workload: U(-0.01, 0.01) inputs, alpha = 1/d
        q, k, v = (torch.empty(n, 1, D).uniform_(-0.01, 0.01, generator=g).to(torch.bfloat16) for _ in range(3))
        alpha = 1.0 / D
    else:  # q, k ~ N(0, sigma^2), alpha = 1/sqrt(d): rms(alpha S) = sigma^2
        q, k = ((sigma * torch.randn(n, 1, D, generator=g)).to(torch.bfloat16) for _ in range(2))
        v = torch.randn(n, 1, D, generator=g).to(torch.bfloat16)
        alpha = 1.0 / D**0.5
    do = torch.randn(n, 1, D, generator=g).to(torch.bfloat16)
    return q, k, v, do, alpha


def _errors(q, k, v, do, alpha, scale_pd=True):
    n = q.shape[0]
    off = torch.tensor([0, n])
    ref = [O.hstu_mha_fwd(n, alpha, q, k, v, off, dtype=torch.float64)]
    ref += list(O.hstu_mha_bwd(n, alpha, do, q, k, v, off, dtype=torch.float64))
    got = emulate(q[:, 0], k[:, 0], v[:, 0], do[:, 0], alpha, n, scale_pd)
    res = {}
    for name, a, r in zip(("out", "dq", "dk", "dv"), got, ref):
        r = r[:, 0].float()
        lim = math.hypot(TOL[torch.bfloat16], O.storage_quantisation(r, torch.bfloat16))
        res[name] = (O.rel_l2(a.float(), r), lim)
    return res


# q, k ~ N(0, sigma^2): rms(alpha S) = 0.09, 1, 2.25, 4 (the sweep of test_gpu_attention_numerics.py)
@pytest.mark.parametrize("rms", [0.09, 1.0, 2.25, 4.0])
def test_scaled_fp16_emulation_within_budget_across_logit_scales(rms):
    for name, (err, lim) in _errors(*_case(300, rms**0.5, 5)).items():
        assert err <= lim, f"{name}: {err:.3e} > {lim:.3e}"


def test_scaled_fp16_emulation_within_budget_at_tiny_logits():
    for name, (err, lim) in _errors(*_case(400, 0, 7, tiny=True)).items():
        assert err <= lim, f"{name}: {err:.3e} > {lim:.3e}"


def test_without_the_p_ds_scales_tiny_logits_fall_into_fp16_subnormals():
    res = _errors(*_case(400, 0, 7, tiny=True), scale_pd=False)
    assert res["out"][0] > res["out"][1], res  # P ~ 1e-5 is below fp16's smallest normal 6.1e-5


def test_exponents_map_each_amax_into_2_14_to_2_15():
    for a in (1e-38, 3.1e-20, 0.01, 1.0, 7.5, 6.5e4, 1e30, 3e38):
        a32 = float(np.float32(a))
        e = operand_exps([a32, 1.0, a32, a32], 1.0 / 32)
        for key in "vo":
            assert 2.0**14 <= math.ldexp(a32, e[key]) < 2.0**15, (a, key, e)
        # the scaled operand holds every bf16 value of the tensor exactly (fp16 normal range)
        assert np.isfinite(np.float16(math.ldexp(a32, e["v"])))


def test_exponent_edge_cases():
    # amax 0: no scale, and no P / dS scale from a zero factor
    e = operand_exps([0.0, 1.0, 0.0, 1.0], 0.125)
    assert e["q"] == 0 and e["v"] == 0 and e["p"] == 0 and e["s"] == 0
    # Inf / NaN: exponent 0 (the sequence is poisoned whatever the scale); the P / dS exponents stay finite integers
    for bad in (float("inf"), float("nan")):
        e = operand_exps([bad, 1.0, 1.0, bad], 0.125)
        assert e["q"] == 0 and e["o"] == 0 and e["p"] == 0 and e["s"] == 0
    # tiny q and k: the pair is lowered so that alpha / 2 * 2^-(e_q + e_k) is a normal fp32 number
    for alpha in (1.0 / 32, 1.0, 64.0):
        e = operand_exps([1e-38, 1e-38, 1.0, 1.0], alpha)
        c_s = np.ldexp(np.float32(alpha / 2), -(e["q"] + e["k"]))
        assert np.isfinite(c_s) and c_s >= np.finfo(np.float32).tiny, (alpha, e)
    # huge amax: scaled down into fp16's range; every combined scalar is a normal fp32 number
    e = operand_exps([3e38, 1.0, 3e38, 3e38], 1.0 / 32)
    assert e["q"] == -113 and e["v"] == -113
    for x in (e["p"], e["s"], e["s"] - e["v"] - e["o"]):
        assert -126 <= x <= 127


def test_p_and_ds_bounds_keep_operands_below_fp16_max():
    # |P| <= |alpha| d amax_q amax_k and |dP (1 + g2)| <= 2.2 d amax_dO amax_v: the scaled bounds stay below 2^15
    for aq, ak, av, ao, alpha in ((1.0, 1.0, 1.0, 1.0, 1.0), (0.01, 0.01, 0.01, 1.0, 1 / 32), (7.9, 3.3, 1e-3, 2e4, 0.3)):
        e = operand_exps([aq, ak, av, ao], alpha)
        assert math.ldexp(alpha * D * aq * ak, e["p"]) < 2.0**15
        assert math.ldexp(2.2 * D * ao * av, e["s"]) < 2.0**15
        assert math.ldexp(alpha * D * aq * ak, e["p"]) >= 2.0**10  # and well above fp16's normal range
