// Exact fp16 operands for the bf16 d = 32 wgmma attention (DESIGN.md 3.0).
//
// wgmma multiplies A and B in one format.  bf16 has an 8-bit significand and fp16 an 11-bit one, so a bf16 value times a
// power of two is an exact fp16 value as long as it lands in fp16's normal range.  Per (sequence, head) the pre-pass
// (attn_fp16_operands.cu) takes amax = max |x| of q, k, v (and dO), and the kernels run on fp16 copies x * 2^e_x with the
// amax in [2^14, 2^15).  P and dS, computed in fp32, become single fp16 operands after scales 2^e_p / 2^e_s derived from
// rigorous bounds (|P| <= |alpha| d amax_q amax_k, |2 dS N / alpha| = |dP (1 + g2)| <= 2.2 d amax_dO amax_v) that put the
// bound below 2^15: no operand overflows, and small scores stay out of fp16 subnormals.  The epilogues undo every scale.
// Scales are per (sequence, head), so a NaN or Inf in one sequence changes no other sequence's scales.
#pragma once
#include <stdint.h>
#include <string.h>

namespace hstu {

// amax slots per (sequence, head): bit patterns of non-negative floats (ordered like the values; NaN above Inf)
enum { kAmaxQ = 0, kAmaxK = 1, kAmaxV = 2, kAmaxDO = 3, kAmaxSlots = 4 };

struct OperandExps {
  int q, k, v, o;  // fp16 copy of x = bf16 x * 2^e
  int p, s;        // P' = P 2^p, dS' = (2 dS N / alpha) 2^s
};

// floor(log2 x) of a finite positive float given by its bits (subnormals included); `special` for 0, Inf and NaN
__host__ __device__ inline int amax_log2(uint32_t bits, bool* special) {
  const uint32_t e = bits >> 23, m = bits & 0x7fffffu;
  *special = bits == 0u || e >= 255u;
  if (*special) return 0;
  if (e != 0u) return (int)e - 127;
  int top = 22;
  while (!(m >> top)) --top;
  return top - 149;
}

__host__ __device__ inline int clamp_exp(int e) { return e < -126 ? -126 : (e > 127 ? 127 : e); }

// Exponents of one (sequence, head) from its amax bits, alpha and the head dim.  An operand whose amax is 0, Inf or NaN gets
// exponent 0 (a zero operand needs no scale; a non-finite one poisons its own sequence whatever the scale), and so do P / dS
// when a factor of their bound is such an operand.  The q / k pair is lowered, if needed, so that the score scalar
// alpha / 2 * 2^-(e_q + e_k) stays a normal fp32 number; the P / dS exponents are clamped to the normal range, so that
// 2^p, 2^s and 2^(s - e_v - e_o) are normal fp32 numbers too.
__host__ __device__ inline OperandExps operand_exps(const uint32_t* amax, float alpha, int d) {
  bool zq, zk, zv, zo, za;
  const int lq = amax_log2(amax[kAmaxQ], &zq), lk = amax_log2(amax[kAmaxK], &zk);
  const int lv = amax_log2(amax[kAmaxV], &zv), lo = amax_log2(amax[kAmaxDO], &zo);
  const float aa = alpha < 0.f ? -alpha : alpha;
  uint32_t abits;
  memcpy(&abits, &aa, 4);
  const int la = amax_log2(abits, &za);
  int ld = 0;
  while ((2 << ld) <= d) ++ld;  // floor(log2 d)
  OperandExps x;
  x.q = zq ? 0 : 14 - lq;
  x.k = zk ? 0 : 14 - lk;
  x.v = zv ? 0 : 14 - lv;
  x.o = zo ? 0 : 14 - lo;
  if (!za) {
    const int lim = (la - 1) + 126;  // alpha / 2 >= 2^(la - 1): its product with 2^-(e_q + e_k) stays >= 2^-126
    const int r = x.q + x.k - lim;
    if (r > 0) {
      x.q -= (r + 1) / 2;
      x.k -= r / 2;
    }
  }
  // |P| <= |alpha| d amax_q amax_k < 2^(la + 1 + ld + 1 + lq + 1 + lk + 1)
  x.p = (zq || zk || za) ? 0 : clamp_exp(15 - (la + ld + lq + lk + 4));
  // |dP (1 + g2)| <= 2.2 d amax_dO amax_v < 2^(2 + ld + 1 + lo + 1 + lv + 1)
  x.s = (zv || zo) ? 0 : clamp_exp(15 - (ld + lo + lv + 5));
  return x;
}

// Exponent p of the fp8 forward's fp16 P operand P' = P 2^p (attn_wgmma_fwd_e4m3.cu, DESIGN.md 3.5).  With e4m3 q, k
// (|x| <= 448) and |silu y| <= |y|, |P| <= B = |alpha q_descale k_descale| d 448^2.  Writing each factor as m 2^e with m in
// [0.5, 1) (frexp) and d <= 2^ld: B < 2^(e_a + e_q + e_k + ld + 18), so p = -3 - (e_a + e_q + e_k + ld) puts B 2^p below
// 2^15, and (d a power of two) at or above 448^2 2^-6 > 2^11: no fp16 overflow, and no amax pass over q and k.  A zero, Inf
// or NaN factor gives p = 0, and p is clamped to fp32's normal exponents (pow2f), as in operand_exps.
__host__ __device__ inline int e4m3_p_exp(float alpha, float q_descale, float k_descale, int d) {
  const float f[3] = {alpha, q_descale, k_descale};
  int sum = 0;
  for (int i = 0; i < 3; ++i) {
    const float a = f[i] < 0.f ? -f[i] : f[i];
    uint32_t bits;
    memcpy(&bits, &a, 4);
    bool special;
    const int l = amax_log2(bits, &special);  // floor(log2 a) = frexp exponent - 1
    if (special) return 0;
    sum += l + 1;
  }
  int ld = 0;
  while ((1 << ld) < d) ++ld;  // ceil(log2 d)
  return clamp_exp(-3 - (sum + ld));
}

// 2^e for e in [-126, 127] (exact, built from the exponent bits)
__host__ __device__ inline float pow2f(int e) {
  const uint32_t b = (uint32_t)(clamp_exp(e) + 127) << 23;
  float f;
  memcpy(&f, &b, 4);
  return f;
}

}  // namespace hstu
