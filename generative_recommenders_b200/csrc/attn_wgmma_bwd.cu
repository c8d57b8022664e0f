// Jagged HSTU attention backward on the Hopper warpgroup tensor cores (wgmma) with TMA-staged tiles.  bf16 / fp16,
// dqk == dv in {32, 64, 128}.
//
// One CTA per (128-row KEY tile, head, sequence); early key tiles (the heavy ones under a causal mask) are scheduled first.
// K and V of the tile stay in shared memory; the CTA streams the 64-row query tiles that can attend to it (Q_j and dO_j,
// TMA ring of STAGES).  Two warpgroups of 64 key rows each.  Per query tile:
//                      S^T  = K Q_j^T,  dP^T = V dO_j^T          (A = K / V, B = Q_j / dO_j, all K-major)
//                      P^T  = silu(alpha S) * mask               (1/N folded into the dV epilogue)
//                      dS^T = dP sig (1 + x (1 - sig)) * mask    (alpha/N folded into the dK epilogue and the dQ convert)
//                      dV  += P^T dO_j,  dK += dS^T Q_j          (A from registers, B = dO_j / Q_j MN-major)
//                    dS^T also goes to shared memory ([kv][q], q contiguous, two alternating buffers), and warpgroup j % 2
//                    computes dQ_j = dS K over all 128 keys (A = dS^T MN-major, B = K MN-major) and adds it to an fp32
//                    accumulator in global memory (each key-tile CTA contributes to every later query tile); a small convert
//                    kernel scales it by alpha/N and writes dq in the input dtype.
// Thread 0 issues the first TMA loads: K and V once, then Q_j and dO_j; afterwards each warp releases a stage once its MMAs
// that read it have completed, and the warp whose release is the last of the eight refills it (release_is_last, wgmma.cuh),
// so no thread waits for a free stage.  No separate producer warp: the dK and dV accumulators (d = 128: 64 registers each
// per thread) need the register budget of a 256-thread block.
// Each warpgroup waits for its own MMAs before the next elementwise step (an MMA batch left in flight across it makes ptxas
// serialise the batch); a Q_j / dO_j stage is released as soon as dV / dK of tile j have completed.
// P and dS are 16-bit operands of the input format: fp16, or for bf16 inputs a hi + lo pair of bf16 operands (wgmma.cuh,
// Operand), so that their rounding stays inside the 1e-3 parity budget whatever the scale of dO.  bf16 inputs at d = 32 run
// the fp16 kernels below on exactly scaled fp16 copies of q, k, v, dO with scaled fp16 P and dS (`amax`,
// attn_fp16_operands.cuh); their epilogues undo the scales and write bf16.
//
//
// d = 32, and d = 64 / 128 when the caller asks for a deterministic backward (hstu_attn_params.deterministic), run two
// kernels instead, with no atomics and no per-tile coupling between the warpgroups (DESIGN.md 3.2):
//   attn_bwd_dkdv_wgmma_kernel  the kernel above without the dS buffers, the dS barrier and dQ: dK and dV only.
//   attn_bwd_dq_wgmma_kernel    query-stationary, shaped like the forward: one CTA per (128-row query tile, head, sequence),
//                               Q and dO resident, K and V streamed in 64-key tiles; it recomputes S = Q K^T and
//                               dP = dO V^T, forms dS from one tanh and accumulates dQ += dS K in registers.  Its K / V ring
//                               is refilled like the forward's, by the last warp to release a stage.
// Every dq / dk / dv element is then summed by one thread in a fixed order, so the result is bitwise reproducible.
// At d = 32 recomputing S and dP costs two MMA units per score against the eight that the whole backward issues, while the
// elementwise work per score is the same; at larger d the recomputed MMAs weigh more and the fused kernel stays the default.
// The split kernels run two CTAs per SM at d = 32 and one at d = 64 / 128 (their accumulators need more than 128
// registers per thread there); bf16 at d = 64 / 128 keeps the hi + lo operand pairs.
//
// Reference math: ops/triton/triton_hstu_attention.py:995-1006,1222 and SURVEY.md appendix A; unlike the Triton
// kernel dQ is accumulated in fp32, not in the input dtype (triton_attention_utils.py:47-60).
#include <string.h>

#include "attn_fp16_operands.cuh"
#include "common.cuh"
#include "internal.h"
#include "wgmma.cuh"

namespace hstu {
using namespace wg;

bool wgmma_fwd_supported(const hstu_attn_params& p);
bool aligned_view(const void* ptr, long long row_stride, long long head_stride);

struct alignas(64) BwdParams {
  CUtensorMap tmQ, tmK, tmV, tmDO;
  const void* seq_offsets;
  const void* num_targets;
  void* dk;
  void* dv;
  float* dq_acc;  // [L, H, D] fp32, zero-initialised (fused kernel)
  void* dq;       // attn_bwd_dq_wgmma_kernel
  long long dk_row_stride, dk_head_stride, dv_row_stride, dv_head_stride, dq_row_stride, dq_head_stride;
  int offsets_i64, targets_i64;
  int max_seq_len, heads;
  int win, min_full, ctx;
  float alpha_half;
  float dv_scale;  // 1 / N
  float dk_scale;  // alpha / (2 N): dS^T holds 2 dS N / alpha
  const uint32_t* amax;  // fp16 kernels on scaled copies of bf16 inputs: [B, H, 4] amax bits (attn_fp16_operands.cuh); else null
};

// Scalars of the d = 32 kernels on scaled fp16 operands (identities for unscaled inputs): the score accumulators hold
// 2^(e_q + e_k) S and 2^(e_v + e_o) dP; P and 2 dS N / alpha are formed as 2^e_p P and 2^e_s (2 dS N / alpha).
struct BwdScales {
  float c_s = 0.f, c_p = 1.f, c_d = 1.f;  // alpha / 2 * 2^-(e_q + e_k), 2^e_p, 2^(e_s - e_v - e_o)
  int e_dv = 0, e_dk = 0, e_dq = 0;       // epilogue exponents: -(e_p + e_o), -(e_s + e_q), -(e_s + e_k)
  __device__ __forceinline__ BwdScales(const BwdParams& p, int b, int h, int d) {
    c_s = p.alpha_half;
    if (p.amax == nullptr) return;
    const OperandExps ex = operand_exps(p.amax + ((long long)b * p.heads + h) * kAmaxSlots, 2.f * p.alpha_half, d);
    c_s = ldexpf(p.alpha_half, -(ex.q + ex.k));
    c_p = pow2f(ex.p);
    c_d = pow2f(ex.s - ex.v - ex.o);
    e_dv = -(ex.p + ex.o);
    e_dk = -(ex.s + ex.q);
    e_dq = -(ex.s + ex.k);
  }
};

// CTAs per SM of the split kernels: two at d = 32 (<= 128 registers per thread), one at d = 64 / 128
constexpr int split_min_blocks(int d) { return d == 32 ? 2 : 1; }
constexpr int kSmemPerSm = 232448;  // dynamic shared memory one CTA may use on sm_90

// FUSED_DQ: the key-tile kernel also computes dQ (dS buffers in shared memory); without it the layout ends after the ring,
// which then has four stages at every d (d = 128: 192 KB, one CTA per SM)
template <int D, bool FUSED_DQ = true>
struct BwdCfg {
  static constexpr int BKV = 128, BQ = 64;
  static constexpr int SW = (D * 2 >= 128) ? 128 : D * 2;
  static constexpr int BOX_COLS = SW / 2;
  static constexpr int NBOX = D / BOX_COLS;
  static constexpr int KV_BOX = BKV * SW;
  static constexpr int QD_BOX = BQ * SW;
  static constexpr int KV_BYTES = BKV * D * 2;
  static constexpr int QD_BYTES = BQ * D * 2;
  static constexpr int STAGES = (D <= 32 || !FUSED_DQ) ? 4 : (D == 64 ? 3 : 2);  // Q_j / dO_j ring depth
  static constexpr int DS_BYTES = BKV * BQ * 2;                      // one [128 kv][64 q] box, 128-byte swizzle
  static constexpr int DQN = D < 64 ? D : 64;                        // dQ columns per pass (one 128-byte box of K)
  static constexpr int OFF_K = 0;
  static constexpr int OFF_V = OFF_K + KV_BYTES;
  static constexpr int OFF_Q = OFF_V + KV_BYTES;
  static constexpr int OFF_DO = OFF_Q + STAGES * QD_BYTES;
  static constexpr int OFF_DS = OFF_DO + STAGES * QD_BYTES;          // [buffer 0/1][hi / lo]
  static constexpr int OFF_BAR = OFF_DS + (FUSED_DQ ? 4 * DS_BYTES : 0);
  static constexpr int SMEM_BYTES = OFF_BAR + 256 + 1024;
  static_assert(SMEM_BYTES * (FUSED_DQ ? 1 : split_min_blocks(D)) <= kSmemPerSm, "shared memory budget");
};
constexpr int kBwdThreads = 256;

struct BwdBars {
  uint64_t kv_full;
  uint64_t qd_full[4];
  uint32_t qd_free[4];  // release counters of the Q_j / dO_j stages (release_is_last: one arrival per warp and use)
};

// query tiles of a key tile: the contextual prefix tiles [0, A), then the causal / window range
struct QTiles {
  int A, first, T;
  __device__ __forceinline__ int at(int i) const { return i < A ? i : first + (i - A); }
};

// Body of the key-stationary kernels: FUSED_DQ = attn_bwd_wgmma_kernel (dK, dV and the dQ atomics), otherwise
// attn_bwd_dkdv_wgmma_kernel (dK and dV only; the warpgroups meet at the ring and once at the query tile that crosses the
// sequence end).
template <int D, bool BF16, bool FUSED_DQ>
__device__ __forceinline__ void bwd_key_tile(const BwdParams& p) {
  using Cfg = BwdCfg<D, FUSED_DQ>;
  constexpr int SW = Cfg::SW, BQ = Cfg::BQ, NST = Cfg::STAGES;
  const int b = blockIdx.z, h = blockIdx.y;
  const int n0 = blockIdx.x * Cfg::BKV;
  const long long row0 = load_index(p.seq_offsets, p.offsets_i64, b);
  int len = (int)(load_index(p.seq_offsets, p.offsets_i64, b + 1) - row0);
  if (len > p.max_seq_len) {  // rows past max_seq_len get zero gradients
    if (blockIdx.x == 0) {
      zero_rows(p.dk, 2, p.dk_row_stride, (long long)h * p.dk_head_stride, D, row0 + p.max_seq_len, row0 + len);
      zero_rows(p.dv, 2, p.dv_row_stride, (long long)h * p.dv_head_stride, D, row0 + p.max_seq_len, row0 + len);
    }
    len = p.max_seq_len;
  }
  if (n0 >= len) return;
  const int n_tgt = p.num_targets ? (int)load_index(p.num_targets, p.targets_i64, b) : -1;
  const SeqMask msk = make_seq_mask(len, n_tgt, p.win, p.min_full, p.ctx);
  const int nrows = min(Cfg::BKV, len - n0);
  QTiles qt;
  {
    int lo, hi, ctx_hi;
    q_range_for_kv_rows(msk, n0, n0 + nrows, &lo, &hi, &ctx_hi);
    qt.A = (ctx_hi + BQ - 1) / BQ;
    qt.first = max(lo / BQ, qt.A);
    qt.T = qt.A + max(0, (hi + BQ - 1) / BQ - qt.first);
  }

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  BwdBars* bars = reinterpret_cast<BwdBars*>(smem + Cfg::OFF_BAR);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (tid == 0) {
    mbar_init(&bars->kv_full, 1);
    for (int i = 0; i < NST; ++i) {
      mbar_init(&bars->qd_full[i], 1);
      bars->qd_free[i] = 0u;
    }
    fence_barrier_init();
  }
  __syncthreads();

  // TMA issue: thread 0 loads K, V and the first STAGES query tiles; the warp that completes the release of a stage (below)
  // loads query tile j + STAGES into it
  auto load_qd = [&](int j) {
    const int st = j % NST;
    const int q_row = (int)(row0 + (long long)qt.at(j) * BQ);
    mbar_arrive_expect_tx(&bars->qd_full[st], 2 * Cfg::QD_BYTES);
#pragma unroll
    for (int bx = 0; bx < Cfg::NBOX; ++bx) {
      tma_load_3d(smem + Cfg::OFF_Q + st * Cfg::QD_BYTES + bx * Cfg::QD_BOX, &p.tmQ, &bars->qd_full[st], bx * Cfg::BOX_COLS, h, q_row);
      tma_load_3d(smem + Cfg::OFF_DO + st * Cfg::QD_BYTES + bx * Cfg::QD_BOX, &p.tmDO, &bars->qd_full[st], bx * Cfg::BOX_COLS, h, q_row);
    }
  };
  if (tid == 0) {
    prefetch_tensormap(&p.tmQ);
    prefetch_tensormap(&p.tmK);
    prefetch_tensormap(&p.tmV);
    prefetch_tensormap(&p.tmDO);
    mbar_arrive_expect_tx(&bars->kv_full, 2 * Cfg::KV_BYTES);
#pragma unroll
    for (int bx = 0; bx < Cfg::NBOX; ++bx) {
      tma_load_3d(smem + Cfg::OFF_K + bx * Cfg::KV_BOX, &p.tmK, &bars->kv_full, bx * Cfg::BOX_COLS, h, (int)(row0 + n0));
      tma_load_3d(smem + Cfg::OFF_V + bx * Cfg::KV_BOX, &p.tmV, &bars->kv_full, bx * Cfg::BOX_COLS, h, (int)(row0 + n0));
    }
    for (int j = 0; j < min(qt.T, NST); ++j) load_qd(j);
  }
  __syncwarp();

  const int wgi = warp >> 2, w = warp & 3, g = lane >> 2, t4 = lane & 3;
  const int r_loc = wgi * 64 + w * 16 + g;  // key row (inside the tile) of accumulator rows g (+ 8)
  const int k_base = n0 + r_loc;
  const uint32_t sk = smem_u32(smem + Cfg::OFF_K), sv = smem_u32(smem + Cfg::OFF_V);
  const uint32_t sq = smem_u32(smem + Cfg::OFF_Q), sdo = smem_u32(smem + Cfg::OFF_DO);
  const uint32_t sds = smem_u32(smem + Cfg::OFF_DS);
  const bool fast = msk.fast != 0;
  // keys of this tile that every query row >= q_full_from may attend (fast mask): all of them are history keys below the row
  const bool keys_hist = !msk.has_tgt || n0 + Cfg::BKV <= msk.max_id;

  constexpr bool kScaled = !BF16 && !FUSED_DQ && D == 32;  // the d = 32 dK / dV kernel also runs bf16 inputs on fp16 copies
  const BwdScales sc(p, b, h, D);
  float dv[D / 2], dk[D / 2];
#pragma unroll
  for (int e = 0; e < D / 2; ++e) dv[e] = dk[e] = 0.f;
  uint32_t pf_hi[4][4], pf_lo[4][4], df_hi[4][4], df_lo[4][4];
#pragma unroll
  for (int kk = 0; kk < 4; ++kk)
#pragma unroll
    for (int r = 0; r < 4; ++r) pf_hi[kk][r] = pf_lo[kk][r] = df_hi[kk][r] = df_lo[kk][r] = 0u;

  mbar_wait(&bars->kv_full, 0);
  // K rows >= len of a key tile that crosses the sequence end are B of dQ = dS K (dS is 0 there, K may be NaN)
  if (FUSED_DQ && n0 + Cfg::BKV > len) {  // CTA-uniform; K is loaded once
    zero_tile_rows<Cfg::BKV, SW, Cfg::NBOX, kBwdThreads>(smem + Cfg::OFF_K, len - n0);
    fence_proxy_async_smem();
    named_bar_sync(kBarZeroRows, kBwdThreads);
  }
  for (int j = 0; j < qt.T; ++j) {
    const int st = j % NST;
    const uint32_t ph = (j / NST) & 1;
    const int q0 = qt.at(j) * BQ;
    mbar_wait(&bars->qd_full[st], ph);
    // Q_j / dO_j rows >= len are B of dK += dS^T Q_j and dV += P^T dO_j (P and dS are 0 there, Q / dO may be NaN).  The query
    // tile that crosses the sequence end is the last one of the key tile (hi <= len, ctx_hi <= len), so its stage is not
    // refilled after the zeroing.
    if (q0 + BQ > len) {  // CTA-uniform
      zero_tile_rows<BQ, SW, Cfg::NBOX, kBwdThreads>(smem + Cfg::OFF_Q + st * Cfg::QD_BYTES, len - q0);
      zero_tile_rows<BQ, SW, Cfg::NBOX, kBwdThreads>(smem + Cfg::OFF_DO + st * Cfg::QD_BYTES, len - q0);
      fence_proxy_async_smem();
      named_bar_sync(kBarZeroRows, kBwdThreads);
    }
    float s[32], dp[32];
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < D / 16; ++ks) {
      const int kb = ks * 32, bx = kb / SW, off = kb % SW;
      const uint32_t ka = sk + bx * Cfg::KV_BOX + wgi * 64 * SW, va = sv + bx * Cfg::KV_BOX + wgi * 64 * SW;
      wgmma_ss<BQ, BF16, 0, 0>(s, desc_kmajor<SW>(ka, off), desc_kmajor<SW>(sq + st * Cfg::QD_BYTES + bx * Cfg::QD_BOX, off), ks > 0);
    }
#pragma unroll
    for (int ks = 0; ks < D / 16; ++ks) {
      const int kb = ks * 32, bx = kb / SW, off = kb % SW;
      const uint32_t va = sv + bx * Cfg::KV_BOX + wgi * 64 * SW;
      wgmma_ss<BQ, BF16, 0, 0>(dp, desc_kmajor<SW>(va, off), desc_kmajor<SW>(sdo + st * Cfg::QD_BYTES + bx * Cfg::QD_BOX, off), ks > 0);
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(s);
    fence_regs(dp);

    // p = x sig(x) and 2 dS = dP (1 + g2) from one tanh (h = alpha s / 2, t = tanh h, p = h (1 + t), g2 = t + h (1 - t^2)).
    // The mask case is chosen once per tile, outside the score loops, so that ptxas can overlap the tanh of independent
    // scores (as in the forward).  `v`: the pair is valid.
    auto score = [&](int n, bool v) {
      const float x = s[n] * (kScaled ? sc.c_s : p.alpha_half), xp = kScaled ? x * sc.c_p : x;
      const float t = tanh_approx(x);
      const float g2 = __fmaf_rn(x, __fmaf_rn(-t, t, 1.f), t);
      const float pv = __fmaf_rn(xp, t, xp);
      float dsv = __fmaf_rn(dp[n], g2, dp[n]);
      if (kScaled) dsv *= sc.c_d;
      s[n] = v ? pv : 0.f;
      dp[n] = v ? dsv : 0.f;
    };
    if (fast && keys_hist && n0 + Cfg::BKV <= q0 && q0 + BQ <= len) {  // tile-uniform: every pair valid
#pragma unroll
      for (int n = 0; n < BQ / 2; ++n) score(n, true);
    } else if (fast) {
      // mask_valid of the fast mask, kj < min(qi, max_id) || kj == qi, with the limit of each query column computed once
#pragma unroll
      for (int nb = 0; nb < BQ / 8; ++nb)
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const int qi = q0 + nb * 8 + 2 * t4 + c, lim = msk.has_tgt ? min(qi, msk.max_id) : qi;
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            const int kj = k_base + hh * 8;
            score(nb * 4 + hh * 2 + c, kj < len && qi < len && (kj < lim || kj == qi));
          }
        }
    } else {
#pragma unroll
      for (int nb = 0; nb < BQ / 8; ++nb)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int kj = k_base + (e >> 1) * 8, qi = q0 + nb * 8 + 2 * t4 + (e & 1);
          score(nb * 4 + e, kj < len && qi < len && mask_valid(msk, qi, kj));
        }
    }
    if constexpr (FUSED_DQ) {
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          const Operand<BF16> pp(s[8 * kk + 2 * r], s[8 * kk + 2 * r + 1]), dd(dp[8 * kk + 2 * r], dp[8 * kk + 2 * r + 1]);
          pf_hi[kk][r] = pp.hi; pf_lo[kk][r] = pp.lo;
          df_hi[kk][r] = dd.hi; df_lo[kk][r] = dd.lo;
        }
      }
      // dV += P^T dO_j, dK += dS^T Q_j
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        const uint64_t dod = desc_mnmajor<SW>(sdo + st * Cfg::QD_BYTES, kk * 16, Cfg::QD_BOX);
        const uint64_t qd = desc_mnmajor<SW>(sq + st * Cfg::QD_BYTES, kk * 16, Cfg::QD_BOX);
        wgmma_rs<D, BF16, 1>(dv, pf_hi[kk], dod, 1);
        wgmma_rs<D, BF16, 1>(dk, df_hi[kk], qd, 1);
        if constexpr (BF16) {
          wgmma_rs<D, BF16, 1>(dv, pf_lo[kk], dod, 1);
          wgmma_rs<D, BF16, 1>(dk, df_lo[kk], qd, 1);
        }
      }
    } else {
      // dV += P^T dO_j issued as soon as P is packed, then dK += dS^T Q_j: P^T and dS^T are never both held in fp32 next to
      // both fragment sets, which keeps a bf16 thread at 128 registers without wgmma serialisation (ptxas C7512)
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          const Operand<BF16> pp(s[8 * kk + 2 * r], s[8 * kk + 2 * r + 1]);
          pf_hi[kk][r] = pp.hi; pf_lo[kk][r] = pp.lo;
        }
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        const uint64_t dod = desc_mnmajor<SW>(sdo + st * Cfg::QD_BYTES, kk * 16, Cfg::QD_BOX);
        wgmma_rs<D, BF16, 1>(dv, pf_hi[kk], dod, 1);
        if constexpr (BF16) wgmma_rs<D, BF16, 1>(dv, pf_lo[kk], dod, 1);
      }
      wgmma_commit();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          const Operand<BF16> dd(dp[8 * kk + 2 * r], dp[8 * kk + 2 * r + 1]);
          df_hi[kk][r] = dd.hi; df_lo[kk][r] = dd.lo;
        }
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        const uint64_t qd = desc_mnmajor<SW>(sq + st * Cfg::QD_BYTES, kk * 16, Cfg::QD_BOX);
        wgmma_rs<D, BF16, 1>(dk, df_hi[kk], qd, 1);
        if constexpr (BF16) wgmma_rs<D, BF16, 1>(dk, df_lo[kk], qd, 1);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();  // an MMA batch never stays in flight across the elementwise code (ptxas would serialise them)
    fence_regs(dv);
    fence_regs(dk);
    fence_regs(pf_hi);
    fence_regs(pf_lo);
    fence_regs(df_hi);
    fence_regs(df_lo);
    // Q_j and dO_j are no longer read by this warp; the last of the eight warps to say so refills the stage
    if (lane == 0 && j + NST < qt.T && release_is_last<kBwdThreads / 32>(&bars->qd_free[st])) load_qd(j + NST);
    __syncwarp();
    if constexpr (!FUSED_DQ) continue;
    // dS^T -> shared memory buffer j & 1: element (kv r, q c) of a [128][64] 16-bit box with 128-byte swizzle
    const uint32_t dsb = sds + (j & 1) * 2 * Cfg::DS_BYTES;
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int row = r_loc + (r & 1) * 8, col = kk * 16 + (r >> 1) * 8 + 2 * t4;
        const uint32_t a = dsb + swizzled_chunk_offset<128>(row, col >> 3) + (col & 7) * 2;
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(a), "r"(df_hi[kk][r]) : "memory");
        if constexpr (BF16) asm volatile("st.shared.b32 [%0], %1;" ::"r"(a + Cfg::DS_BYTES), "r"(df_lo[kk][r]) : "memory");
      }
    fence_proxy_async_smem();
    named_bar_sync(1, 256);
    if (wgi == (j & 1)) {
      // dQ_j = dS K over the 128 keys of the tile, DQN columns per pass
      const int qrow = q0 + w * 16 + g;
#pragma unroll
      for (int pass = 0; pass < D / Cfg::DQN; ++pass) {
        float dq[Cfg::DQN / 2];
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < Cfg::BKV / 16; ++kk) {
          const uint64_t kd = desc_mnmajor<SW>(sk + pass * Cfg::KV_BOX, kk * 16, Cfg::KV_BOX);
          wgmma_ss<Cfg::DQN, BF16, 1, 1>(dq, desc_mnmajor<128>(dsb, kk * 16, Cfg::DS_BYTES), kd, kk > 0);
          if constexpr (BF16) wgmma_ss<Cfg::DQN, BF16, 1, 1>(dq, desc_mnmajor<128>(dsb + Cfg::DS_BYTES, kk * 16, Cfg::DS_BYTES), kd, 1);
        }
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(dq);
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int qi = qrow + hh * 8;
          if (qi < len) {
            float* dst = p.dq_acc + ((row0 + qi) * p.heads + h) * D + pass * Cfg::DQN + 2 * t4;
#pragma unroll
            for (int nb = 0; nb < Cfg::DQN / 8; ++nb)
              atomicAdd(reinterpret_cast<float2*>(dst + nb * 8), make_float2(dq[nb * 4 + hh * 2], dq[nb * 4 + hh * 2 + 1]));
          }
        }
      }
    }
  }

  // ---------------- epilogue: dK * alpha / (2N), dV * 1/N -> global ----------------
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int kj = k_base + hh * 8;
    if (kj < len) {
      uint16_t* krow = reinterpret_cast<uint16_t*>(p.dk) + (row0 + kj) * p.dk_row_stride + (long long)h * p.dk_head_stride + 2 * t4;
      uint16_t* vrow = reinterpret_cast<uint16_t*>(p.dv) + (row0 + kj) * p.dv_row_stride + (long long)h * p.dv_head_stride + 2 * t4;
#pragma unroll
      for (int nb = 0; nb < D / 8; ++nb) {
        float k0 = dk[nb * 4 + hh * 2] * p.dk_scale, k1 = dk[nb * 4 + hh * 2 + 1] * p.dk_scale;
        float v0 = dv[nb * 4 + hh * 2] * p.dv_scale, v1 = dv[nb * 4 + hh * 2 + 1] * p.dv_scale;
        if (kScaled) {
          k0 = scalbnf(k0, sc.e_dk), k1 = scalbnf(k1, sc.e_dk);
          v0 = scalbnf(v0, sc.e_dv), v1 = scalbnf(v1, sc.e_dv);
        }
        const bool out_bf16 = BF16 || p.amax != nullptr;
        *reinterpret_cast<uint32_t*>(krow + nb * 8) = out_bf16 ? pack_bf16x2(k0, k1) : pack_f16x2(k0, k1);
        *reinterpret_cast<uint32_t*>(vrow + nb * 8) = out_bf16 ? pack_bf16x2(v0, v1) : pack_f16x2(v0, v1);
      }
    }
  }
}

template <int D, bool BF16>
__global__ void __launch_bounds__(kBwdThreads, 1) attn_bwd_wgmma_kernel(const __grid_constant__ BwdParams p) {
  bwd_key_tile<D, BF16, true>(p);
}

// d = 32: two CTAs per SM (<= 128 registers per thread, 49 KB of shared memory)
template <int D, bool BF16>
__global__ void __launch_bounds__(kBwdThreads, split_min_blocks(D)) attn_bwd_dkdv_wgmma_kernel(const __grid_constant__ BwdParams p) {
  bwd_key_tile<D, BF16, false>(p);
}

// ---------------- dQ, query-stationary (split path) ----------------
template <int D>
struct DqCfg {
  static constexpr int BM = 128;  // query rows per CTA (two warpgroups of 64)
  static constexpr int BN = 64;   // key rows per tile
  static constexpr int SW = (D * 2 >= 128) ? 128 : D * 2;
  static constexpr int BOX_COLS = SW / 2;
  static constexpr int NBOX = D / BOX_COLS;
  static constexpr int Q_BOX = BM * SW;
  static constexpr int KV_BOX = BN * SW;
  static constexpr int Q_BYTES = BM * D * 2;
  static constexpr int KV_BYTES = BN * D * 2;
  static constexpr int STAGES = 3;  // K / V ring depth (d = 128: 161 KB, one CTA per SM)
  static constexpr int OFF_Q = 0;
  static constexpr int OFF_DO = OFF_Q + Q_BYTES;
  static constexpr int OFF_K = OFF_DO + Q_BYTES;
  static constexpr int OFF_V = OFF_K + STAGES * KV_BYTES;
  static constexpr int OFF_BAR = OFF_V + STAGES * KV_BYTES;
  static constexpr int SMEM_BYTES = OFF_BAR + 256 + 1024;
  static_assert(SMEM_BYTES * split_min_blocks(D) <= kSmemPerSm, "shared memory budget of split_min_blocks(D) CTAs per SM");
};

struct DqBars {
  uint64_t qd_full;
  uint64_t k_full[3], v_full[3];
  uint32_t k_free[3], v_free[3];  // release counters of the K / V stages (release_is_last: one arrival per warp and use)
};

// One CTA per (128-row query tile, head, sequence), heavy (late) tiles first; the forward's schedule, tile ranges and ring.
// Per 64-key tile each warpgroup runs S = Q K^T and dP = dO V^T (A and B K-major), releases V, forms
// 2 dS N / alpha = dP (1 + g2) * mask from one tanh, and runs dQ += dS K (A from registers, K read MN-major), then releases K.
template <int D, bool BF16>
__global__ void __launch_bounds__(kBwdThreads, split_min_blocks(D)) attn_bwd_dq_wgmma_kernel(const __grid_constant__ BwdParams p) {
  using Cfg = DqCfg<D>;
  constexpr int SW = Cfg::SW, BN = Cfg::BN, NST = Cfg::STAGES;
  constexpr bool kScaled = !BF16 && D == 32;  // also runs bf16 inputs on scaled fp16 copies
  const int b = blockIdx.z, h = blockIdx.y;
  const int m0 = (int)(gridDim.x - 1 - blockIdx.x) * Cfg::BM;
  const long long row0 = load_index(p.seq_offsets, p.offsets_i64, b);
  int len = (int)(load_index(p.seq_offsets, p.offsets_i64, b + 1) - row0);
  if (len > p.max_seq_len) {  // rows past max_seq_len get zero gradients
    if (blockIdx.x == 0) zero_rows(p.dq, 2, p.dq_row_stride, (long long)h * p.dq_head_stride, D, row0 + p.max_seq_len, row0 + len);
    len = p.max_seq_len;
  }
  if (m0 >= len) return;
  const int n_tgt = p.num_targets ? (int)load_index(p.num_targets, p.targets_i64, b) : -1;
  const SeqMask msk = make_seq_mask(len, n_tgt, p.win, p.min_full, p.ctx);
  const int mrows = min(Cfg::BM, len - m0);
  int lo, hi;
  kv_range_for_q_rows(msk, m0, m0 + mrows, &lo, &hi);
  const int t0 = lo / BN;
  const int T = (hi + BN - 1) / BN - t0;  // >= 1 (the diagonal tile)

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  DqBars* bars = reinterpret_cast<DqBars*>(smem + Cfg::OFF_BAR);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (tid == 0) {
    mbar_init(&bars->qd_full, 1);
    for (int i = 0; i < NST; ++i) {
      mbar_init(&bars->k_full[i], 1);
      mbar_init(&bars->v_full[i], 1);
      bars->k_free[i] = bars->v_free[i] = 0u;
    }
    fence_barrier_init();
  }
  __syncthreads();

  // TMA issue of key tile i into its K or V stage (tm = &p.tmK / &p.tmV, off = Cfg::OFF_K / OFF_V, full = its full barriers)
  auto load = [&](const CUtensorMap* tm, int off, uint64_t* full, int i) {
    const int st = i % NST;
    mbar_arrive_expect_tx(&full[st], Cfg::KV_BYTES);
#pragma unroll
    for (int bx = 0; bx < Cfg::NBOX; ++bx)
      tma_load_3d(smem + off + st * Cfg::KV_BYTES + bx * Cfg::KV_BOX, tm, &full[st], bx * Cfg::BOX_COLS, h,
                  (int)(row0 + (long long)(t0 + i) * BN));
  };
  // Thread 0 loads Q, dO and the first STAGES key tiles.  Afterwards each warp releases the V stage of tile i once its S / dP
  // MMAs have completed and the K stage once its dQ MMAs have, and the warp whose release is the last of the eight loads tile
  // i + STAGES into the stage (the forward's protocol).
  auto release = [&](const CUtensorMap* tm, int off, uint64_t* full, uint32_t* ctr, int i) {
    if (lane == 0 && i + NST < T && release_is_last<kBwdThreads / 32>(&ctr[i % NST])) load(tm, off, full, i + NST);
  };
  if (tid == 0) {
    prefetch_tensormap(&p.tmQ);
    prefetch_tensormap(&p.tmK);
    prefetch_tensormap(&p.tmV);
    prefetch_tensormap(&p.tmDO);
    mbar_arrive_expect_tx(&bars->qd_full, 2 * Cfg::Q_BYTES);
#pragma unroll
    for (int bx = 0; bx < Cfg::NBOX; ++bx) {
      tma_load_3d(smem + Cfg::OFF_Q + bx * Cfg::Q_BOX, &p.tmQ, &bars->qd_full, bx * Cfg::BOX_COLS, h, (int)(row0 + m0));
      tma_load_3d(smem + Cfg::OFF_DO + bx * Cfg::Q_BOX, &p.tmDO, &bars->qd_full, bx * Cfg::BOX_COLS, h, (int)(row0 + m0));
    }
    for (int i = 0; i < min(T, NST); ++i) {
      load(&p.tmK, Cfg::OFF_K, bars->k_full, i);
      load(&p.tmV, Cfg::OFF_V, bars->v_full, i);
    }
  }
  __syncwarp();

  const int wgi = warp >> 2, w = warp & 3, g = lane >> 2, t4 = lane & 3;
  const int q_base = m0 + wgi * 64 + w * 16 + g;  // query position of accumulator rows g (+ 8)
  const uint32_t sq = smem_u32(smem + Cfg::OFF_Q) + wgi * 64 * SW, sdo = smem_u32(smem + Cfg::OFF_DO) + wgi * 64 * SW;
  const uint32_t sk = smem_u32(smem + Cfg::OFF_K), sv = smem_u32(smem + Cfg::OFF_V);
  const bool fast = msk.fast != 0;
  const int full_lim = fast ? min(m0, msk.has_tgt ? msk.max_id : 0x7fffffff) : -1;  // keys < full_lim: valid for every row

  const BwdScales sc(p, b, h, D);
  float dq[D / 2];
#pragma unroll
  for (int e = 0; e < D / 2; ++e) dq[e] = 0.f;
  uint32_t a_hi[BN / 16][4], a_lo[BN / 16][4];
#pragma unroll
  for (int kk = 0; kk < BN / 16; ++kk)
#pragma unroll
    for (int r = 0; r < 4; ++r) a_hi[kk][r] = a_lo[kk][r] = 0u;
  // One wait per MMA batch: S and dP of tile i + 1 in the batch of dQ += dS_i K_i would hold S, dP, dQ and both dS fragment
  // sets at once, which does not fit in 128 registers with bf16 inputs (ptxas spills and serialises the MMAs).
  mbar_wait(&bars->qd_full, 0);
  for (int i = 0; i < T; ++i) {
    const int st = i % NST;
    const uint32_t ph = (i / NST) & 1;
    const uint32_t kst = sk + st * Cfg::KV_BYTES, vst = sv + st * Cfg::KV_BYTES;
    const int n0 = (t0 + i) * BN;
    float s[BN / 2], dp[BN / 2];
    mbar_wait(&bars->k_full[st], ph);
    mbar_wait(&bars->v_full[st], ph);
    // the last key tile may cross the sequence end: its K rows >= len are B of dQ += dS K (dS is 0 there, K may be NaN)
    if (n0 + BN > len) {  // CTA-uniform; the last tile, so its stage is not refilled
      zero_tile_rows<BN, SW, Cfg::NBOX, kBwdThreads>(smem + Cfg::OFF_K + st * Cfg::KV_BYTES, len - n0);
      fence_proxy_async_smem();
      named_bar_sync(kBarZeroRows, kBwdThreads);
    }
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < D / 16; ++ks) {
      const int kb = ks * 32, bx = kb / SW, off = kb % SW;
      wgmma_ss<BN, BF16, 0, 0>(s, desc_kmajor<SW>(sq + bx * Cfg::Q_BOX, off), desc_kmajor<SW>(kst + bx * Cfg::KV_BOX, off), ks > 0);
    }
#pragma unroll
    for (int ks = 0; ks < D / 16; ++ks) {
      const int kb = ks * 32, bx = kb / SW, off = kb % SW;
      wgmma_ss<BN, BF16, 0, 0>(dp, desc_kmajor<SW>(sdo + bx * Cfg::Q_BOX, off), desc_kmajor<SW>(vst + bx * Cfg::KV_BOX, off), ks > 0);
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(s);
    fence_regs(dp);
    release(&p.tmV, Cfg::OFF_V, bars->v_full, bars->v_free, i);
    __syncwarp();

    // 2 dS N / alpha = dP (1 + g2), g2 = t + h (1 - t^2), t = tanh h, h = alpha s / 2.  The mask case is chosen once per
    // tile, outside the score loops, so that ptxas can overlap the tanh of independent scores (as in the forward).
    auto dscore = [&](int n) {
      const float x = s[n] * sc.c_s;
      const float t = tanh_approx(x);
      const float g2 = __fmaf_rn(x, __fmaf_rn(-t, t, 1.f), t);
      float dsv = __fmaf_rn(dp[n], g2, dp[n]);
      if (kScaled) dsv *= sc.c_d;
      return dsv;
    };
    if (n0 + BN <= full_lim) {  // tile-uniform: every pair valid
#pragma unroll
      for (int n = 0; n < BN / 2; ++n) dp[n] = dscore(n);
    } else if (fast) {
      // mask_valid of the fast mask, kj < min(qi, max_id) || kj == qi, with the limits of the thread's two rows hoisted
      int lim[2];
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) lim[hh] = msk.has_tgt ? min(q_base + hh * 8, msk.max_id) : q_base + hh * 8;
#pragma unroll
      for (int nb = 0; nb < BN / 8; ++nb)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int qi = q_base + (e >> 1) * 8, kj = n0 + nb * 8 + 2 * t4 + (e & 1);
          const float dsv = dscore(nb * 4 + e);
          dp[nb * 4 + e] = (kj < len && (kj < lim[e >> 1] || kj == qi)) ? dsv : 0.f;
        }
    } else {
#pragma unroll
      for (int nb = 0; nb < BN / 8; ++nb)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int qi = q_base + (e >> 1) * 8, kj = n0 + nb * 8 + 2 * t4 + (e & 1);
          const float dsv = dscore(nb * 4 + e);
          dp[nb * 4 + e] = (kj < len && mask_valid(msk, qi, kj)) ? dsv : 0.f;
        }
    }
#pragma unroll
    for (int kk = 0; kk < BN / 16; ++kk) {
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const Operand<BF16> x(dp[8 * kk + 2 * r], dp[8 * kk + 2 * r + 1]);
        a_hi[kk][r] = x.hi;
        a_lo[kk][r] = x.lo;
      }
    }
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < BN / 16; ++kk) {
      const uint64_t kd = desc_mnmajor<SW>(kst, kk * 16, Cfg::KV_BOX);
      wgmma_rs<D, BF16, 1>(dq, a_hi[kk], kd, 1);
      if constexpr (BF16) wgmma_rs<D, BF16, 1>(dq, a_lo[kk], kd, 1);
    }
    wgmma_commit();
    wgmma_wait<0>();  // an MMA batch never stays in flight across the elementwise code (ptxas would serialise them)
    fence_regs(dq);
    fence_regs(a_hi);
    fence_regs(a_lo);
    release(&p.tmK, Cfg::OFF_K, bars->k_full, bars->k_free, i);
    __syncwarp();
  }

  // ---------------- epilogue: dQ * alpha / (2N) -> global ----------------
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int qi = q_base + hh * 8;
    if (qi - m0 < mrows) {
      uint16_t* qrow = reinterpret_cast<uint16_t*>(p.dq) + (row0 + qi) * p.dq_row_stride + (long long)h * p.dq_head_stride;
#pragma unroll
      for (int nb = 0; nb < D / 8; ++nb) {
        float a = dq[nb * 4 + hh * 2] * p.dk_scale, c = dq[nb * 4 + hh * 2 + 1] * p.dk_scale;
        if (kScaled) a = scalbnf(a, sc.e_dq), c = scalbnf(c, sc.e_dq);
        *reinterpret_cast<uint32_t*>(qrow + nb * 8 + 2 * t4) = (BF16 || p.amax != nullptr) ? pack_bf16x2(a, c) : pack_f16x2(a, c);
      }
    }
  }
}

// dq[r, h, :] = convert(dq_acc[r, h, :] * scale)
template <bool BF16>
__global__ void dq_convert_kernel(const float* __restrict__ acc, uint16_t* __restrict__ dq, long long rows, int heads, int D,
                                  long long row_stride, long long head_stride, float scale) {
  const long long nvec = rows * heads * (D / 8);
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < nvec; idx += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(idx % (D / 8));
    const long long rh = idx / (D / 8);
    const int hh = (int)(rh % heads);
    const long long r = rh / heads;
    const float4 a = *reinterpret_cast<const float4*>(acc + rh * D + v * 8);
    const float4 c = *reinterpret_cast<const float4*>(acc + rh * D + v * 8 + 4);
    uint4 o;
    if (BF16) {
      o = make_uint4(pack_bf16x2(a.x * scale, a.y * scale), pack_bf16x2(a.z * scale, a.w * scale),
                     pack_bf16x2(c.x * scale, c.y * scale), pack_bf16x2(c.z * scale, c.w * scale));
    } else {
      o = make_uint4(pack_f16x2(a.x * scale, a.y * scale), pack_f16x2(a.z * scale, a.w * scale),
                     pack_f16x2(c.x * scale, c.y * scale), pack_f16x2(c.z * scale, c.w * scale));
    }
    *reinterpret_cast<uint4*>(dq + r * row_stride + hh * head_stride + v * 8) = o;
  }
}

// ------------------------------------------------------------------------------------------------
// host
// ------------------------------------------------------------------------------------------------
static bool wgmma_bwd_supported(const hstu_attn_params& p) {
  if (!wgmma_fwd_supported(p)) return false;  // dtype / dims / alignment of q, k, v (out is not used by the backward)
  // d = 256: dK and dV alone would take all the registers of a consumer thread; the backward runs on the generic path
  if (p.dqk != 32 && p.dqk != 64 && p.dqk != 128) return false;
  return aligned_view(p.dout, p.do_row_stride, p.do_head_stride) && aligned_view(p.dq, p.dq_row_stride, p.dq_head_stride) &&
         aligned_view(p.dk, p.dk_row_stride, p.dk_head_stride) && aligned_view(p.dv_out, p.dv_row_stride, p.dv_head_stride);
}

bool wgmma_supported(const hstu_attn_params& p, bool bwd) {
  if (!bwd) return wgmma_fwd_supported(p);
  hstu_attn_params q = p;
  if (q.out == nullptr) q.out = const_cast<void*>(q.q);  // the forward check also looks at `out`
  q.o_row_stride = 8;
  q.o_head_stride = 8;
  return wgmma_bwd_supported(q);
}

// d = 32, or a deterministic backward: dK / dV and dQ in two kernels, without atomics or dQ workspace; otherwise the fused
// kernel (DESIGN.md 3.2)
static bool split_dq(const hstu_attn_params& p) { return p.dqk == 32 || p.deterministic != 0; }

// bf16 at d = 32: the fp16 kernels on exactly scaled copies (attn_fp16_operands.cu)
static bool fp16_copies(const hstu_attn_params& p) { return p.dtype == HSTU_BF16 && p.dqk == 32; }

size_t wgmma_workspace_bytes(const hstu_attn_params& p, bool bwd) {
  if (fp16_copies(p)) return fp16_operands_workspace_bytes(p, bwd);
  if (!bwd || split_dq(p)) return 0;
  return (size_t)p.total_rows * p.heads * p.dqk * sizeof(float);  // fp32 dQ accumulator [L, H, D]
}

// kSplit: the dK / dV and dQ kernels, else the fused kernel and the dQ convert.  f16: the scaled fp16 copies of bf16 inputs
// (the kernels are then the fp16 ones), or null
template <int D, bool BF16, bool kSplit>
static int launch_bwd_wgmma(const hstu_attn_params& p, cudaStream_t st, const Fp16Operands* f16 = nullptr) {
  using Cfg = BwdCfg<D, !kSplit>;
  const size_t need = f16 ? 0 : wgmma_workspace_bytes(p, true);
  if (need > 0 && (p.workspace == nullptr || p.workspace_bytes < need)) {
    set_error("hstu_attn_bwd: workspace of %zu bytes required (got %zu)", need, p.workspace_bytes);
    return HSTU_ERR_WORKSPACE;
  }
  // operands the kernels read: the inputs, or their contiguous fp16 copies
  const void* src[4] = {p.q, p.k, p.v, p.dout};
  long long rs[4] = {p.q_row_stride, p.k_row_stride, p.v_row_stride, p.do_row_stride};
  long long hs[4] = {p.q_head_stride, p.k_head_stride, p.v_head_stride, p.do_head_stride};
  if (f16)
    for (int i = 0; i < 4; ++i) src[i] = f16->copy[i], rs[i] = (long long)p.heads * D, hs[i] = D;
  BwdParams bp;
  memset(&bp, 0, sizeof(bp));
  if (f16) bp.amax = f16->amax;
  if (int e = make_tmap_rows_heads(&bp.tmQ, src[0], p.total_rows, p.heads, D, rs[0], hs[0], Cfg::BOX_COLS, Cfg::BQ)) return e;
  if (int e = make_tmap_rows_heads(&bp.tmK, src[1], p.total_rows, p.heads, D, rs[1], hs[1], Cfg::BOX_COLS, Cfg::BKV)) return e;
  if (int e = make_tmap_rows_heads(&bp.tmV, src[2], p.total_rows, p.heads, D, rs[2], hs[2], Cfg::BOX_COLS, Cfg::BKV)) return e;
  if (int e = make_tmap_rows_heads(&bp.tmDO, src[3], p.total_rows, p.heads, D, rs[3], hs[3], Cfg::BOX_COLS, Cfg::BQ)) return e;
  bp.seq_offsets = p.seq_offsets;
  bp.num_targets = p.num_targets;
  bp.dk = p.dk;
  bp.dv = p.dv_out;
  bp.dq_acc = reinterpret_cast<float*>(p.workspace);
  bp.dq = p.dq;
  bp.dk_row_stride = p.dk_row_stride;
  bp.dk_head_stride = p.dk_head_stride;
  bp.dv_row_stride = p.dv_row_stride;
  bp.dv_head_stride = p.dv_head_stride;
  bp.dq_row_stride = p.dq_row_stride;
  bp.dq_head_stride = p.dq_head_stride;
  bp.offsets_i64 = p.offsets_are_i64;
  bp.targets_i64 = p.num_targets_are_i64;
  bp.max_seq_len = p.max_seq_len;
  bp.heads = p.heads;
  bp.win = p.max_attn_len;
  bp.min_full = p.min_full_attn_seq_len;
  bp.ctx = p.contextual_seq_len;
  bp.alpha_half = 0.5f * p.alpha;
  bp.dv_scale = 1.0f / (float)p.max_seq_len;
  bp.dk_scale = 0.5f * p.alpha / (float)p.max_seq_len;
  if constexpr (kSplit) {
    auto kdkdv = attn_bwd_dkdv_wgmma_kernel<D, BF16>;
    HSTU_CUDA_OK(cudaFuncSetAttribute(kdkdv, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    kdkdv<<<dim3((p.max_seq_len + Cfg::BKV - 1) / Cfg::BKV, p.heads, p.batch), kBwdThreads, Cfg::SMEM_BYTES, st>>>(bp);
    HSTU_CUDA_OK(cudaGetLastError());
    // the dQ kernel tiles 128 query rows and 64 key rows
    using QC = DqCfg<D>;
    if (int e = make_tmap_rows_heads(&bp.tmQ, src[0], p.total_rows, p.heads, D, rs[0], hs[0], QC::BOX_COLS, QC::BM)) return e;
    if (int e = make_tmap_rows_heads(&bp.tmK, src[1], p.total_rows, p.heads, D, rs[1], hs[1], QC::BOX_COLS, QC::BN)) return e;
    if (int e = make_tmap_rows_heads(&bp.tmV, src[2], p.total_rows, p.heads, D, rs[2], hs[2], QC::BOX_COLS, QC::BN)) return e;
    if (int e = make_tmap_rows_heads(&bp.tmDO, src[3], p.total_rows, p.heads, D, rs[3], hs[3], QC::BOX_COLS, QC::BM)) return e;
    auto kdq = attn_bwd_dq_wgmma_kernel<D, BF16>;
    HSTU_CUDA_OK(cudaFuncSetAttribute(kdq, cudaFuncAttributeMaxDynamicSharedMemorySize, QC::SMEM_BYTES));
    kdq<<<dim3((p.max_seq_len + QC::BM - 1) / QC::BM, p.heads, p.batch), kBwdThreads, QC::SMEM_BYTES, st>>>(bp);
    HSTU_CUDA_OK(cudaGetLastError());
  } else {
    HSTU_CUDA_OK(cudaMemsetAsync(p.workspace, 0, need, st));
    auto kern = attn_bwd_wgmma_kernel<D, BF16>;
    HSTU_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    dim3 grid((p.max_seq_len + Cfg::BKV - 1) / Cfg::BKV, p.heads, p.batch);
    kern<<<grid, kBwdThreads, Cfg::SMEM_BYTES, st>>>(bp);
    HSTU_CUDA_OK(cudaGetLastError());
    const long long nvec = p.total_rows * p.heads * (D / 8);
    long long blocks = (nvec + 255) / 256;
    if (blocks > 132 * 16) blocks = 132 * 16;
    dq_convert_kernel<BF16><<<(int)blocks, 256, 0, st>>>(bp.dq_acc, reinterpret_cast<uint16_t*>(p.dq), p.total_rows, p.heads, D,
                                                         p.dq_row_stride, p.dq_head_stride, bp.dk_scale);
    HSTU_CUDA_OK(cudaGetLastError());
  }
  return 0;
}

int attn_wgmma_bwd(const hstu_attn_params& p, cudaStream_t st) {
  const bool bf = p.dtype == HSTU_BF16;
  const bool split = split_dq(p);
  switch (p.dqk) {
    case 32: {  // bf16: the fp16 kernels on exactly scaled copies (DESIGN.md 3.0)
      if (!bf) return launch_bwd_wgmma<32, false, true>(p, st);
      Fp16Operands f16;
      if (int e = fp16_operands_prepass(p, true, &f16, st)) return e;
      return launch_bwd_wgmma<32, false, true>(p, st, &f16);
    }
    case 64:
      if (split) return bf ? launch_bwd_wgmma<64, true, true>(p, st) : launch_bwd_wgmma<64, false, true>(p, st);
      return bf ? launch_bwd_wgmma<64, true, false>(p, st) : launch_bwd_wgmma<64, false, false>(p, st);
    case 128:
      if (split) return bf ? launch_bwd_wgmma<128, true, true>(p, st) : launch_bwd_wgmma<128, false, true>(p, st);
      return bf ? launch_bwd_wgmma<128, true, false>(p, st) : launch_bwd_wgmma<128, false, false>(p, st);
  }
  set_error("wgmma backward: unsupported head dim %d", p.dqk);
  return HSTU_ERR_UNSUPPORTED;
}

}  // namespace hstu
