// Jagged HSTU attention backward on the Hopper warpgroup tensor cores (wgmma) with TMA-staged tiles: the kernel bodies and
// their launchers (fused and split), shared by attn_wgmma_bwd.cu (dqk == dv in {32, 64, 128, 256}) and
// attn_wgmma_mixed_bwd.cu (dqk < dv, both in that set, split kernels only).  bf16 / fp16.  Two widths: DQK, of Q, K, dQ, dK
// and the reduction of S = Q K^T, and DV, of V, dO, dV and the reduction of dP = dO V^T; each operand is TMA boxes of its own
// swizzle width.  Every existing instantiation is DQK == DV == d.
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
//                               dP = dO V^T, forms dS from one tanh and accumulates dQ += dS K in registers.  Its prologue,
//                               K / V ring and mask cases are the forward's (attn_wgmma_qtile.cuh).
// Every dq / dk / dv element is then summed by one thread in a fixed order, so the result is bitwise reproducible.
// At d = 32 recomputing S and dP costs two MMA units per score against the eight that the whole backward issues, while the
// elementwise work per score is the same; at larger d the recomputed MMAs weigh more and the fused kernel stays the default.
// The split kernels run two CTAs per SM at d = 32 and one at d = 64 / 128 / 256 (their accumulators need more than 128
// registers per thread there); bf16 at d >= 64 keeps the hi + lo operand pairs.
// d = 256 always runs the split kernels (a fused dQ accumulator would be L * H * 1 KB of fp32), except that a deterministic
// backward there stays on the generic kernels.  Full-width dK + dV would take 256 registers per thread, so two CTAs share
// each key tile, one 128-column half of dK / dV each (bwd_key_tile's DN), and both compute S^T / dP^T over all 256 columns;
// with K and V taking 128 KB, the query tiles are 32 rows in a 3-stage ring.  The dQ kernel keeps the full width on 32-key
// tiles (3 stages).
//
// Reference math: ops/triton/triton_hstu_attention.py:995-1006,1222 and SURVEY.md appendix A; unlike the Triton
// kernel dQ is accumulated in fp32, not in the input dtype (triton_attention_utils.py:47-60).
#pragma once
#include <string.h>

#include <algorithm>
#include <type_traits>

#include "attn_fp16_operands.cuh"
#include "attn_wgmma_qtile.cuh"
#include "common.cuh"
#include "internal.h"
#include "wgmma.cuh"

namespace hstu {
using namespace wg;

struct alignas(64) BwdParams {
  CUtensorMap tmQ, tmK, tmV, tmDO;
  SeqArgs seq;
  void* dk;
  void* dv;
  float* dq_acc;  // [L, H, DQK] fp32, zero-initialised (fused kernel)
  void* dq;       // attn_bwd_dq_wgmma_kernel
  long long dk_row_stride, dk_head_stride, dv_row_stride, dv_head_stride, dq_row_stride, dq_head_stride;
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
    c_s = p.seq.alpha_half;
    if (p.amax == nullptr) return;
    const OperandExps ex = operand_exps(p.amax + ((long long)b * p.seq.heads + h) * kAmaxSlots, 2.f * p.seq.alpha_half, d);
    c_s = ldexpf(p.seq.alpha_half, -(ex.q + ex.k));
    c_p = pow2f(ex.p);
    c_d = pow2f(ex.s - ex.v - ex.o);
    e_dv = -(ex.p + ex.o);
    e_dk = -(ex.s + ex.q);
    e_dq = -(ex.s + ex.k);
  }
};

// CTAs per SM of the split kernels: two at dv = 32 (<= 128 registers per thread), one at dv = 64 / 128 / 256
constexpr int split_min_blocks(int dv) { return dv == 32 ? 2 : 1; }
constexpr int kSmemPerSm = 232448;  // dynamic shared memory one CTA may use on sm_90
// CTAs of the dK / dV kernel per key tile (column slices): one, except at dv = 256, where the dV accumulator alone is 128
// registers per thread (and 64 + 64 fp32 accumulators of d = 256 would take 256); there two CTAs per key tile take one half
// of the dK and of the dV columns each
__host__ __device__ constexpr int dkdv_slices(int dv) { return dv == 256 ? 2 : 1; }
__host__ __device__ constexpr int imax(int a, int b) { return a > b ? a : b; }

// FUSED_DQ: the key-tile kernel also computes dQ (dS buffers in shared memory); without it the layout ends after the ring,
// which then has four stages (d = 128: 192 KB, one CTA per SM), or at d = 256, where K and V alone take 128 KB, three
// stages of 32 query rows (224 KB).  The dqk < dv pairs all have four (at most 192 KB, at (128, 256)).
// Swizzle widths: SW of K, SWQ of the Q_j stages, SWV of V and dO_j.  A slice's dK columns must be whole Q_j boxes (the
// B operand of dK += dS^T Q_j starts at a box), so Q_j takes the swizzle of DQK / NSL columns: narrower than K's at
// dqk <= 64 with dv = 256 (32 or 16 columns), the same everywhere else.
template <int DQK, int DV, bool FUSED_DQ>
struct BwdCfg {
  static_assert(DQK <= DV && (DQK == DV || !FUSED_DQ), "dqk < dv runs the split kernels only");
  static constexpr int NSL = FUSED_DQ ? 1 : dkdv_slices(DV);  // CTAs (column slices) per key tile
  static constexpr int BKV = 128;
  static constexpr int BQ = DV == 256 ? 32 : 64;  // query rows per streamed tile
  static constexpr int SW = swizzle_bytes(DQK), SWQ = swizzle_bytes(DQK / NSL), SWV = swizzle_bytes(DV);
  static constexpr int BOX_COLS = SW / 2, BOX_COLS_Q = SWQ / 2, BOX_COLS_V = SWV / 2;
  static constexpr int NBOX = DQK / BOX_COLS, NBOX_Q = DQK / BOX_COLS_Q, NBOX_V = DV / BOX_COLS_V;
  static constexpr int K_BOX = BKV * SW, V_BOX = BKV * SWV;
  static constexpr int Q_BOX = BQ * SWQ, DO_BOX = BQ * SWV;
  static constexpr int K_BYTES = BKV * DQK * 2, V_BYTES = BKV * DV * 2;
  static constexpr int Q_BYTES = BQ * DQK * 2, DO_BYTES = BQ * DV * 2;
  // Q_j / dO_j ring depth
  static constexpr int STAGES = DQK != DV ? 4 : DQK == 256 ? 3 : (DQK <= 32 || !FUSED_DQ) ? 4 : (DQK == 64 ? 3 : 2);
  static constexpr int DS_BYTES = BKV * BQ * 2;                      // one [128 kv][64 q] box, 128-byte swizzle
  static constexpr int DQN = DQK < 64 ? DQK : 64;                    // dQ columns per pass (one 128-byte box of K)
  static constexpr int OFF_K = 0;
  static constexpr int OFF_V = OFF_K + K_BYTES;
  static constexpr int OFF_Q = OFF_V + V_BYTES;
  static constexpr int OFF_DO = OFF_Q + STAGES * Q_BYTES;
  static constexpr int OFF_DS = OFF_DO + STAGES * DO_BYTES;          // [buffer 0/1][hi / lo]
  static constexpr int OFF_BAR = OFF_DS + (FUSED_DQ ? 4 * DS_BYTES : 0);
  static constexpr int SMEM_BYTES = OFF_BAR + 256 + 1024;
  static_assert(SMEM_BYTES * (FUSED_DQ ? 1 : split_min_blocks(DV)) <= kSmemPerSm, "shared memory budget");
  static_assert(STAGES <= 4, "BwdBars holds four stages");
};

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
// sequence end).  With Cfg::NSL > 1 slices, NSL CTAs share a key tile: CTA x takes key tile x / NSL, dK columns
// [ck0, ck0 + DQK / NSL) and dV columns [cv0, cv0 + DV / NSL), ck0 = DQK / NSL (x % NSL) and cv0 likewise; its S^T / dP^T MMAs
// still reduce over all DQK / DV columns.
// kBidir: the non-causal mask (attn_wgmma_bidir.cu; split kernels only): the query range of q_range_for_kv_rows_bidir and
// its mask cases, nothing else.
template <int DQK, int DV, bool BF16, bool FUSED_DQ, bool kBidir = false>
__device__ __forceinline__ void bwd_key_tile(const BwdParams& p) {
  static_assert(!(FUSED_DQ && kBidir), "the non-causal backward runs the split kernels");
  using Cfg = BwdCfg<DQK, DV, FUSED_DQ>;
  constexpr int SW = Cfg::SW, SWQ = Cfg::SWQ, SWV = Cfg::SWV, BQ = Cfg::BQ, NST = Cfg::STAGES;
  constexpr int NSL = Cfg::NSL, DNK = DQK / NSL, DNV = DV / NSL;  // column slices per key tile, and their widths
  static_assert(DNK % Cfg::BOX_COLS_Q == 0 && DNV % Cfg::BOX_COLS_V == 0, "a slice is whole boxes");
  const int b = blockIdx.z, h = blockIdx.y;
  const int n0 = (blockIdx.x / NSL) * Cfg::BKV;
  const int ck0 = (blockIdx.x % NSL) * DNK, cv0 = (blockIdx.x % NSL) * DNV;
  const long long row0 = load_index(p.seq.seq_offsets, p.seq.offsets_i64, b);
  int len = (int)(load_index(p.seq.seq_offsets, p.seq.offsets_i64, b + 1) - row0);
  if (len > p.seq.max_seq_len) {  // rows past max_seq_len get zero gradients
    if (blockIdx.x == 0) {
      zero_rows(p.dk, 2, p.dk_row_stride, (long long)h * p.dk_head_stride, DQK, row0 + p.seq.max_seq_len, row0 + len);
      zero_rows(p.dv, 2, p.dv_row_stride, (long long)h * p.dv_head_stride, DV, row0 + p.seq.max_seq_len, row0 + len);
    }
    len = p.seq.max_seq_len;
  }
  if (n0 >= len) return;
  const int n_tgt = p.seq.num_targets ? (int)load_index(p.seq.num_targets, p.seq.targets_i64, b) : -1;
  const SeqMask msk = make_seq_mask(len, n_tgt, p.seq.win, p.seq.min_full, p.seq.ctx);
  const int nrows = min(Cfg::BKV, len - n0);
  QTiles qt;
  {
    int lo, hi, ctx_hi;
    if constexpr (kBidir) q_range_for_kv_rows_bidir(msk, n0, n0 + nrows, &lo, &hi, &ctx_hi);
    else q_range_for_kv_rows(msk, n0, n0 + nrows, &lo, &hi, &ctx_hi);
    qt.A = (ctx_hi + BQ - 1) / BQ;
    qt.first = max(lo / BQ, qt.A);
    qt.T = qt.A + max(0, (hi + BQ - 1) / BQ - qt.first);
  }

  uint8_t* smem = dyn_smem_1k();
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
    mbar_arrive_expect_tx(&bars->qd_full[st], Cfg::Q_BYTES + Cfg::DO_BYTES);
#pragma unroll
    for (int bx = 0; bx < imax(Cfg::NBOX_Q, Cfg::NBOX_V); ++bx) {
      if (bx < Cfg::NBOX_Q)
        tma_load_3d(smem + Cfg::OFF_Q + st * Cfg::Q_BYTES + bx * Cfg::Q_BOX, &p.tmQ, &bars->qd_full[st], bx * Cfg::BOX_COLS_Q, h, q_row);
      if (bx < Cfg::NBOX_V)
        tma_load_3d(smem + Cfg::OFF_DO + st * Cfg::DO_BYTES + bx * Cfg::DO_BOX, &p.tmDO, &bars->qd_full[st], bx * Cfg::BOX_COLS_V, h, q_row);
    }
  };
  if (tid == 0) {
    prefetch_tensormap(&p.tmQ);
    prefetch_tensormap(&p.tmK);
    prefetch_tensormap(&p.tmV);
    prefetch_tensormap(&p.tmDO);
    mbar_arrive_expect_tx(&bars->kv_full, Cfg::K_BYTES + Cfg::V_BYTES);
#pragma unroll
    for (int bx = 0; bx < imax(Cfg::NBOX, Cfg::NBOX_V); ++bx) {
      if (bx < Cfg::NBOX) tma_load_3d(smem + Cfg::OFF_K + bx * Cfg::K_BOX, &p.tmK, &bars->kv_full, bx * Cfg::BOX_COLS, h, (int)(row0 + n0));
      if (bx < Cfg::NBOX_V) tma_load_3d(smem + Cfg::OFF_V + bx * Cfg::V_BOX, &p.tmV, &bars->kv_full, bx * Cfg::BOX_COLS_V, h, (int)(row0 + n0));
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
  // Q_j columns [ck0, ck0 + DNK) and dO_j columns [cv0, cv0 + DNV) as B of dK / dV: whole boxes
  const uint32_t sq_c = sq + ck0 / Cfg::BOX_COLS_Q * Cfg::Q_BOX, sdo_c = sdo + cv0 / Cfg::BOX_COLS_V * Cfg::DO_BOX;
  const bool fast = msk.fast != 0;
  // keys of this tile that every query row >= q_full_from may attend (fast mask): all of them are history keys below the row
  const bool keys_hist = !msk.has_tgt || n0 + Cfg::BKV <= msk.max_id;

  // the d = 32 dK / dV kernel also runs bf16 inputs on fp16 copies
  constexpr bool kScaled = !BF16 && !FUSED_DQ && DQK == 32 && DV == 32;
  const BwdScales sc(p, b, h, DQK);
  constexpr int KQ = BQ / 16;  // k16 slices of a query tile (A fragments of P^T / dS^T)
  float dv[DNV / 2], dk[DNK / 2];
#pragma unroll
  for (int e = 0; e < imax(DNV, DNK) / 2; ++e) {
    if (e < DNV / 2) dv[e] = 0.f;
    if (e < DNK / 2) dk[e] = 0.f;
  }
  uint32_t pf_hi[KQ][4], pf_lo[KQ][4], df_hi[KQ][4], df_lo[KQ][4];
#pragma unroll
  for (int kk = 0; kk < KQ; ++kk)
#pragma unroll
    for (int r = 0; r < 4; ++r) pf_hi[kk][r] = pf_lo[kk][r] = df_hi[kk][r] = df_lo[kk][r] = 0u;

  mbar_wait(&bars->kv_full, 0);
  // K rows >= len of a key tile that crosses the sequence end are B of dQ = dS K (dS is 0 there, K may be NaN)
  if (FUSED_DQ && n0 + Cfg::BKV > len)  // CTA-uniform; K is loaded once
    zero_tile_rows_sync<Cfg::BKV, SW, Cfg::NBOX, kAttnThreads>(smem + Cfg::OFF_K, len - n0);
  for (int j = 0; j < qt.T; ++j) {
    const int st = j % NST;
    const uint32_t ph = (j / NST) & 1;
    const int q0 = qt.at(j) * BQ;
    mbar_wait(&bars->qd_full[st], ph);
    // Q_j / dO_j rows >= len are B of dK += dS^T Q_j and dV += P^T dO_j (P and dS are 0 there, Q / dO may be NaN).  The query
    // tile that crosses the sequence end is the last one of the key tile (hi <= len, ctx_hi <= len), so its stage is not
    // refilled after the zeroing.
    if (q0 + BQ > len) {  // CTA-uniform
      zero_tile_rows<BQ, SWQ, Cfg::NBOX_Q, kAttnThreads>(smem + Cfg::OFF_Q + st * Cfg::Q_BYTES, len - q0);
      zero_tile_rows_sync<BQ, SWV, Cfg::NBOX_V, kAttnThreads>(smem + Cfg::OFF_DO + st * Cfg::DO_BYTES, len - q0);
    }
    float s[BQ / 2], dp[BQ / 2];
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < DQK / 16; ++ks) {
      const int kb = ks * 32, bx = kb / SW, off = kb % SW, bq = kb / SWQ, offq = kb % SWQ;
      const uint32_t ka = sk + bx * Cfg::K_BOX + wgi * 64 * SW;
      wgmma_ss<BQ, BF16, 0, 0>(s, desc_kmajor<SW>(ka, off), desc_kmajor<SWQ>(sq + st * Cfg::Q_BYTES + bq * Cfg::Q_BOX, offq), ks > 0);
    }
#pragma unroll
    for (int ks = 0; ks < DV / 16; ++ks) {
      const int kb = ks * 32, bx = kb / SWV, off = kb % SWV;
      const uint32_t va = sv + bx * Cfg::V_BOX + wgi * 64 * SWV;
      wgmma_ss<BQ, BF16, 0, 0>(dp, desc_kmajor<SWV>(va, off), desc_kmajor<SWV>(sdo + st * Cfg::DO_BYTES + bx * Cfg::DO_BOX, off), ks > 0);
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(s);
    fence_regs(dp);

    // p = x sig(x) and 2 dS = dP (1 + g2) from one tanh (h = alpha s / 2, t = tanh h, p = h (1 + t), g2 = t + h (1 - t^2)).
    // The mask case is chosen once per tile, outside the score loops, so that ptxas can overlap the tanh of independent
    // scores (as in the forward).  `v`: the pair is valid.
    auto score = [&](int n, bool v) {
      const float x = s[n] * (kScaled ? sc.c_s : p.seq.alpha_half), xp = kScaled ? x * sc.c_p : x;
      const float t = tanh_approx(x);
      const float g2 = __fmaf_rn(x, __fmaf_rn(-t, t, 1.f), t);
      const float pv = __fmaf_rn(xp, t, xp);
      float dsv = __fmaf_rn(dp[n], g2, dp[n]);
      if (kScaled) dsv *= sc.c_d;
      s[n] = v ? pv : 0.f;
      dp[n] = v ? dsv : 0.f;
    };
    if constexpr (kBidir) {
      // the cases of mask_scores_bidir (attn_wgmma_qtile.cuh), here with the key rows fixed and the query tile streamed
      if (n0 + Cfg::BKV <= len && q0 + BQ <= len && bidir_block_all_valid(msk, q0, q0 + BQ, n0, n0 + Cfg::BKV)) {
#pragma unroll
        for (int n = 0; n < BQ / 2; ++n) score(n, true);
      } else if (msk.win == 0 && msk.max_id >= 1) {
        const int t_first = target_start(msk);
#pragma unroll
        for (int nb = 0; nb < BQ / 8; ++nb)
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int kj = k_base + (e >> 1) * 8, qi = q0 + nb * 8 + 2 * t4 + (e & 1);
            score(nb * 4 + e, kj < len && qi < len && (qi < t_first || kj < t_first || kj == qi));
          }
      } else {
#pragma unroll
        for (int nb = 0; nb < BQ / 8; ++nb)
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int kj = k_base + (e >> 1) * 8, qi = q0 + nb * 8 + 2 * t4 + (e & 1);
            score(nb * 4 + e, kj < len && qi < len && mask_valid_bidir(msk, qi, kj));
          }
      }
    } else if (fast && keys_hist && n0 + Cfg::BKV <= q0 && q0 + BQ <= len) {  // tile-uniform: every pair valid
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
        const uint64_t dod = desc_mnmajor<SWV>(sdo + st * Cfg::DO_BYTES, kk * 16, Cfg::DO_BOX);
        const uint64_t qd = desc_mnmajor<SWQ>(sq + st * Cfg::Q_BYTES, kk * 16, Cfg::Q_BOX);
        wgmma_rs<DV, BF16, 1>(dv, pf_hi[kk], dod, 1);
        wgmma_rs<DQK, BF16, 1>(dk, df_hi[kk], qd, 1);
        if constexpr (BF16) {
          wgmma_rs<DV, BF16, 1>(dv, pf_lo[kk], dod, 1);
          wgmma_rs<DQK, BF16, 1>(dk, df_lo[kk], qd, 1);
        }
      }
    } else {
      // dV += P^T dO_j issued as soon as P is packed, then dK += dS^T Q_j: P^T and dS^T are never both held in fp32 next to
      // both fragment sets, which keeps a bf16 thread at 128 registers without wgmma serialisation (ptxas C7512)
#pragma unroll
      for (int kk = 0; kk < KQ; ++kk)
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          const Operand<BF16> pp(s[8 * kk + 2 * r], s[8 * kk + 2 * r + 1]);
          pf_hi[kk][r] = pp.hi; pf_lo[kk][r] = pp.lo;
        }
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < KQ; ++kk) {
        const uint64_t dod = desc_mnmajor<SWV>(sdo_c + st * Cfg::DO_BYTES, kk * 16, Cfg::DO_BOX);
        wgmma_rs<DNV, BF16, 1>(dv, pf_hi[kk], dod, 1);
        if constexpr (BF16) wgmma_rs<DNV, BF16, 1>(dv, pf_lo[kk], dod, 1);
      }
      wgmma_commit();
#pragma unroll
      for (int kk = 0; kk < KQ; ++kk)
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          const Operand<BF16> dd(dp[8 * kk + 2 * r], dp[8 * kk + 2 * r + 1]);
          df_hi[kk][r] = dd.hi; df_lo[kk][r] = dd.lo;
        }
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < KQ; ++kk) {
        const uint64_t qd = desc_mnmajor<SWQ>(sq_c + st * Cfg::Q_BYTES, kk * 16, Cfg::Q_BOX);
        wgmma_rs<DNK, BF16, 1>(dk, df_hi[kk], qd, 1);
        if constexpr (BF16) wgmma_rs<DNK, BF16, 1>(dk, df_lo[kk], qd, 1);
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
    if (lane == 0 && j + NST < qt.T && release_is_last<kAttnThreads / 32>(&bars->qd_free[st])) load_qd(j + NST);
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
      for (int pass = 0; pass < DQK / Cfg::DQN; ++pass) {
        float dq[Cfg::DQN / 2];
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < Cfg::BKV / 16; ++kk) {
          const uint64_t kd = desc_mnmajor<SW>(sk + pass * Cfg::K_BOX, kk * 16, Cfg::K_BOX);
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
            float* dst = p.dq_acc + ((row0 + qi) * p.seq.heads + h) * DQK + pass * Cfg::DQN + 2 * t4;
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
      uint16_t* krow = reinterpret_cast<uint16_t*>(p.dk) + (row0 + kj) * p.dk_row_stride + (long long)h * p.dk_head_stride + ck0 + 2 * t4;
      uint16_t* vrow = reinterpret_cast<uint16_t*>(p.dv) + (row0 + kj) * p.dv_row_stride + (long long)h * p.dv_head_stride + cv0 + 2 * t4;
      // (DNK < DNV: the first DNK / 8 column blocks carry dK too)
#pragma unroll
      for (int nb = 0; nb < DNV / 8; ++nb) {
        const bool has_k = nb < DNK / 8;
        const int nk = has_k ? nb : 0;
        float k0 = dk[nk * 4 + hh * 2] * p.dk_scale, k1 = dk[nk * 4 + hh * 2 + 1] * p.dk_scale;
        float v0 = dv[nb * 4 + hh * 2] * p.dv_scale, v1 = dv[nb * 4 + hh * 2 + 1] * p.dv_scale;
        if (kScaled) {
          k0 = scalbnf(k0, sc.e_dk), k1 = scalbnf(k1, sc.e_dk);
          v0 = scalbnf(v0, sc.e_dv), v1 = scalbnf(v1, sc.e_dv);
        }
        const bool out_bf16 = BF16 || p.amax != nullptr;
        if (has_k) *reinterpret_cast<uint32_t*>(krow + nb * 8) = out_bf16 ? pack_bf16x2(k0, k1) : pack_f16x2(k0, k1);
        *reinterpret_cast<uint32_t*>(vrow + nb * 8) = out_bf16 ? pack_bf16x2(v0, v1) : pack_f16x2(v0, v1);
      }
    }
  }
}

// ---------------- dQ, query-stationary (split path) ----------------
template <int DQK, int DV>
struct DqCfg {
  static constexpr int BM = 128;  // query rows per CTA (two warpgroups of 64)
  // key rows per tile: 64, unless Q and dO leave no room for three stages of 64 keys -- d = 256 (Q and dO take 128 KB) and
  // (128, 256) (96 KB) -- which run three stages of 32 keys with the full-width dQ accumulator
  static constexpr int BN = DQK + DV >= 384 ? 32 : 64;
  static constexpr int SW = swizzle_bytes(DQK), SWV = swizzle_bytes(DV);  // Q / K, and dO / V
  static constexpr int BOX_COLS = SW / 2, BOX_COLS_V = SWV / 2;
  static constexpr int NBOX = DQK / BOX_COLS, NBOX_V = DV / BOX_COLS_V;
  static constexpr int Q_BOX = BM * SW, DO_BOX = BM * SWV;
  static constexpr int K_BOX = BN * SW, V_BOX = BN * SWV;
  static constexpr int Q_BYTES = BM * DQK * 2, DO_BYTES = BM * DV * 2;
  static constexpr int K_BYTES = BN * DQK * 2, V_BYTES = BN * DV * 2;
  static constexpr int STAGES = 3;  // K / V ring depth (d = 128: 161 KB, d = 256: 225 KB, (64, 256): 201 KB, one CTA per SM)
  static constexpr int OFF_Q = 0;
  static constexpr int OFF_DO = OFF_Q + Q_BYTES;
  static constexpr int OFF_K = OFF_DO + DO_BYTES;
  static constexpr int OFF_V = OFF_K + STAGES * K_BYTES;
  static constexpr int OFF_BAR = OFF_V + STAGES * V_BYTES;
  static constexpr int SMEM_BYTES = OFF_BAR + 256 + 1024;
  static_assert(SMEM_BYTES * split_min_blocks(DV) <= kSmemPerSm, "shared memory budget of split_min_blocks(dv) CTAs per SM");
};

// One CTA per (128-row query tile, head, sequence), heavy (late) tiles first; the forward's schedule, tile ranges and ring
// (attn_wgmma_qtile.cuh).
// Per 64-key tile each warpgroup runs S = Q K^T and dP = dO V^T (A and B K-major), releases V, forms
// 2 dS N / alpha = dP (1 + g2) * mask from one tanh, and runs dQ += dS K (A from registers, K read MN-major), then releases K.
// Q, K and dQ are DQK wide, dO and V DV wide.
// kBidir: the non-causal mask (attn_wgmma_bidir.cu): the key range and mask cases of the non-causal forward, nothing else.
template <int DQK, int DV, bool BF16, bool kBidir = false>
__device__ __forceinline__ void bwd_dq_body(const BwdParams& p) {
  using Cfg = DqCfg<DQK, DV>;
  constexpr int SW = Cfg::SW, SWV = Cfg::SWV, BN = Cfg::BN, NST = Cfg::STAGES;
  constexpr bool kScaled = !BF16 && DQK == 32 && DV == 32;  // also runs bf16 inputs on scaled fp16 copies
  const int b = blockIdx.z, h = blockIdx.y;
  const int m0 = (int)(gridDim.x - 1 - blockIdx.x) * Cfg::BM;
  QTileSeq qs;  // (rows past max_seq_len get zero gradients)
  if (!qtile_prologue<Cfg::BM, BN, kBidir>(p.seq, b, h, m0, p.dq, p.dq_row_stride, p.dq_head_stride, DQK, &qs)) return;

  uint8_t* smem = dyn_smem_1k();
  // V of tile i is released once the warp's S / dP MMAs have completed, K once its dQ MMAs have
  KvRing<Cfg> ring{smem, &p.tmK, &p.tmV, h, qs.row0, qs.t0, qs.T};
  ring.init();
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (tid == 0) {
    prefetch_tensormap(&p.tmQ);
    prefetch_tensormap(&p.tmK);
    prefetch_tensormap(&p.tmV);
    prefetch_tensormap(&p.tmDO);
    mbar_arrive_expect_tx(&ring.bars->q_full, Cfg::Q_BYTES + Cfg::DO_BYTES);
#pragma unroll
    for (int bx = 0; bx < imax(Cfg::NBOX, Cfg::NBOX_V); ++bx) {
      if (bx < Cfg::NBOX) tma_load_3d(smem + Cfg::OFF_Q + bx * Cfg::Q_BOX, &p.tmQ, &ring.bars->q_full, bx * Cfg::BOX_COLS, h, (int)(qs.row0 + m0));
      if (bx < Cfg::NBOX_V)
        tma_load_3d(smem + Cfg::OFF_DO + bx * Cfg::DO_BOX, &p.tmDO, &ring.bars->q_full, bx * Cfg::BOX_COLS_V, h, (int)(qs.row0 + m0));
    }
    ring.fill();
  }
  __syncwarp();

  const int wgi = warpgroup_index(), w = warp & 3, g = lane >> 2, t4 = lane & 3;
  const int q_base = m0 + wgi * 64 + w * 16 + g;  // query position of accumulator rows g (+ 8)
  // wgmma descriptors, built once (warp-uniform): Q and dO of the warpgroup, K / V of ring stage 0 K-major (S, dP) and K
  // MN-major (dQ); the rest are constant steps from them (desc_add, desc_stage)
  const uint64_t dq0 = desc_pin(desc_kmajor<SW>(smem_u32(smem + Cfg::OFF_Q) + wgi * 64 * SW, 0));
  const uint64_t ddo0 = desc_pin(desc_kmajor<SWV>(smem_u32(smem + Cfg::OFF_DO) + wgi * 64 * SWV, 0));
  const uint64_t dk0 = desc_pin(desc_kmajor<SW>(smem_u32(smem + Cfg::OFF_K), 0));
  const uint64_t dv0 = desc_pin(desc_kmajor<SWV>(smem_u32(smem + Cfg::OFF_V), 0));
  const uint64_t dkn0 = desc_pin(desc_mnmajor<SW>(smem_u32(smem + Cfg::OFF_K), 0, Cfg::K_BOX));
  const bool fast = qs.msk.fast != 0;
  const int full_lim = full_valid_limit(qs.msk, m0);

  const BwdScales sc(p, b, h, DQK);
  float dq[DQK / 2];
#pragma unroll
  for (int e = 0; e < DQK / 2; ++e) dq[e] = 0.f;
  uint32_t a_hi[BN / 16][4], a_lo[BN / 16][4];
#pragma unroll
  for (int kk = 0; kk < BN / 16; ++kk)
#pragma unroll
    for (int r = 0; r < 4; ++r) a_hi[kk][r] = a_lo[kk][r] = 0u;
  // One wait per MMA batch: S and dP of tile i + 1 in the batch of dQ += dS_i K_i would hold S, dP, dQ and both dS fragment
  // sets at once, which does not fit in 128 registers with bf16 inputs (ptxas spills and serialises the MMAs).
  mbar_wait(&ring.bars->q_full, 0);
  // The last tile (kLast) is peeled off the loop: it is the only one that can cross the sequence end (its key range ends at
  // hi <= len), so the loop itself does not test for it.
  RingPos<NST> cur;  // ring stage and phase parity of tile i
  auto tile = [&](int i, auto last_c) {
    constexpr bool kLast = decltype(last_c)::value;
    const int st = cur.st;
    const int n0 = (qs.t0 + i) * BN;
    float s[BN / 2], dp[BN / 2];
    ring.wait(kKey, st, cur.ph);
    ring.wait(kVal, st, cur.ph);
    // the last key tile may cross the sequence end: its K rows >= len are B of dQ += dS K (dS is 0 there, K may be NaN)
    if (kLast && n0 + BN > qs.len)  // CTA-uniform; the last tile, so its stage is not refilled
      zero_tile_rows_sync<BN, SW, Cfg::NBOX, kAttnThreads>(smem + Cfg::OFF_K + st * Cfg::K_BYTES, qs.len - n0);
    wgmma_fence();
    const uint64_t kd = desc_stage(dk0, st, Cfg::K_BYTES), vd = desc_stage(dv0, st, Cfg::V_BYTES);
#pragma unroll
    for (int ks = 0; ks < DQK / 16; ++ks) {
      const int kb = ks * 32, bx = kb / SW, off = kb % SW;
      wgmma_ss<BN, BF16, 0, 0>(s, desc_add(dq0, bx * Cfg::Q_BOX + off), desc_add(kd, bx * Cfg::K_BOX + off), ks > 0);
    }
#pragma unroll
    for (int ks = 0; ks < DV / 16; ++ks) {
      const int kb = ks * 32, bx = kb / SWV, off = kb % SWV;
      wgmma_ss<BN, BF16, 0, 0>(dp, desc_add(ddo0, bx * Cfg::DO_BOX + off), desc_add(vd, bx * Cfg::V_BOX + off), ks > 0);
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(s);
    fence_regs(dp);
    ring.release(kVal, i, st);
    __syncwarp();

    // 2 dS N / alpha = dP (1 + g2), g2 = t + h (1 - t^2), t = tanh h, h = alpha s / 2
    auto dscore = [&](int n) {
      const float x = s[n] * sc.c_s;
      const float t = tanh_approx(x);
      const float g2 = __fmaf_rn(x, __fmaf_rn(-t, t, 1.f), t);
      float dsv = __fmaf_rn(dp[n], g2, dp[n]);
      if (kScaled) dsv *= sc.c_d;
      return dsv;
    };
    if constexpr (kBidir) mask_scores_bidir<BN>(qs.msk, qs.len, m0, m0 + qs.mrows, q_base, n0, t4, dp, dscore);
    else mask_scores<BN>(qs.msk, fast, full_lim, qs.len, q_base, n0, t4, dp, dscore);
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
    const uint64_t kn = desc_stage(dkn0, st, Cfg::K_BYTES);
#pragma unroll
    for (int kk = 0; kk < BN / 16; ++kk) {
      wgmma_rs<DQK, BF16, 1>(dq, a_hi[kk], desc_add(kn, kk * 16 * SW), 1);
      if constexpr (BF16) wgmma_rs<DQK, BF16, 1>(dq, a_lo[kk], desc_add(kn, kk * 16 * SW), 1);
    }
    wgmma_commit();
    wgmma_wait<0>();  // an MMA batch never stays in flight across the elementwise code (ptxas would serialise them)
    fence_regs(dq);
    fence_regs(a_hi);
    fence_regs(a_lo);
    ring.release(kKey, i, st);
    __syncwarp();
    cur.advance();
  };
  for (int i = 0; i < qs.T - 1; ++i) tile(i, std::false_type{});
  tile(qs.T - 1, std::true_type{});

  // ---------------- epilogue: dQ * alpha / (2N) -> global ----------------
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int qi = q_base + hh * 8;
    if (qi - m0 < qs.mrows) {
      uint16_t* qrow = reinterpret_cast<uint16_t*>(p.dq) + (qs.row0 + qi) * p.dq_row_stride + (long long)h * p.dq_head_stride;
#pragma unroll
      for (int nb = 0; nb < DQK / 8; ++nb) {
        float a = dq[nb * 4 + hh * 2] * p.dk_scale, c = dq[nb * 4 + hh * 2 + 1] * p.dk_scale;
        if (kScaled) a = scalbnf(a, sc.e_dq), c = scalbnf(c, sc.e_dq);
        *reinterpret_cast<uint32_t*>(qrow + nb * 8 + 2 * t4) = (BF16 || p.amax != nullptr) ? pack_bf16x2(a, c) : pack_f16x2(a, c);
      }
    }
  }
}


// ------------------------------------------------------------------------------------------------
// host
// ------------------------------------------------------------------------------------------------
// The BwdParams of a call without its tensor maps; f16: the scaled fp16 copies of bf16 inputs, or null
inline BwdParams bwd_params(const hstu_attn_params& p, const Fp16Operands* f16) {
  BwdParams bp;
  memset(&bp, 0, sizeof(bp));
  if (f16) bp.amax = f16->amax;
  bp.seq = seq_args(p);
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
  bp.dv_scale = 1.0f / (float)p.max_seq_len;
  bp.dk_scale = 0.5f * p.alpha / (float)p.max_seq_len;
  return bp;
}

// The tensor maps of q, k, v, dO for one kernel: q in boxes of q_cols x q_rows, k in k_cols x kv_rows, v in v_cols x kv_rows,
// dO in v_cols x q_rows
template <int DQK, int DV>
int bwd_tmaps(BwdParams& bp, const hstu_attn_params& p, const Operands& o, int q_cols, int k_cols, int v_cols, int q_rows, int kv_rows) {
  if (int e = make_tmap_rows_heads(&bp.tmQ, o.src[0], p.total_rows, p.heads, DQK, o.rs[0], o.hs[0], q_cols, q_rows)) return e;
  if (int e = make_tmap_rows_heads(&bp.tmK, o.src[1], p.total_rows, p.heads, DQK, o.rs[1], o.hs[1], k_cols, kv_rows)) return e;
  if (int e = make_tmap_rows_heads(&bp.tmV, o.src[2], p.total_rows, p.heads, DV, o.rs[2], o.hs[2], v_cols, kv_rows)) return e;
  return make_tmap_rows_heads(&bp.tmDO, o.src[3], p.total_rows, p.heads, DV, o.rs[3], o.hs[3], v_cols, q_rows);
}

// The fused backward at dqk == dv == D: kern (an instance of bwd_key_tile<D, D, BF16, true>) adds dQ into the fp32
// accumulator in the workspace, and convert (dq_convert_kernel<BF16>) scales it into dq
template <int D>
int launch_bwd_fused(const hstu_attn_params& p, cudaStream_t st, void (*kern)(BwdParams),
                     void (*convert)(const float*, uint16_t*, long long, int, int, long long, long long, float)) {
  using Cfg = BwdCfg<D, D, true>;
  const size_t need = wgmma_workspace_bytes(p, true, false);
  if (p.workspace == nullptr || p.workspace_bytes < need) {
    set_error("hstu_attn_bwd: workspace of %zu bytes required (got %zu)", need, p.workspace_bytes);
    return HSTU_ERR_WORKSPACE;
  }
  BwdParams bp = bwd_params(p, nullptr);
  if (int e = bwd_tmaps<D, D>(bp, p, operands(p, nullptr), Cfg::BOX_COLS, Cfg::BOX_COLS, Cfg::BOX_COLS, Cfg::BQ, Cfg::BKV)) return e;
  HSTU_CUDA_OK(cudaMemsetAsync(p.workspace, 0, need, st));
  HSTU_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
  dim3 grid((p.max_seq_len + Cfg::BKV - 1) / Cfg::BKV, p.heads, p.batch);
  kern<<<grid, kAttnThreads, Cfg::SMEM_BYTES, st>>>(bp);
  HSTU_CUDA_OK(cudaGetLastError());
  const long long nvec = p.total_rows * p.heads * (D / 8);
  const long long blocks = std::min<long long>((nvec + 255) / 256, kH100Sms * 16);
  convert<<<(int)blocks, 256, 0, st>>>(bp.dq_acc, reinterpret_cast<uint16_t*>(p.dq), p.total_rows, p.heads, D, p.dq_row_stride,
                                       p.dq_head_stride, bp.dk_scale);
  HSTU_CUDA_OK(cudaGetLastError());
  return 0;
}

// The split backward: kdkdv (an instance of bwd_key_tile<DQK, DV, BF16, false>), then kdq (of bwd_dq_body<DQK, DV, BF16>);
// no atomics and no workspace.  f16: the scaled fp16 copies of bf16 inputs (the kernels are then the fp16 ones), or null
template <int DQK, int DV, bool BF16>
int launch_bwd_split(const hstu_attn_params& p, cudaStream_t st, void (*kdkdv)(BwdParams), void (*kdq)(BwdParams),
                     const Fp16Operands* f16 = nullptr) {
  using Cfg = BwdCfg<DQK, DV, false>;
  const Operands o = operands(p, f16);
  BwdParams bp = bwd_params(p, f16);
  // the dK / dV kernel: K and V of a 128-row key tile, streamed Q_j / dO_j tiles
  if (int e = bwd_tmaps<DQK, DV>(bp, p, o, Cfg::BOX_COLS_Q, Cfg::BOX_COLS, Cfg::BOX_COLS_V, Cfg::BQ, Cfg::BKV)) return e;
  HSTU_CUDA_OK(cudaFuncSetAttribute(kdkdv, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
  // the column slices of one key tile are adjacent CTAs (they read the same K, V and query tiles)
  const int key_ctas = (p.max_seq_len + Cfg::BKV - 1) / Cfg::BKV * Cfg::NSL;
  kdkdv<<<dim3(key_ctas, p.heads, p.batch), kAttnThreads, Cfg::SMEM_BYTES, st>>>(bp);
  HSTU_CUDA_OK(cudaGetLastError());
  // the dQ kernel tiles 128 query rows and DqCfg::BN key rows
  using QC = DqCfg<DQK, DV>;
  if (int e = bwd_tmaps<DQK, DV>(bp, p, o, QC::BOX_COLS, QC::BOX_COLS, QC::BOX_COLS_V, QC::BM, QC::BN)) return e;
  HSTU_CUDA_OK(cudaFuncSetAttribute(kdq, cudaFuncAttributeMaxDynamicSharedMemorySize, QC::SMEM_BYTES));
  kdq<<<dim3((p.max_seq_len + QC::BM - 1) / QC::BM, p.heads, p.batch), kAttnThreads, QC::SMEM_BYTES, st>>>(bp);
  HSTU_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace hstu
