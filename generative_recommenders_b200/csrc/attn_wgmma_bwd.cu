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
// Thread 0 issues the TMA loads: K and V once, then Q_j and dO_j; a stage is refilled once all 256 threads have released it
// (the MMAs that read it have completed).  No separate producer warp: the dK and dV accumulators (d = 128: 64 registers each
// per thread) need the register budget of a 256-thread block.
// Each warpgroup waits for its own MMAs before the next elementwise step (an MMA batch left in flight across it makes ptxas
// serialise the batch); a Q_j / dO_j stage is released as soon as dV / dK of tile j have completed.
// P and dS are 16-bit operands of the input format: fp16, or for bf16 inputs a hi + lo pair of bf16 operands (wgmma.cuh,
// Operand), so that their rounding stays inside the 1e-3 parity budget whatever the scale of dO.
//
// Reference math: ops/triton/triton_hstu_attention.py:995-1006,1222 and SURVEY.md appendix A; unlike the Triton
// kernel dQ is accumulated in fp32, not in the input dtype (triton_attention_utils.py:47-60).
#include <string.h>

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
  float* dq_acc;  // [L, H, D] fp32, zero-initialised
  long long dk_row_stride, dk_head_stride, dv_row_stride, dv_head_stride;
  int offsets_i64, targets_i64;
  int max_seq_len, heads;
  int win, min_full, ctx;
  float alpha_half;
  float dv_scale;  // 1 / N
  float dk_scale;  // alpha / (2 N): dS^T holds 2 dS N / alpha
};

template <int D>
struct BwdCfg {
  static constexpr int BKV = 128, BQ = 64;
  static constexpr int SW = (D * 2 >= 128) ? 128 : D * 2;
  static constexpr int BOX_COLS = SW / 2;
  static constexpr int NBOX = D / BOX_COLS;
  static constexpr int KV_BOX = BKV * SW;
  static constexpr int QD_BOX = BQ * SW;
  static constexpr int KV_BYTES = BKV * D * 2;
  static constexpr int QD_BYTES = BQ * D * 2;
  static constexpr int STAGES = (D <= 32) ? 4 : (D == 64 ? 3 : 2);  // Q_j / dO_j ring depth
  static constexpr int DS_BYTES = BKV * BQ * 2;                      // one [128 kv][64 q] box, 128-byte swizzle
  static constexpr int DQN = D < 64 ? D : 64;                        // dQ columns per pass (one 128-byte box of K)
  static constexpr int OFF_K = 0;
  static constexpr int OFF_V = OFF_K + KV_BYTES;
  static constexpr int OFF_Q = OFF_V + KV_BYTES;
  static constexpr int OFF_DO = OFF_Q + STAGES * QD_BYTES;
  static constexpr int OFF_DS = OFF_DO + STAGES * QD_BYTES;          // [buffer 0/1][hi / lo]
  static constexpr int OFF_BAR = OFF_DS + 4 * DS_BYTES;
  static constexpr int SMEM_BYTES = OFF_BAR + 256 + 1024;
  static_assert(SMEM_BYTES <= 232448, "shared memory budget");
};
constexpr int kBwdThreads = 256;

struct BwdBars {
  uint64_t kv_full;
  uint64_t qd_full[4], qd_empty[4];
};

// query tiles of a key tile: the contextual prefix tiles [0, A), then the causal / window range
struct QTiles {
  int A, first, T;
  __device__ __forceinline__ int at(int i) const { return i < A ? i : first + (i - A); }
};

template <int D, bool BF16>
__global__ void __launch_bounds__(kBwdThreads, 1) attn_bwd_wgmma_kernel(const __grid_constant__ BwdParams p) {
  using Cfg = BwdCfg<D>;
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
      mbar_init(&bars->qd_empty[i], 256);
    }
    fence_barrier_init();
  }
  __syncthreads();

  // TMA issue (thread 0): K, V and the first STAGES query tiles now; stage st is refilled once both warpgroups have released it
  auto load_qd = [&](int j) {
    const int st = j % NST;
    const int q_row = (int)(row0 + (long long)qt.at(j) * BQ);
    if (j >= NST) mbar_wait(&bars->qd_empty[st], ((j / NST) - 1) & 1);
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

  float dv[D / 2], dk[D / 2];
#pragma unroll
  for (int e = 0; e < D / 2; ++e) dv[e] = dk[e] = 0.f;
  uint32_t pf_hi[4][4], pf_lo[4][4], df_hi[4][4], df_lo[4][4];
#pragma unroll
  for (int kk = 0; kk < 4; ++kk)
#pragma unroll
    for (int r = 0; r < 4; ++r) pf_hi[kk][r] = pf_lo[kk][r] = df_hi[kk][r] = df_lo[kk][r] = 0u;

  mbar_wait(&bars->kv_full, 0);
  for (int j = 0; j < qt.T; ++j) {
    const int st = j % NST;
    const uint32_t ph = (j / NST) & 1;
    const int q0 = qt.at(j) * BQ;
    mbar_wait(&bars->qd_full[st], ph);
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

    // p = x sig(x) and 2 dS = dP (1 + g2) from one tanh (h = alpha s / 2, t = tanh h, p = h (1 + t), g2 = t + h (1 - t^2))
    const bool full = fast && keys_hist && n0 + Cfg::BKV <= q0 && q0 + BQ <= len;  // tile-uniform: every pair valid
#pragma unroll
    for (int nb = 0; nb < BQ / 8; ++nb)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float x = s[nb * 4 + e] * p.alpha_half;
        const float t = tanh_approx(x);
        const float g2 = __fmaf_rn(x, __fmaf_rn(-t, t, 1.f), t);
        float pv = __fmaf_rn(x, t, x), dsv = __fmaf_rn(dp[nb * 4 + e], g2, dp[nb * 4 + e]);
        if (!full) {
          const int kj = k_base + (e >> 1) * 8, qi = q0 + nb * 8 + 2 * t4 + (e & 1);
          const bool v = kj < len && qi < len && mask_valid(msk, qi, kj);
          pv = v ? pv : 0.f;
          dsv = v ? dsv : 0.f;
        }
        s[nb * 4 + e] = pv;
        dp[nb * 4 + e] = dsv;
      }
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
    wgmma_commit();
    wgmma_wait<0>();  // an MMA batch never stays in flight across the elementwise code (ptxas would serialise them)
    fence_regs(dv);
    fence_regs(dk);
    fence_regs(pf_hi);
    fence_regs(pf_lo);
    fence_regs(df_hi);
    fence_regs(df_lo);
    mbar_arrive(&bars->qd_empty[st]);
    if (tid == 0 && j + NST < qt.T) load_qd(j + NST);  // Q_j and dO_j are no longer read
    __syncwarp();
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
        const float k0 = dk[nb * 4 + hh * 2] * p.dk_scale, k1 = dk[nb * 4 + hh * 2 + 1] * p.dk_scale;
        const float v0 = dv[nb * 4 + hh * 2] * p.dv_scale, v1 = dv[nb * 4 + hh * 2 + 1] * p.dv_scale;
        *reinterpret_cast<uint32_t*>(krow + nb * 8) = BF16 ? pack_bf16x2(k0, k1) : pack_f16x2(k0, k1);
        *reinterpret_cast<uint32_t*>(vrow + nb * 8) = BF16 ? pack_bf16x2(v0, v1) : pack_f16x2(v0, v1);
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

size_t wgmma_workspace_bytes(const hstu_attn_params& p, bool bwd) {
  if (!bwd) return 0;
  return (size_t)p.total_rows * p.heads * p.dqk * sizeof(float);  // fp32 dQ accumulator [L, H, D]
}

template <int D, bool BF16>
static int launch_bwd_wgmma(const hstu_attn_params& p, cudaStream_t st) {
  using Cfg = BwdCfg<D>;
  const size_t need = wgmma_workspace_bytes(p, true);
  if (p.workspace == nullptr || p.workspace_bytes < need) {
    set_error("hstu_attn_bwd: workspace of %zu bytes required (got %zu)", need, p.workspace_bytes);
    return HSTU_ERR_WORKSPACE;
  }
  BwdParams bp;
  memset(&bp, 0, sizeof(bp));
  if (int e = make_tmap_rows_heads(&bp.tmQ, p.q, p.total_rows, p.heads, D, p.q_row_stride, p.q_head_stride, Cfg::BOX_COLS, Cfg::BQ)) return e;
  if (int e = make_tmap_rows_heads(&bp.tmK, p.k, p.total_rows, p.heads, D, p.k_row_stride, p.k_head_stride, Cfg::BOX_COLS, Cfg::BKV)) return e;
  if (int e = make_tmap_rows_heads(&bp.tmV, p.v, p.total_rows, p.heads, D, p.v_row_stride, p.v_head_stride, Cfg::BOX_COLS, Cfg::BKV)) return e;
  if (int e = make_tmap_rows_heads(&bp.tmDO, p.dout, p.total_rows, p.heads, D, p.do_row_stride, p.do_head_stride, Cfg::BOX_COLS, Cfg::BQ)) return e;
  bp.seq_offsets = p.seq_offsets;
  bp.num_targets = p.num_targets;
  bp.dk = p.dk;
  bp.dv = p.dv_out;
  bp.dq_acc = reinterpret_cast<float*>(p.workspace);
  bp.dk_row_stride = p.dk_row_stride;
  bp.dk_head_stride = p.dk_head_stride;
  bp.dv_row_stride = p.dv_row_stride;
  bp.dv_head_stride = p.dv_head_stride;
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
  return 0;
}

int attn_wgmma_bwd(const hstu_attn_params& p, cudaStream_t st) {
  const bool bf = p.dtype == HSTU_BF16;
  switch (p.dqk) {
    case 32: return bf ? launch_bwd_wgmma<32, true>(p, st) : launch_bwd_wgmma<32, false>(p, st);
    case 64: return bf ? launch_bwd_wgmma<64, true>(p, st) : launch_bwd_wgmma<64, false>(p, st);
    case 128: return bf ? launch_bwd_wgmma<128, true>(p, st) : launch_bwd_wgmma<128, false>(p, st);
  }
  set_error("wgmma backward: unsupported head dim %d", p.dqk);
  return HSTU_ERR_UNSUPPORTED;
}

}  // namespace hstu
