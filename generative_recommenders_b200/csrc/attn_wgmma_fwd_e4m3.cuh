// Jagged HSTU attention forward on float8 e4m3 q, k, v with per (sequence, head) descales, bf16 output, on the Hopper
// warpgroup tensor cores: the kernel body and its launcher, shared by attn_wgmma_fwd_e4m3.cu (dqk == dv in {32, 64, 128,
// 256}) and attn_wgmma_mixed_fwd_e4m3.cu (dqk < dv, both in that set), DESIGN.md 3.5.  Two widths: DQK, of the e4m3 Q and
// K and the reduction of S = Q K^T, and DV, of the fp16 copy of v and of O (the N of P' V); every instantiation of
// attn_wgmma_fwd_e4m3.cu is DQK == DV == d.
//
//   out = attention(q * qd[b, h], k * kd[b, h], v * vd[b, h])
//
// The structure is the bf16 / fp16 forward's (attn_wgmma_fwd.cuh): one CTA per (128-row query tile, head, sequence), heavy
// tiles first; two warpgroups of 64 query rows; the prologue, the K / V ring protocol of 64-key tiles and the tile-uniform
// mask cases of attn_wgmma_qtile.cuh; where kMerge, O += P_i V_i and S_{i+1} = Q K_{i+1}^T form one MMA batch with one
// wait.  What differs:
//   S = Q K^T  on fp8 tensor cores (wgmma m64n64k32 e4m3, both operands K-major).  Q and K are TMA-staged as bytes; a row
//              of dqk e4m3 values has the layout of a 16-bit row of dqk / 2, so the K-major descriptors apply with 32-byte k
//              steps.  Swizzle: 32 B at dqk = 32, 64 B at dqk = 64, 128-byte boxes at dqk >= 128.
//   P          = silu(alpha qd kd S) * mask, formed as one fp16 operand P' = P 2^p (e4m3_p_exp: a bound from the e4m3
//              range and the dqk terms of S, no amax pass).
//   O += P' V  16-bit, N = dv, on the exact fp16 copy of v that a pre-pass writes into the workspace (attn_fp16_operands.cu):
//              fp16 P keeps the operand rounding inside the bf16 parity bound, which an e4m3 P would not (DESIGN.md 3.5).
//   epilogue   O * (1/N) vd 2^-p -> bf16.
// Rows of the fp16 v copy past a sequence end are the next sequence's rows (or rows at positions >= max_seq_len, which the
// pre-pass never writes), so the V stage of the tile that crosses the end is zeroed past it (zero_tile_rows), as in the
// bf16 forward.  Scales are per (sequence, head): a NaN or Inf descale or input value changes no other (sequence, head).
#pragma once
#include <string.h>

#include "attn_fp16_operands.cuh"
#include "attn_wgmma_qtile.cuh"
#include "common.cuh"
#include "internal.h"
#include "wgmma.cuh"

namespace hstu {
using namespace wg;

struct alignas(64) E4m3FwdParams {
  CUtensorMap tmQ, tmK, tmV;  // Q, K: the e4m3 inputs (bytes); V: the fp16 copy of v
  SeqArgs seq;
  void* out;  // bf16
  long long o_row_stride, o_head_stride;
  const float* descale[3];  // q, k, v: [B, H] fp32, or null (= 1)
  long long ds_batch[3], ds_head[3];
  float alpha;
  float inv_n;       // 1 / max_seq_len
};

template <int DQK, int DV = DQK>
struct E4m3FwdCfg {
  static constexpr int BM = 128;  // query rows per CTA (two warpgroups of 64)
  static constexpr int BN = 64;   // key rows per tile
  static constexpr int SWK = swizzle_bytes(DQK, 1);  // swizzle (bytes) of the e4m3 Q / K boxes: one byte per element
  static constexpr int SWV = swizzle_bytes(DV);      // of the fp16 V boxes
  static constexpr int BOX_COLS = SWK, BOX_COLS_V = SWV / 2;
  static constexpr int NBOX = DQK / BOX_COLS, NBOX_V = DV / BOX_COLS_V;
  static constexpr int Q_BOX = BM * SWK, K_BOX = BN * SWK, V_BOX = BN * SWV;
  static constexpr int Q_BYTES = BM * DQK, K_BYTES = BN * DQK, V_BYTES = BN * DV * 2;
  static constexpr int STAGES = 3;  // 128 dqk + 3 (64 dqk + 128 dv) bytes: 136 KB at (128, 256), 177 KB at d = 256
  static constexpr int OFF_Q = 0;
  static constexpr int OFF_K = OFF_Q + Q_BYTES;
  static constexpr int OFF_V = OFF_K + STAGES * K_BYTES;
  static constexpr int OFF_BAR = OFF_V + STAGES * V_BYTES;
  static constexpr int SMEM_BYTES = OFF_BAR + 256 + 1024;  // + barriers + alignment slack
  static_assert(SMEM_BYTES <= 232448, "shared memory budget");
  static_assert(OFF_K % 1024 == 0 && OFF_V % 1024 == 0 && K_BYTES % 256 == 0 && V_BYTES % 1024 == 0, "swizzle atom alignment");
  static_assert(DQK <= DV, "dqk > dv has no instantiation");
};
// dv <= 64: two CTAs per SM (<= 128 registers per thread), and S_{i+1} merged into the P_i V_i batch.  The O accumulator is
// dv / 2 registers per thread, so every pair with dv >= 128 runs one CTA per SM and waits for each batch separately
// (ptxas -v of each choice: DESIGN.md 3.5)
template <int DV> constexpr int kE4m3MinBlocks = (DV <= 64) ? 2 : 1;
template <int DV> constexpr bool kE4m3Merge = DV <= 64;

__device__ __forceinline__ float load_descale(const float* d, long long bs, long long hs, int b, int h) {
  return d ? d[(long long)b * bs + (long long)h * hs] : 1.f;
}

// Its only instantiations are the kernels of attn_wgmma_fwd_e4m3.cu and attn_wgmma_mixed_fwd_e4m3.cu.
template <int DQK, int DV>
__device__ __forceinline__ void attn_fwd_e4m3_body(const E4m3FwdParams& p) {
  using Cfg = E4m3FwdCfg<DQK, DV>;
  constexpr int SWK = Cfg::SWK, SWV = Cfg::SWV, BN = Cfg::BN, NST = Cfg::STAGES;
  constexpr bool kMerge = kE4m3Merge<DV>;  // as in the bf16 forward: S_{i+1} and P_i V_i in one batch where the registers allow
  const int b = blockIdx.z, h = blockIdx.y;
  const int m0 = (int)(gridDim.x - 1 - blockIdx.x) * Cfg::BM;
  QTileSeq qs;
  if (!qtile_prologue<Cfg::BM, BN>(p.seq, b, h, m0, p.out, p.o_row_stride, p.o_head_stride, DV, &qs)) return;

  uint8_t* smem = dyn_smem_1k();
  KvRing<Cfg> ring{smem, &p.tmK, &p.tmV, h, qs.row0, qs.t0, qs.T};
  ring.init();
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  // The protocol of KvRing (barriers, waits, release_is_last), but this loop issues the fill and the refills itself: the
  // stage of each load is recomputed from its tile index, and the key row is 32-bit.  KvRing::fill / release take the
  // caller's stage, which makes ptxas keep this loop's ring state in vector rather than uniform registers (up to +23
  // registers and +3 instructions per tile), and KvRing::load's 64-bit row costs a uniform -> vector -> uniform round trip
  // per TMA box of every refill (DESIGN.md 3.5).
  const int key_row0 = (int)(qs.row0 + (long long)qs.t0 * BN);
  auto load = [&](auto val_c, int i) {
    constexpr bool kIsV = decltype(val_c)::value;
    const int st = i % NST;
    uint64_t* full = kIsV ? ring.bars->v_full : ring.bars->k_full;
    mbar_arrive_expect_tx(&full[st], kIsV ? Cfg::V_BYTES : Cfg::K_BYTES);
#pragma unroll
    for (int bx = 0; bx < (kIsV ? Cfg::NBOX_V : Cfg::NBOX); ++bx)
      tma_load_3d(smem + (kIsV ? Cfg::OFF_V + st * Cfg::V_BYTES + bx * Cfg::V_BOX : Cfg::OFF_K + st * Cfg::K_BYTES + bx * Cfg::K_BOX),
                  kIsV ? &p.tmV : &p.tmK, &full[st], bx * (kIsV ? Cfg::BOX_COLS_V : Cfg::BOX_COLS), h, key_row0 + i * BN);
  };
  auto release = [&](auto val_c, int i) {
    uint32_t* ctr = decltype(val_c)::value ? ring.bars->v_free : ring.bars->k_free;
    if (lane == 0 && i + NST < qs.T && release_is_last<kAttnThreads / 32>(&ctr[i % NST])) load(val_c, i + NST);
  };
  if (tid == 0) {
    prefetch_tensormap(&p.tmQ);
    prefetch_tensormap(&p.tmK);
    prefetch_tensormap(&p.tmV);
    mbar_arrive_expect_tx(&ring.bars->q_full, Cfg::Q_BYTES);
#pragma unroll
    for (int bx = 0; bx < Cfg::NBOX; ++bx)
      tma_load_3d(smem + Cfg::OFF_Q + bx * Cfg::Q_BOX, &p.tmQ, &ring.bars->q_full, bx * Cfg::BOX_COLS, h, (int)(qs.row0 + m0));
    for (int i = 0; i < min(qs.T, NST); ++i) {
      load(kKey, i);
      load(kVal, i);
    }
  }
  __syncwarp();

  const int wgi = warp >> 2, w = warp & 3, g = lane >> 2, t4 = lane & 3;
  const int q_base = m0 + wgi * 64 + w * 16 + g;  // query position of accumulator rows g (+ 8)
  const uint32_t sq = smem_u32(smem + Cfg::OFF_Q) + wgi * 64 * SWK;
  const uint32_t sk = smem_u32(smem + Cfg::OFF_K), sv = smem_u32(smem + Cfg::OFF_V);
  const bool fast = qs.msk.fast != 0;
  const int full_lim = full_valid_limit(qs.msk, m0);
  // scales of this (sequence, head): S holds S / (qd kd), P is formed as 2^e_p P, O holds 2^e_p O / vd.
  const float qd = load_descale(p.descale[0], p.ds_batch[0], p.ds_head[0], b, h);
  const float kd = load_descale(p.descale[1], p.ds_batch[1], p.ds_head[1], b, h);
  const float vd = load_descale(p.descale[2], p.ds_batch[2], p.ds_head[2], b, h);
  // The scalars are built from the frexp mantissas (in [0.5, 1)) and exponents of the factors, so that small but legal
  // descales lose no precision in fp32 subnormals: c_sp = alpha/2 qd kd 2^e_p forms P' and is a normal number (m 2^(-4 -
  // log2 dqk) unless e_p is clamped); c_s = alpha/2 qd kd is only the tanh argument's scale, and where it underflows |x| <
  // 2^-100, so tanh x is nothing next to the 1 of 1 + tanh x.  The output scale (1/N) vd 2^-e_p is applied as the normal c_o =
  // (1/N) m_v and an exact power of two.  Zero, Inf and NaN factors propagate as before (frexpf keeps them).
  // The bound of e_p is on |alpha qd kd S|, and S sums dqk products: it takes dqk, whatever dv is.
  const int e_p = e4m3_p_exp(p.alpha, qd, kd, DQK);
  int ea, eq, ek, ev;
  const float m_s = frexpf(p.seq.alpha_half, &ea) * frexpf(qd, &eq) * frexpf(kd, &ek);
  const float c_s = scalbnf(m_s, ea + eq + ek), c_sp = scalbnf(m_s, ea + eq + ek + e_p);
  const float c_o = p.inv_n * frexpf(vd, &ev);
  const int e_o = ev - e_p;

  float o[DV / 2];
#pragma unroll
  for (int e = 0; e < DV / 2; ++e) o[e] = 0.f;
  uint32_t a[BN / 16][4];
#pragma unroll
  for (int kk = 0; kk < BN / 16; ++kk)
#pragma unroll
    for (int r = 0; r < 4; ++r) a[kk][r] = 0u;
  float s[BN / 2];
  // S = Q K_i^T into s (issue only; the caller fences, commits and waits)
  auto issue_s = [&](int i) {
    const uint32_t kst = sk + (i % NST) * Cfg::K_BYTES;
#pragma unroll
    for (int ks = 0; ks < DQK / 32; ++ks) {
      const int kb = ks * 32, bx = kb / SWK, off = kb % SWK;
      wgmma_ss_64_e4m3(s, desc_kmajor<SWK>(sq + bx * Cfg::Q_BOX, off), desc_kmajor<SWK>(kst + bx * Cfg::K_BOX, off), ks > 0);
    }
  };
  mbar_wait(&ring.bars->q_full, 0);
  ring.wait(kKey, 0, 0);
  wgmma_fence();
  issue_s(0);
  wgmma_commit();
  wgmma_wait<0>();
  fence_regs(s);
  release(kKey, 0);
  __syncwarp();
  for (int i = 0; i < qs.T; ++i) {
    const int st = i % NST;
    const bool next = i + 1 < qs.T;
    const int n0 = (qs.t0 + i) * BN;
    // P' = 2^e_p silu(alpha S) * mask; the mask case is chosen once per tile, so each score loop is one basic block
    auto silu = [&](int n) {
      const float x = s[n] * c_s, xp = s[n] * c_sp;
      return __fmaf_rn(xp, tanh_approx(x), xp);  // silu(2x) = x (1 + tanh x)
    };
    mask_scores<BN>(qs.msk, fast, full_lim, qs.len, q_base, n0, t4, s, silu);
#pragma unroll
    for (int kk = 0; kk < BN / 16; ++kk)
#pragma unroll
      for (int r = 0; r < 4; ++r) a[kk][r] = pack_f16x2_sat(s[8 * kk + 2 * r], s[8 * kk + 2 * r + 1]);
    ring.wait(kVal, st, (i / NST) & 1);
    // the last tile may cross the sequence end: its V rows >= len belong to the next sequence (P is 0 there, V may be NaN)
    if (n0 + BN > qs.len)  // CTA-uniform; the last tile, so its stage is not refilled
      zero_tile_rows_sync<BN, SWV, Cfg::NBOX_V, kAttnThreads>(smem + Cfg::OFF_V + st * Cfg::V_BYTES, qs.len - n0);
    if (kMerge && next) ring.wait(kKey, (i + 1) % NST, ((i + 1) / NST) & 1);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < BN / 16; ++kk)
      wgmma_rs<DV, false, 1>(o, a[kk], desc_mnmajor<SWV>(sv + st * Cfg::V_BYTES, kk * 16, Cfg::V_BOX), 1);
    if (kMerge && next) issue_s(i + 1);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(o);
    fence_regs(a);
    fence_regs(s);
    release(kVal, i);
    if (!kMerge && next) {
      ring.wait(kKey, (i + 1) % NST, ((i + 1) / NST) & 1);
      wgmma_fence();
      issue_s(i + 1);
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs(s);
    }
    if (next) release(kKey, i + 1);
    __syncwarp();
  }

  // ---------------- epilogue: O * (1/N) vd 2^-e_p -> bf16 ----------------
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int qi = q_base + hh * 8;
    if (qi - m0 < qs.mrows) {
      uint16_t* orow = reinterpret_cast<uint16_t*>(p.out) + (qs.row0 + qi) * p.o_row_stride + (long long)h * p.o_head_stride;
#pragma unroll
      for (int nb = 0; nb < DV / 8; ++nb)
        *reinterpret_cast<uint32_t*>(orow + nb * 8 + 2 * t4) =
            pack_bf16x2(scalbnf(o[nb * 4 + hh * 2] * c_o, e_o), scalbnf(o[nb * 4 + hh * 2 + 1] * c_o, e_o));
    }
  }
}

// ------------------------------------------------------------------------------------------------
// host
// ------------------------------------------------------------------------------------------------
// kern: the kernel of this DQK / DV (an instance of attn_fwd_e4m3_body); v16: the fp16 copy of v, [L, H, DV] contiguous
template <int DQK, int DV>
int launch_fwd_e4m3(const hstu_attn_params& p, const hstu_attn_descales& ds, const void* v16, cudaStream_t st,
                    void (*kern)(E4m3FwdParams)) {
  using Cfg = E4m3FwdCfg<DQK, DV>;
  E4m3FwdParams fp;
  memset(&fp, 0, sizeof(fp));
  if (int e = make_tmap_rows_heads(&fp.tmQ, p.q, p.total_rows, p.heads, DQK, p.q_row_stride, p.q_head_stride, Cfg::BOX_COLS, Cfg::BM, 1))
    return e;
  if (int e = make_tmap_rows_heads(&fp.tmK, p.k, p.total_rows, p.heads, DQK, p.k_row_stride, p.k_head_stride, Cfg::BOX_COLS, Cfg::BN, 1))
    return e;
  if (int e = make_tmap_rows_heads(&fp.tmV, v16, p.total_rows, p.heads, DV, (long long)p.heads * DV, DV, Cfg::BOX_COLS_V, Cfg::BN, 2))
    return e;
  fp.seq = seq_args(p);
  fp.out = p.out;
  fp.o_row_stride = p.o_row_stride;
  fp.o_head_stride = p.o_head_stride;
  fp.descale[0] = ds.q, fp.ds_batch[0] = ds.q_batch_stride, fp.ds_head[0] = ds.q_head_stride;
  fp.descale[1] = ds.k, fp.ds_batch[1] = ds.k_batch_stride, fp.ds_head[1] = ds.k_head_stride;
  fp.descale[2] = ds.v, fp.ds_batch[2] = ds.v_batch_stride, fp.ds_head[2] = ds.v_head_stride;
  fp.alpha = p.alpha;
  fp.inv_n = 1.0f / (float)p.max_seq_len;
  HSTU_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
  dim3 grid((p.max_seq_len + Cfg::BM - 1) / Cfg::BM, p.heads, p.batch);
  kern<<<grid, kAttnThreads, Cfg::SMEM_BYTES, st>>>(fp);
  HSTU_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace hstu
