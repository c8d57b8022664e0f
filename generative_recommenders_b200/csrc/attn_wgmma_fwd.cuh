// Jagged HSTU attention forward on the Hopper warpgroup tensor cores (wgmma) with TMA-staged tiles: the kernel body and its
// launcher, shared by attn_wgmma_fwd.cu (dqk == dv in {32, 64, 128, 256}) and attn_wgmma_mixed_fwd.cu (dqk < dv, both in
// that set).  bf16 / fp16.  Two widths: DQK, of Q and K and the reduction of S = Q K^T, and DV, of V and O (the N of P V).
// Q / K and V are TMA boxes of their own swizzle width; every existing instantiation is DQK == DV == d.
//
// One CTA per (128-row query tile, head, sequence); heavy (late) query tiles are scheduled first.  Two warpgroups
// of 64 query rows each.  Per key tile:
//   S = Q K^T            (wgmma, A = Q and B = K both K-major in shared memory, fp32 accumulators)
//   P = silu(alpha S) * mask   (one tanh per score, in registers)
//   O += P V             (wgmma, A = P from registers, B = V MN-major in shared memory)
// Key tiles of 64 rows keep a thread at <= 128 registers for d <= 64, so two CTAs share an SM there.
// Each warpgroup waits for its own MMAs; the two warpgroups overlap each other's tensor-core and elementwise phases.  With
// d <= 64, O += P_i V_i and S_{i+1} = Q K_{i+1}^T are one MMA batch with one wait per tile (O is never read in the loop).
// Q is loaded once; the K and V tiles go through the ring of attn_wgmma_qtile.cuh (STAGES buffers each, refilled by the last
// warp to release a stage, no producer warp: the 64 x d fp32 O accumulator, 128 registers per thread at d = 256, needs the
// register budget of a 256-thread block).
// P is a 16-bit MMA operand of the same format as V (wgmma takes one format for A and B): fp16 for fp16 inputs, and for
// bf16 inputs a hi + lo pair of bf16 operands multiplied twice (wgmma.cuh, Operand), so that its rounding stays well inside
// the 1e-3 parity budget.  bf16 inputs at d = 32 instead run the fp16 kernel on exactly scaled fp16 copies of q, k, v with
// a scaled fp16 P (`amax`, attn_fp16_operands.cuh); its epilogue undoes the scales and writes bf16.  The 1/N factor of the reference is applied once in the epilogue (registers -> global, rows past
// the sequence end are not written).  Rows past the sequence end that a TMA box drags in are masked out of P, and zeroed in the
// V stage of the one key tile that crosses the end (zero_tile_rows), since P = 0 does not neutralise a NaN or Inf in V.
//
// Delta-q (kDelta, KV-cached inference, DESIGN.md 3.6): query row i of sequence b is row b * delta + i of q / out, at sequence
// position len - delta + i; keys are the whole (unclipped) sequence; no zero-fill past max_seq_len.  The grid is (sequence x
// head, query tile, key chunk): HSTU has no softmax, so outputs over disjoint key ranges simply add.  Each CTA takes chunk c
// of the key tiles its rows attend (an even split in whole 64-key tiles).  With one chunk it writes out itself; with more it
// writes unscaled fp32 partials to the workspace and delta_reduce_kernel sums them in chunk order (bitwise reproducible).
// Padding rows past delta cost nothing: a warpgroup with no valid row issues no MMA and only releases its stages once
// they have landed (so its releases never run ahead into the next use of a stage), and a warp with no valid row skips the
// elementwise stage with P = 0.  bf16 keeps the hi / lo split of P at every d, d = 32 included (no pre-pass over the cache).
//
// Reference semantics: ops/pytorch/pt_hstu_attention.py:130-171 (delta: :175-235); tile skipping mirrors the idea of
// ops/triton/triton_hstu_attention.py:517-543 (loop bounds from the mask) but is derived from common.cuh's ranges.
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

struct alignas(64) FwdParams {
  CUtensorMap tmQ, tmK, tmV;
  SeqArgs seq;
  void* out;
  long long o_row_stride, o_head_stride;
  float inv_n;  // 1 / max_seq_len
  const uint32_t* amax;  // fp16 kernel on scaled copies of bf16 inputs: [B, H, 4] amax bits (attn_fp16_operands.cuh); else null
  // delta-q only (kDelta): query rows per sequence, and with gridDim.z > 1 key chunks the fp32 partials [chunks, B * delta, H, DV]
  int delta;
  float* part;
};

template <int DQK, int DV = DQK>
struct FwdCfg {
  static constexpr int BM = 128;                     // query rows per CTA (two warpgroups of 64)
  static constexpr int BN = 64;                      // key rows per tile
  static constexpr int SW = swizzle_bytes(DQK), SWV = swizzle_bytes(DV);  // swizzle width (bytes) of the Q / K boxes, of the V boxes
  static constexpr int BOX_COLS = SW / 2;
  static constexpr int BOX_COLS_V = SWV / 2;
  static constexpr int Q_BOX = BM * SW;
  static constexpr int K_BOX = BN * SW;
  static constexpr int V_BOX = BN * SWV;
  static constexpr int Q_BYTES = BM * DQK * 2;
  static constexpr int K_BYTES = BN * DQK * 2;
  static constexpr int V_BYTES = BN * DV * 2;
  static constexpr int NBOX = DQK / BOX_COLS;
  static constexpr int NBOX_V = DV / BOX_COLS_V;
  // d = 256: 64 KB of Q and 64 KB per stage; every dqk < dv pair has room for three (128, 256: 32 + 3 x 48 KB)
  static constexpr int STAGES = (DQK == 256) ? 2 : 3;
  static constexpr int OFF_Q = 0;
  static constexpr int OFF_K = OFF_Q + Q_BYTES;
  static constexpr int OFF_V = OFF_K + STAGES * K_BYTES;
  static constexpr int OFF_BAR = OFF_V + STAGES * V_BYTES;
  static constexpr int SMEM_BYTES = OFF_BAR + 256 + 1024;  // + barriers + alignment slack
  static_assert(SMEM_BYTES <= 232448, "shared memory budget");
  static_assert(DQK <= DV, "dqk > dv has no instantiation");
};
// dv <= 64: two CTAs per SM (<= 128 registers per thread; the O accumulator is dv / 2 of them)
template <int DV> constexpr int kFwdMinBlocks = (DV <= 64) ? 2 : 1;

// Delta-q: the output row (of q / out, and of the partials of chunk blockIdx.z) of local query row 0 of the CTA, and the CTA's
// valid query rows.  Recomputed from the grid where needed, so that nothing extra stays live through the key loop.
struct DeltaRows {
  long long out_row, part_row;
  int rows;
};
template <int BM>
__device__ __forceinline__ DeltaRows delta_rows(const FwdParams& p) {
  const int m0 = (int)blockIdx.y * BM;
  const long long r = (long long)(blockIdx.x / p.seq.heads) * p.delta + m0;
  return {r, (long long)blockIdx.z * (gridDim.x / p.seq.heads) * p.delta + r, min(BM, p.delta - m0)};
}

// kDelta: the delta-q geometry and key chunks described at the top (grid (B * H, query tiles, chunks)); otherwise the full
// attention of grid (query tiles, H, B).  kBidir: the non-causal mask (attn_wgmma_bidir.cu; full attention only): the key
// range of kv_range_for_q_rows_bidir and the mask cases of mask_scores_bidir, nothing else.  Its only instantiations are
// the kernels of attn_wgmma_fwd.cu, attn_wgmma_mixed_fwd.cu and attn_wgmma_bidir.cu.
template <int DQK, int DV, bool BF16, bool kDelta, bool kBidir = false>
__device__ __forceinline__ void attn_fwd_wgmma_body(const FwdParams& p) {
  static_assert(!(kDelta && kBidir), "the delta-q forward is causal");
  using Cfg = FwdCfg<DQK, DV>;
  constexpr int SW = Cfg::SW, SWV = Cfg::SWV, BN = Cfg::BN, NST = Cfg::STAGES;
  // dv <= 64: P V of tile i and S of tile i + 1 form one MMA batch with one wait (both fit in 128 registers); larger dv waits
  // for each batch separately, since the O accumulator leaves no room for S next to the P fragments
  constexpr bool kMerge = DV <= 64;
  const int b = kDelta ? (int)blockIdx.x / p.seq.heads : (int)blockIdx.z, h = kDelta ? (int)blockIdx.x % p.seq.heads : (int)blockIdx.y;
  const int m0 = kDelta ? (int)blockIdx.y * Cfg::BM : (int)(gridDim.x - 1 - blockIdx.x) * Cfg::BM;  // first query row of the CTA
  QTileSeq qs;
  if constexpr (kDelta) {  // query row i at position len - delta + i; the whole sequence, unclipped
    seq_rows(p.seq, b, &qs);
  } else if (!qtile_rows(p.seq, b, h, m0, p.out, p.o_row_stride, p.o_head_stride, DV, &qs)) {
    return;
  }
  const int p0 = kDelta ? qs.len - p.delta + m0 : m0;  // sequence position of query row m0 (delta: the last delta rows)
  key_tiles<Cfg::BM, BN, kBidir>(p.seq, b, p0, (kDelta ? p.delta : qs.len) - m0, &qs);
  if constexpr (kDelta) {
    // chunk blockIdx.z of gridDim.z even shares of whole tiles; an empty share (or no key at all) writes zeros, so that
    // every partial the reduction reads is defined
    const int per = (qs.T + (int)gridDim.z - 1) / (int)gridDim.z;
    qs.t0 += (int)blockIdx.z * per;
    qs.T = min(per, qs.T - (int)blockIdx.z * per);
    if (qs.T <= 0) {
      const DeltaRows dr = delta_rows<Cfg::BM>(p);
      for (int idx = threadIdx.x; idx < dr.rows * DV; idx += kAttnThreads) {
        if (gridDim.z > 1) p.part[((dr.part_row + idx / DV) * p.seq.heads + h) * DV + idx % DV] = 0.f;
        else reinterpret_cast<uint16_t*>(p.out)[(dr.out_row + idx / DV) * p.o_row_stride + (long long)h * p.o_head_stride + idx % DV] = 0;
      }
      return;
    }
  }

  uint8_t* smem = dyn_smem_1k();
  KvRing<Cfg> ring{smem, &p.tmK, &p.tmV, h, qs.row0, qs.t0, qs.T};
  ring.init();
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (tid == 0) {
    prefetch_tensormap(&p.tmQ);
    prefetch_tensormap(&p.tmK);
    prefetch_tensormap(&p.tmV);
    mbar_arrive_expect_tx(&ring.bars->q_full, Cfg::Q_BYTES);
#pragma unroll
    for (int bx = 0; bx < Cfg::NBOX; ++bx)
      tma_load_3d(smem + Cfg::OFF_Q + bx * Cfg::Q_BOX, &p.tmQ, &ring.bars->q_full, bx * Cfg::BOX_COLS, h,
                  kDelta ? b * p.delta + m0 : (int)(qs.row0 + m0));
    ring.fill();
  }
  __syncwarp();

  // (delta: the plain index; the descriptors held in registers through its loop would spill at d = 64 with bf16 inputs)
  const int wgi = kDelta ? warp >> 2 : warpgroup_index(), w = warp & 3, g = lane >> 2, t4 = lane & 3;
  if constexpr (kDelta) {
    if (wgi * 64 >= qs.mrows) {
      // a warpgroup of padding rows only: no MMA, no tanh, no output.  It still releases every stage use, once that use has
      // landed (its full barrier), so that its releases cannot run ahead into the next use of the stage and complete a
      // release while another warp still reads it; and it helps zero the V rows past the sequence end (CTA-wide barrier)
      ring.wait(kKey, 0, 0);
      ring.release(kKey, 0, 0);
      for (int i = 0; i < qs.T; ++i) {
        const int st = i % NST;
        const bool next = i + 1 < qs.T;
        const int n0 = (qs.t0 + i) * BN;
        ring.wait(kVal, st, (i / NST) & 1);
        if (n0 + BN > qs.len) zero_tile_rows_sync<BN, SWV, Cfg::NBOX_V, kAttnThreads>(smem + Cfg::OFF_V + st * Cfg::V_BYTES, qs.len - n0);
        if (next) ring.wait(kKey, (i + 1) % NST, ((i + 1) / NST) & 1);
        __syncwarp();
        ring.release(kVal, i, st);
        if (next) ring.release(kKey, i + 1, (i + 1) % NST);
        __syncwarp();
      }
      return;
    }
  }
  const int q_base = p0 + wgi * 64 + w * 16 + g;  // query position of accumulator rows g (+ 8)
  // delta: a warp whose 16 rows all lie past delta skips the elementwise stage (warp-uniform)
  const bool rows_idle = kDelta && wgi * 64 + w * 16 >= qs.mrows;
  // wgmma descriptors, built once: Q of the warpgroup, and K (K-major) and V (MN-major) of ring stage 0; everything else is
  // a constant step from them (desc_add), and all three are warp-uniform
  const uint64_t dq0 = desc_pin(desc_kmajor<SW>(smem_u32(smem + Cfg::OFF_Q) + wgi * 64 * SW, 0));
  const uint64_t dk0 = desc_pin(desc_kmajor<SW>(smem_u32(smem + Cfg::OFF_K), 0));
  const uint64_t dv0 = desc_pin(desc_mnmajor<SWV>(smem_u32(smem + Cfg::OFF_V), 0, Cfg::V_BOX));
  const bool fast = qs.msk.fast != 0;
  const int full_lim = full_valid_limit(qs.msk, p0);
  // scaled fp16 operands: S holds 2^(e_q + e_k) S, P is formed as 2^e_p P and O holds 2^(e_p + e_v) O
  constexpr bool kScaled = !kDelta && !BF16 && DQK == 32 && DV == 32;  // the only instantiation that runs bf16 inputs on fp16 copies
  float c_s = p.seq.alpha_half, c_p = 1.f;
  int e_out = 0;
  if (kScaled && p.amax != nullptr) {
    const OperandExps ex = operand_exps(p.amax + ((long long)b * p.seq.heads + h) * kAmaxSlots, 2.f * p.seq.alpha_half, DQK);
    c_s = ldexpf(p.seq.alpha_half, -(ex.q + ex.k));
    c_p = pow2f(ex.p);
    e_out = -(ex.p + ex.v);
  }

  float o[DV / 2];
#pragma unroll
  for (int e = 0; e < DV / 2; ++e) o[e] = 0.f;
  uint32_t a_hi[BN / 16][4], a_lo[BN / 16][4];
#pragma unroll
  for (int kk = 0; kk < BN / 16; ++kk)
#pragma unroll
    for (int r = 0; r < 4; ++r) a_hi[kk][r] = a_lo[kk][r] = 0u;
  float s[BN / 2];
  // S = Q K^T of the key tile in stage st into s (issue only; the caller fences, commits and waits)
  auto issue_s = [&](int st) {
    const uint64_t kd = desc_stage(dk0, st, Cfg::K_BYTES);
#pragma unroll
    for (int ks = 0; ks < DQK / 16; ++ks) {
      const int kb = ks * 32, bx = kb / SW, off = kb % SW;
      wgmma_ss<BN, BF16, 0, 0>(s, desc_add(dq0, bx * Cfg::Q_BOX + off), desc_add(kd, bx * Cfg::K_BOX + off), ks > 0);
    }
  };
  mbar_wait(&ring.bars->q_full, 0);
  ring.wait(kKey, 0, 0);
  wgmma_fence();
  issue_s(0);
  wgmma_commit();
  wgmma_wait<0>();
  fence_regs(s);
  ring.release(kKey, 0, 0);
  __syncwarp();
  // Per tile i (s holds S_i): P_i -> A fragments; one MMA batch of O += P_i V_i and (kMerge) S_{i+1} = Q K_{i+1}^T; one wait;
  // V_i and K_{i+1} are released.  O is never read inside the loop, so no MMA waits on the elementwise code of its own tile.
  // The last tile (kLast) is peeled off the loop: it has no next tile, and it is the only one that can cross the sequence
  // end (its key range ends at hi <= len), so the loop itself tests neither.
  RingPos<NST> cur;  // ring stage and phase parity of tile i
  auto tile = [&](int i, auto last_c) {
    constexpr bool kLast = decltype(last_c)::value;
    RingPos<NST> nx = cur;  // tile i + 1
    nx.advance();
    const int st = cur.st;
    const int n0 = (qs.t0 + i) * BN;
    // P = silu(alpha S) * mask
    auto silu = [&](int n) {
      const float x = s[n] * c_s, xp = kScaled ? x * c_p : x;
      return __fmaf_rn(xp, tanh_approx(x), xp);  // silu(2x) = x (1 + tanh x)
    };
    // a warp of padding rows only (delta) skips this stage: its A fragments keep the zeros they start with, so its P is 0
    if (!rows_idle) {
      if constexpr (kBidir) mask_scores_bidir<BN>(qs.msk, qs.len, p0, p0 + qs.mrows, q_base, n0, t4, s, silu);
      else mask_scores<BN>(qs.msk, fast, full_lim, qs.len, q_base, n0, t4, s, silu);
#pragma unroll
      for (int kk = 0; kk < BN / 16; ++kk) {
        const Operand<BF16> x0(s[8 * kk + 0], s[8 * kk + 1]), x1(s[8 * kk + 2], s[8 * kk + 3]);
        const Operand<BF16> x2(s[8 * kk + 4], s[8 * kk + 5]), x3(s[8 * kk + 6], s[8 * kk + 7]);
        a_hi[kk][0] = x0.hi; a_hi[kk][1] = x1.hi; a_hi[kk][2] = x2.hi; a_hi[kk][3] = x3.hi;
        a_lo[kk][0] = x0.lo; a_lo[kk][1] = x1.lo; a_lo[kk][2] = x2.lo; a_lo[kk][3] = x3.lo;
      }
    }
    ring.wait(kVal, st, cur.ph);
    // the last tile may cross the sequence end: its V rows >= len belong to the next sequence (P is 0 there, V may be NaN)
    if (kLast && n0 + BN > qs.len)  // CTA-uniform; the last tile, so its stage is not refilled
      zero_tile_rows_sync<BN, SWV, Cfg::NBOX_V, kAttnThreads>(smem + Cfg::OFF_V + st * Cfg::V_BYTES, qs.len - n0);
    if (kMerge && !kLast) ring.wait(kKey, nx.st, nx.ph);
    wgmma_fence();
    const uint64_t vd = desc_stage(dv0, st, Cfg::V_BYTES);
#pragma unroll
    for (int kk = 0; kk < BN / 16; ++kk) {
      wgmma_rs<DV, BF16, 1>(o, a_hi[kk], desc_add(vd, kk * 16 * SWV), 1);
      if constexpr (BF16) wgmma_rs<DV, BF16, 1>(o, a_lo[kk], desc_add(vd, kk * 16 * SWV), 1);
    }
    if (kMerge && !kLast) issue_s(nx.st);
    wgmma_commit();
    wgmma_wait<0>();  // an MMA batch never stays in flight across the elementwise code (ptxas would serialise them)
    fence_regs(o);
    fence_regs(a_hi);
    fence_regs(a_lo);
    fence_regs(s);
    ring.release(kVal, i, st);
    if (!kMerge && !kLast) {
      ring.wait(kKey, nx.st, nx.ph);
      wgmma_fence();
      issue_s(nx.st);
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs(s);
    }
    if (!kLast) ring.release(kKey, i + 1, nx.st);
    __syncwarp();
    cur = nx;
  };
  for (int i = 0; i < qs.T - 1; ++i) tile(i, std::false_type{});
  tile(qs.T - 1, std::true_type{});

  // ---------------- epilogue: O * 1/N -> global ----------------
  if constexpr (kDelta) {  // row (local row lr) of out, or with more than one chunk the unscaled fp32 partial
    const DeltaRows dr = delta_rows<Cfg::BM>(p);
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int lr = wgi * 64 + w * 16 + g + hh * 8;
      if (lr >= dr.rows) continue;
      if (gridDim.z > 1) {
        float* prow = p.part + ((dr.part_row + lr) * p.seq.heads + h) * DV;
#pragma unroll
        for (int nb = 0; nb < DV / 8; ++nb)
          *reinterpret_cast<float2*>(prow + nb * 8 + 2 * t4) = make_float2(o[nb * 4 + hh * 2], o[nb * 4 + hh * 2 + 1]);
      } else {
        uint16_t* orow = reinterpret_cast<uint16_t*>(p.out) + (dr.out_row + lr) * p.o_row_stride + (long long)h * p.o_head_stride;
#pragma unroll
        for (int nb = 0; nb < DV / 8; ++nb) {
          const float a = o[nb * 4 + hh * 2] * p.inv_n, c = o[nb * 4 + hh * 2 + 1] * p.inv_n;
          *reinterpret_cast<uint32_t*>(orow + nb * 8 + 2 * t4) = BF16 ? pack_bf16x2(a, c) : pack_f16x2(a, c);
        }
      }
    }
    return;
  }
  const bool out_bf16 = BF16 || p.amax != nullptr;
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int qi = q_base + hh * 8;
    if (qi - m0 < qs.mrows) {
      uint16_t* orow = reinterpret_cast<uint16_t*>(p.out) + (qs.row0 + qi) * p.o_row_stride + (long long)h * p.o_head_stride;
#pragma unroll
      for (int nb = 0; nb < DV / 8; ++nb) {
        float a = o[nb * 4 + hh * 2] * p.inv_n, c = o[nb * 4 + hh * 2 + 1] * p.inv_n;
        if (kScaled) a = scalbnf(a, e_out), c = scalbnf(c, e_out);
        *reinterpret_cast<uint32_t*>(orow + nb * 8 + 2 * t4) = out_bf16 ? pack_bf16x2(a, c) : pack_f16x2(a, c);
      }
    }
  }
}


// ------------------------------------------------------------------------------------------------
// host
// ------------------------------------------------------------------------------------------------
// attn_wgmma_fwd.cu: the key chunks of a delta-q call (sizes only), and the reduction of their fp32 partials into out
int delta_chunks(const hstu_attn_params& p);
int launch_delta_reduce(bool bf16, const float* part, void* out, long long rows, int heads, int d, int chunks,
                        long long o_row_stride, long long o_head_stride, float inv_n, cudaStream_t st);

// kern: the kernel of this DQK / DV / BF16 / kDelta (an instance of attn_fwd_wgmma_body).  f16: the scaled fp16 copies of
// bf16 inputs (the kernel is then the fp16 one), or null.  kDelta: a delta-q call, with the key chunks of delta_chunks and,
// for more than one, the partials in the workspace and delta_reduce_kernel after the attention
template <int DQK, int DV, bool BF16, bool kDelta>
int launch_fwd_wgmma(const hstu_attn_params& p, cudaStream_t st, void (*kern)(FwdParams), const Fp16Operands* f16 = nullptr) {
  using Cfg = FwdCfg<DQK, DV>;
  FwdParams fp;
  memset(&fp, 0, sizeof(fp));
  const int chunks = kDelta ? delta_chunks(p) : 1;
  if (chunks > 1) {
    const size_t need = wgmma_delta_workspace_bytes(p);
    if (p.workspace == nullptr || p.workspace_bytes < need) {
      set_error("hstu_attn_fwd: delta_q workspace of %zu bytes required (got %zu)", need, p.workspace_bytes);
      return HSTU_ERR_WORKSPACE;
    }
    fp.part = reinterpret_cast<float*>(p.workspace);
  }
  const long long q_rows = kDelta ? (long long)p.batch * p.delta_q_len : p.total_rows;
  const Operands o = operands(p, f16);
  if (int e = make_tmap_rows_heads(&fp.tmQ, o.src[0], q_rows, p.heads, DQK, o.rs[0], o.hs[0], Cfg::BOX_COLS, Cfg::BM)) return e;
  if (int e = make_tmap_rows_heads(&fp.tmK, o.src[1], p.total_rows, p.heads, DQK, o.rs[1], o.hs[1], Cfg::BOX_COLS, Cfg::BN)) return e;
  if (int e = make_tmap_rows_heads(&fp.tmV, o.src[2], p.total_rows, p.heads, DV, o.rs[2], o.hs[2], Cfg::BOX_COLS_V, Cfg::BN)) return e;
  if (f16) fp.amax = f16->amax;
  fp.seq = seq_args(p);
  fp.out = p.out;
  fp.o_row_stride = p.o_row_stride;
  fp.o_head_stride = p.o_head_stride;
  fp.inv_n = 1.0f / (float)p.max_seq_len;
  fp.delta = p.delta_q_len;
  HSTU_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
  const dim3 grid = kDelta ? dim3(p.batch * p.heads, (p.delta_q_len + Cfg::BM - 1) / Cfg::BM, chunks)
                           : dim3((p.max_seq_len + Cfg::BM - 1) / Cfg::BM, p.heads, p.batch);
  kern<<<grid, kAttnThreads, Cfg::SMEM_BYTES, st>>>(fp);
  HSTU_CUDA_OK(cudaGetLastError());
  if (chunks > 1) return launch_delta_reduce(BF16, fp.part, p.out, q_rows, p.heads, DV, chunks, p.o_row_stride, p.o_head_stride, fp.inv_n, st);
  return 0;
}

}  // namespace hstu
