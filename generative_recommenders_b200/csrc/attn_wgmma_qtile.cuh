// What the query-stationary wgmma attention kernels share around their MMAs: the bf16 / fp16 forward (attn_wgmma_fwd.cuh),
// the split backward's dQ kernel (attn_wgmma_bwd.cuh) and the fp8 forward (attn_wgmma_fwd_e4m3.cuh).  Each keeps a 128-row
// query tile resident (two warpgroups of 64 rows) and streams the key tiles its rows attend through a ring of K and V
// stages.  Here, once: the sequence arguments and the prologue that turns them into the CTA's rows and key tiles, the K / V
// ring, and the choice of the mask case per tile.  The tile loops (MMA order, waits, what is released when) differ for
// reasons given at each kernel and stay there.
#pragma once
#include <type_traits>

#include "common.cuh"
#include "internal.h"
#include "wgmma.cuh"

namespace hstu {
using namespace wg;

constexpr int kAttnThreads = 256;  // every wgmma attention kernel: two warpgroups

// The jagged layout, head count and mask of a call, as the wgmma attention kernels take them.  (The order keeps the
// pairs of 32-bit fields that the backward kernels read with one 64-bit constant load.)
struct SeqArgs {
  const void* seq_offsets;
  const void* num_targets;
  int offsets_i64, targets_i64;
  int max_seq_len, heads;
  int win, min_full, ctx;
  float alpha_half;  // alpha / 2
};
inline SeqArgs seq_args(const hstu_attn_params& p) {
  return {p.seq_offsets,  p.num_targets,           p.offsets_are_i64,    p.num_targets_are_i64, p.max_seq_len, p.heads,
          p.max_attn_len, p.min_full_attn_seq_len, p.contextual_seq_len, 0.5f * p.alpha};
}

// The CTA's part of sequence b: its first row in the jagged tensors, its length, the valid ones of the CTA's BM query rows,
// its mask, and the BN-row key tiles [t0, t0 + T) that those rows attend (T >= 1: the diagonal tile)
struct QTileSeq {
  long long row0;
  int len, mrows, t0, T;
  SeqMask msk;
};
__device__ __forceinline__ void seq_rows(const SeqArgs& a, int b, QTileSeq* q) {
  const long long row0 = load_index(a.seq_offsets, a.offsets_i64, b);
  q->len = (int)(load_index(a.seq_offsets, a.offsets_i64, b + 1) - row0);
  q->row0 = row0;
}
// First row and length of sequence b for a CTA of query rows from m0 on.  Rows past max_seq_len are ignored on the way in and zero on
// the way out: the CTAs of blockIdx.x == 0 zero them in head h of `out` (d columns, strides in elements).  False: no
// row of the CTA is left.
__device__ __forceinline__ bool qtile_rows(const SeqArgs& a, int b, int h, int m0, void* out, long long row_stride,
                                           long long head_stride, int d, QTileSeq* q) {
  seq_rows(a, b, q);
  if (q->len > a.max_seq_len) {
    if (blockIdx.x == 0) zero_rows(out, 2, row_stride, (long long)h * head_stride, d, q->row0 + a.max_seq_len, q->row0 + q->len);
    q->len = a.max_seq_len;
  }
  return m0 < q->len;
}

// The CTA's valid query rows, of the `rows` left from its first row on, which is at sequence position p0; the mask, and
// the key tiles those rows attend (kBidir: under the non-causal mask, common.cuh)
template <int BM, int BN, bool kBidir = false>
__device__ __forceinline__ void key_tiles(const SeqArgs& a, int b, int p0, int rows, QTileSeq* q) {
  const int n_tgt = a.num_targets ? (int)load_index(a.num_targets, a.targets_i64, b) : -1;
  q->msk = make_seq_mask(q->len, n_tgt, a.win, a.min_full, a.ctx);
  q->mrows = min(BM, rows);
  int lo, hi;
  if constexpr (kBidir) kv_range_for_q_rows_bidir(q->msk, p0, p0 + q->mrows, &lo, &hi);
  else kv_range_for_q_rows(q->msk, p0, p0 + q->mrows, &lo, &hi);
  q->t0 = lo / BN;
  q->T = (hi + BN - 1) / BN - q->t0;
}
// Both, for a CTA whose rows [m0, m0 + BM) sit at their own positions
template <int BM, int BN, bool kBidir = false>
__device__ __forceinline__ bool qtile_prologue(const SeqArgs& a, int b, int h, int m0, void* out, long long row_stride,
                                               long long head_stride, int d, QTileSeq* q) {
  if (!qtile_rows(a, b, h, m0, out, row_stride, head_stride, d, q)) return false;
  key_tiles<BM, BN, kBidir>(a, b, m0, q->len - m0, q);
  return true;
}

// ------------------------------------------------------------------------------------------------
// The K / V ring.  Key tile i of the CTA goes through stage i % STAGES of the K buffers and of the V buffers, each with a
// full barrier (TMA completion) and a release counter.  Thread 0 issues the loads of the kernel's resident operands (q_full)
// and the first STAGES key tiles (fill).  Afterwards nobody waits for a free stage: each warp releases the K (V) stage of
// tile i once its MMAs that read it have completed, and the warp whose release is the last of the eight (release_is_last,
// wgmma.cuh) issues the load of tile i + STAGES into it, so neither warpgroup holds the other back.  A warp waits for tile i
// on the full barrier of stage i % STAGES with parity (i / STAGES) & 1 (RingPos).  No separate producer warp: the accumulators need
// the register budget of a 256-thread block.
// Cfg: BN, STAGES, and for K and V the stage bytes, box bytes, boxes, box columns and offset in shared memory.
// ------------------------------------------------------------------------------------------------
struct QTileBars {
  uint64_t q_full;  // the resident operands: Q, or Q and dO
  uint64_t k_full[3], v_full[3];
  uint32_t k_free[3], v_free[3];  // release counters of the K / V stages (release_is_last: one arrival per warp and use)
};
constexpr std::false_type kKey{};  // selects the K or the V half of the ring
constexpr std::true_type kVal{};

template <class Cfg>
struct KvRing {
  static_assert(Cfg::STAGES <= 3, "QTileBars holds three stages");
  uint8_t* smem;
  const CUtensorMap *tmK, *tmV;
  int h;            // head
  long long row0;   // of the sequence
  int t0, T;        // the CTA's key tiles
  QTileBars* bars;

  // (all threads)
  __device__ __forceinline__ void init() {
    bars = reinterpret_cast<QTileBars*>(smem + Cfg::OFF_BAR);
    if (threadIdx.x == 0) {
      mbar_init(&bars->q_full, 1);
      for (int i = 0; i < Cfg::STAGES; ++i) {
        mbar_init(&bars->k_full[i], 1);
        mbar_init(&bars->v_full[i], 1);
        bars->k_free[i] = bars->v_free[i] = 0u;
      }
      fence_barrier_init();
    }
    __syncthreads();
  }
  // TMA issue of key tile i into its K (kKey) or V (kVal) stage st = i % STAGES
  template <class ValC>
  __device__ __forceinline__ void load(ValC, int i, int st) const {
    constexpr bool kIsV = ValC::value;
    constexpr int bytes = kIsV ? Cfg::V_BYTES : Cfg::K_BYTES, box = kIsV ? Cfg::V_BOX : Cfg::K_BOX;
    constexpr int nbox = kIsV ? Cfg::NBOX_V : Cfg::NBOX, cols = kIsV ? Cfg::BOX_COLS_V : Cfg::BOX_COLS;
    uint64_t* full = kIsV ? bars->v_full : bars->k_full;
    mbar_arrive_expect_tx(&full[st], bytes);
#pragma unroll
    for (int bx = 0; bx < nbox; ++bx)
      tma_load_3d(smem + (kIsV ? Cfg::OFF_V : Cfg::OFF_K) + st * bytes + bx * box, kIsV ? tmV : tmK, &full[st], bx * cols, h,
                  (int)(row0 + (long long)(t0 + i) * Cfg::BN));
  }
  // Until tile i, of ring position (st, ph), has landed in its K (V) stage
  template <class ValC>
  __device__ __forceinline__ void wait(ValC, int st, uint32_t ph) const {
    mbar_wait(ValC::value ? &bars->v_full[st] : &bars->k_full[st], ph);
  }
  // The calling warp no longer reads the K (V) stage st of tile i
  template <class ValC>
  __device__ __forceinline__ void release(ValC val_c, int i, int st) const {
    uint32_t* ctr = ValC::value ? bars->v_free : bars->k_free;
    if ((threadIdx.x & 31) == 0 && i + Cfg::STAGES < T && release_is_last<kAttnThreads / 32>(&ctr[st])) load(val_c, i + Cfg::STAGES, st);
  }
  // (thread 0) the first STAGES key tiles
  __device__ __forceinline__ void fill() const {
    for (int i = 0; i < min(T, Cfg::STAGES); ++i) {
      load(kKey, i, i);
      load(kVal, i, i);
    }
  }
};

// ------------------------------------------------------------------------------------------------
// Mask of one key tile.  The thread holds scores (row q_base + 8 (e >> 1), key n0 + 8 nb + 2 t4 + (e & 1)) at index 4 nb + e
// (the wgmma accumulator layout).  x[n] = f(n) where the pair is valid, else 0.  The case is chosen once per tile -- every
// pair valid (keys below full_lim) / the fast mask with the limits of the thread's two rows hoisted / the general mask --
// outside the score loops, so that each loop is one basic block and ptxas can overlap the tanh (in f) of independent scores
// instead of waiting out each one in turn.
// ------------------------------------------------------------------------------------------------
// Keys below this are valid for every query row at positions >= p0 (fast mask; none otherwise)
__device__ __forceinline__ int full_valid_limit(const SeqMask& msk, int p0) {
  return msk.fast != 0 ? min(p0, msk.has_tgt ? msk.max_id : 0x7fffffff) : -1;
}
template <int BN, class F>
__device__ __forceinline__ void mask_scores(const SeqMask& msk, bool fast, int full_lim, int len, int q_base, int n0, int t4, float (&x)[BN / 2], F f) {
  if (n0 + BN <= full_lim) {  // tile-uniform: every pair valid
#pragma unroll
    for (int n = 0; n < BN / 2; ++n) x[n] = f(n);
  } else if (fast) {
    // mask_valid of the fast mask, kj < min(qi, max_id) || kj == qi
    int lim[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) lim[hh] = msk.has_tgt ? min(q_base + hh * 8, msk.max_id) : q_base + hh * 8;
#pragma unroll
    for (int nb = 0; nb < BN / 8; ++nb)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int qi = q_base + (e >> 1) * 8, kj = n0 + nb * 8 + 2 * t4 + (e & 1);
        const float v = f(nb * 4 + e);
        x[nb * 4 + e] = (kj < len && (kj < lim[e >> 1] || kj == qi)) ? v : 0.f;
      }
  } else {
#pragma unroll
    for (int nb = 0; nb < BN / 8; ++nb)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int qi = q_base + (e >> 1) * 8, kj = n0 + nb * 8 + 2 * t4 + (e & 1);
        const float v = f(nb * 4 + e);
        x[nb * 4 + e] = (kj < len && mask_valid(msk, qi, kj)) ? v : 0.f;
      }
  }
}

// The same under the non-causal mask, for the CTA's query rows [q_lo, q_hi).  Cases, chosen once per tile: every pair valid
// (bidir_block_all_valid: no target x target pair, and with a window every id distance within it) / no window: only the
// target x target pairs off the diagonal are masked (keys and rows below t_first = target_start are never) / the general
// mask (window edges, degenerate sequences).
template <int BN, class F>
__device__ __forceinline__ void mask_scores_bidir(const SeqMask& msk, int len, int q_lo, int q_hi, int q_base, int n0, int t4,
                                                  float (&x)[BN / 2], F f) {
  if (n0 + BN <= len && bidir_block_all_valid(msk, q_lo, q_hi, n0, n0 + BN)) {
#pragma unroll
    for (int n = 0; n < BN / 2; ++n) x[n] = f(n);
  } else if (msk.win == 0 && msk.max_id >= 1) {
    const int t_first = target_start(msk);
    bool row_hist[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) row_hist[hh] = q_base + hh * 8 < t_first;
#pragma unroll
    for (int nb = 0; nb < BN / 8; ++nb)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int qi = q_base + (e >> 1) * 8, kj = n0 + nb * 8 + 2 * t4 + (e & 1);
        const float v = f(nb * 4 + e);
        x[nb * 4 + e] = (kj < len && (row_hist[e >> 1] || kj < t_first || kj == qi)) ? v : 0.f;
      }
  } else {
#pragma unroll
    for (int nb = 0; nb < BN / 8; ++nb)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int qi = q_base + (e >> 1) * 8, kj = n0 + nb * 8 + 2 * t4 + (e & 1);
        const float v = f(nb * 4 + e);
        x[nb * 4 + e] = (kj < len && mask_valid_bidir(msk, qi, kj)) ? v : 0.f;
      }
  }
}

// ------------------------------------------------------------------------------------------------
// host
// ------------------------------------------------------------------------------------------------
// SMs of an H100 SXM: the grid caps of the grid-strided helper kernels and the delta-q chunk sizing (any grid is correct)
constexpr int kH100Sms = 132;

// The q, k, v, dO views the kernels read: the inputs, or their contiguous scaled fp16 copies (f16, bf16 at d = 32)
struct Operands {
  const void* src[4];
  long long rs[4], hs[4];  // row / head strides (elements)
};
inline Operands operands(const hstu_attn_params& p, const Fp16Operands* f16) {
  Operands o = {{p.q, p.k, p.v, p.dout},
                {p.q_row_stride, p.k_row_stride, p.v_row_stride, p.do_row_stride},
                {p.q_head_stride, p.k_head_stride, p.v_head_stride, p.do_head_stride}};
  if (f16)
    for (int i = 0; i < 4; ++i) o.src[i] = f16->copy[i], o.rs[i] = (long long)p.heads * p.dqk, o.hs[i] = p.dqk;
  return o;
}

// Runs launch.template operator()<B>(f16), which launches the kernels of dtype B (bf16 if B) on the operands f16 (null: the
// inputs).  bf16 at d = 32 runs the fp16 kernels on exactly scaled copies that fp16_operands_prepass writes first (DESIGN.md
// 3.0); every other call runs the kernels of its own dtype on its inputs.  The bf16 kernels at d = 32 are never named here,
// so they are never instantiated.
template <int D, bool BF16, class Launch>
int launch_on_operands(const hstu_attn_params& p, bool bwd, cudaStream_t st, Launch&& launch) {
  if constexpr (scaled_fp16_dims(BF16, D, D)) {
    Fp16Operands f16;
    if (int e = fp16_operands_prepass(p, bwd, &f16, st)) return e;
    return launch.template operator()<false>(&f16);
  } else {
    return launch.template operator()<BF16>(nullptr);
  }
}

}  // namespace hstu
