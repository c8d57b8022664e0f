// Jagged HSTU attention forward on the Hopper warpgroup tensor cores (wgmma) with TMA-staged tiles.  bf16 / fp16,
// dqk == dv in {32, 64, 128, 256}.
//
// One CTA per (128-row query tile, head, sequence); heavy (late) query tiles are scheduled first.  Two warpgroups
// of 64 query rows each.  Per key tile:
//   S = Q K^T            (wgmma, A = Q and B = K both K-major in shared memory, fp32 accumulators)
//   P = silu(alpha S) * mask   (one tanh per score, in registers)
//   O += P V             (wgmma, A = P from registers, B = V MN-major in shared memory)
// Key tiles of 64 rows keep a thread at <= 128 registers for d <= 64, so two CTAs share an SM there.
// Each warpgroup waits for its own MMAs; the two warpgroups overlap each other's tensor-core and elementwise phases.
// Thread 0 issues the TMA loads: Q once, then the K and V tiles through a ring of STAGES buffers each; a stage is refilled
// once all 256 threads have released it (the MMAs that read it have completed).  No separate producer warp: the 64 x d
// fp32 O accumulator (d = 256: 128 registers per thread) needs the register budget of a 256-thread block.
// P is a 16-bit MMA operand of the same format as V (wgmma takes one format for A and B): fp16 for fp16 inputs, and for
// bf16 inputs a hi + lo pair of bf16 operands multiplied twice (wgmma.cuh, Operand), so that its rounding stays well inside
// the 1e-3 parity budget.  The 1/N factor of the reference is applied once in the epilogue (registers -> global, rows past
// the sequence end are not written).  Rows of neighbouring sequences that a TMA box drags in are neutralised by the mask.
//
// Reference semantics: ops/pytorch/pt_hstu_attention.py:130-171; tile skipping mirrors the idea of
// ops/triton/triton_hstu_attention.py:517-543 (loop bounds from the mask) but is derived from common.cuh's ranges.
#include <string.h>

#include "common.cuh"
#include "internal.h"
#include "wgmma.cuh"

namespace hstu {
using namespace wg;

struct alignas(64) FwdParams {
  CUtensorMap tmQ, tmK, tmV;
  const void* seq_offsets;
  const void* num_targets;
  void* out;
  long long o_row_stride, o_head_stride;
  int offsets_i64, targets_i64;
  int max_seq_len;
  int win, min_full, ctx;
  float alpha_half;  // alpha / 2
  float inv_n;       // 1 / max_seq_len
};

template <int D>
struct FwdCfg {
  static constexpr int BM = 128;                     // query rows per CTA (two warpgroups of 64)
  static constexpr int BN = 64;                      // key rows per tile
  static constexpr int SW = (D * 2 >= 128) ? 128 : D * 2;  // swizzle width (bytes) of the Q/K/V boxes
  static constexpr int BOX_COLS = SW / 2;
  static constexpr int Q_BOX = BM * SW;
  static constexpr int KV_BOX = BN * SW;
  static constexpr int Q_BYTES = BM * D * 2;
  static constexpr int KV_BYTES = BN * D * 2;
  static constexpr int NBOX = D / BOX_COLS;
  static constexpr int STAGES = (D == 256) ? 2 : 3;
  static constexpr int OFF_Q = 0;
  static constexpr int OFF_K = OFF_Q + Q_BYTES;
  static constexpr int OFF_V = OFF_K + STAGES * KV_BYTES;
  static constexpr int OFF_BAR = OFF_V + STAGES * KV_BYTES;
  static constexpr int SMEM_BYTES = OFF_BAR + 256 + 1024;  // + barriers + alignment slack
  static_assert(SMEM_BYTES <= 232448, "shared memory budget");
};
constexpr int kFwdThreads = 256;
template <int D> constexpr int kFwdMinBlocks = (D <= 64) ? 2 : 1;  // d <= 64: two CTAs per SM (<= 128 registers per thread)

struct FwdBars {
  uint64_t q_full;
  uint64_t k_full[3], v_full[3], k_empty[3], v_empty[3];
};

template <int D, bool BF16>
__global__ void __launch_bounds__(kFwdThreads, kFwdMinBlocks<D>) attn_fwd_wgmma_kernel(const __grid_constant__ FwdParams p) {
  using Cfg = FwdCfg<D>;
  constexpr int SW = Cfg::SW, BN = Cfg::BN, NST = Cfg::STAGES;
  const int b = blockIdx.z, h = blockIdx.y;
  const int m0 = (int)(gridDim.x - 1 - blockIdx.x) * Cfg::BM;
  const long long row0 = load_index(p.seq_offsets, p.offsets_i64, b);
  int len = (int)(load_index(p.seq_offsets, p.offsets_i64, b + 1) - row0);
  if (len > p.max_seq_len) {  // rows past max_seq_len are ignored on the way in and zero on the way out
    if (blockIdx.x == 0) zero_rows(p.out, 2, p.o_row_stride, (long long)h * p.o_head_stride, D, row0 + p.max_seq_len, row0 + len);
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
  FwdBars* bars = reinterpret_cast<FwdBars*>(smem + Cfg::OFF_BAR);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (tid == 0) {
    mbar_init(&bars->q_full, 1);
    for (int i = 0; i < NST; ++i) {
      mbar_init(&bars->k_full[i], 1);
      mbar_init(&bars->v_full[i], 1);
      mbar_init(&bars->k_empty[i], 256);
      mbar_init(&bars->v_empty[i], 256);
    }
    fence_barrier_init();
  }
  __syncthreads();

  // TMA issue (thread 0): Q and the first STAGES key tiles now; stage st is refilled once both warpgroups have released it
  auto load_kv = [&](int i) {
    const int st = i % NST;
    const int kv_row = (int)(row0 + (long long)(t0 + i) * BN);
    if (i >= NST) mbar_wait(&bars->k_empty[st], ((i / NST) - 1) & 1);
    mbar_arrive_expect_tx(&bars->k_full[st], Cfg::KV_BYTES);
#pragma unroll
    for (int bx = 0; bx < Cfg::NBOX; ++bx)
      tma_load_3d(smem + Cfg::OFF_K + st * Cfg::KV_BYTES + bx * Cfg::KV_BOX, &p.tmK, &bars->k_full[st], bx * Cfg::BOX_COLS, h, kv_row);
    if (i >= NST) mbar_wait(&bars->v_empty[st], ((i / NST) - 1) & 1);
    mbar_arrive_expect_tx(&bars->v_full[st], Cfg::KV_BYTES);
#pragma unroll
    for (int bx = 0; bx < Cfg::NBOX; ++bx)
      tma_load_3d(smem + Cfg::OFF_V + st * Cfg::KV_BYTES + bx * Cfg::KV_BOX, &p.tmV, &bars->v_full[st], bx * Cfg::BOX_COLS, h, kv_row);
  };
  if (tid == 0) {
    prefetch_tensormap(&p.tmQ);
    prefetch_tensormap(&p.tmK);
    prefetch_tensormap(&p.tmV);
    mbar_arrive_expect_tx(&bars->q_full, Cfg::Q_BYTES);
#pragma unroll
    for (int bx = 0; bx < Cfg::NBOX; ++bx)
      tma_load_3d(smem + Cfg::OFF_Q + bx * Cfg::Q_BOX, &p.tmQ, &bars->q_full, bx * Cfg::BOX_COLS, h, (int)(row0 + m0));
    for (int i = 0; i < min(T, NST); ++i) load_kv(i);
  }
  __syncwarp();

  const int wgi = warp >> 2, w = warp & 3, g = lane >> 2, t4 = lane & 3;
  const int q_base = m0 + wgi * 64 + w * 16 + g;  // query position of accumulator rows g (+ 8)
  const uint32_t sq = smem_u32(smem + Cfg::OFF_Q) + wgi * 64 * SW;
  const uint32_t sk = smem_u32(smem + Cfg::OFF_K), sv = smem_u32(smem + Cfg::OFF_V);
  const bool fast = msk.fast != 0;
  const int full_lim = fast ? min(m0, msk.has_tgt ? msk.max_id : 0x7fffffff) : -1;  // keys < full_lim: valid for every row

  float o[D / 2];
#pragma unroll
  for (int e = 0; e < D / 2; ++e) o[e] = 0.f;
  uint32_t a_hi[BN / 16][4], a_lo[BN / 16][4];
#pragma unroll
  for (int kk = 0; kk < BN / 16; ++kk)
#pragma unroll
    for (int r = 0; r < 4; ++r) a_hi[kk][r] = a_lo[kk][r] = 0u;
  mbar_wait(&bars->q_full, 0);
  for (int i = 0; i < T; ++i) {
    const int st = i % NST;
    const uint32_t ph = (i / NST) & 1;
    mbar_wait(&bars->k_full[st], ph);
    float s[BN / 2];
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < D / 16; ++ks) {
      const int kb = ks * 32, bx = kb / SW, off = kb % SW;
      wgmma_ss<BN, BF16, 0, 0>(s, desc_kmajor<SW>(sq + bx * Cfg::Q_BOX, off),
                               desc_kmajor<SW>(sk + st * Cfg::KV_BYTES + bx * Cfg::KV_BOX, off), ks > 0);
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(s);
    mbar_arrive(&bars->k_empty[st]);

    const int n0 = (t0 + i) * BN;
    const bool full = n0 + BN <= full_lim;  // tile-uniform
#pragma unroll
    for (int nb = 0; nb < BN / 8; ++nb)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float x = s[nb * 4 + e] * p.alpha_half;
        float pv = __fmaf_rn(x, tanh_approx(x), x);  // silu(2x) = x (1 + tanh x)
        if (!full) {
          const int qi = q_base + (e >> 1) * 8, kj = n0 + nb * 8 + 2 * t4 + (e & 1);
          pv = (kj < len && mask_valid(msk, qi, kj)) ? pv : 0.f;
        }
        s[nb * 4 + e] = pv;
      }
#pragma unroll
    for (int kk = 0; kk < BN / 16; ++kk) {
      const Operand<BF16> x0(s[8 * kk + 0], s[8 * kk + 1]), x1(s[8 * kk + 2], s[8 * kk + 3]);
      const Operand<BF16> x2(s[8 * kk + 4], s[8 * kk + 5]), x3(s[8 * kk + 6], s[8 * kk + 7]);
      a_hi[kk][0] = x0.hi; a_hi[kk][1] = x1.hi; a_hi[kk][2] = x2.hi; a_hi[kk][3] = x3.hi;
      a_lo[kk][0] = x0.lo; a_lo[kk][1] = x1.lo; a_lo[kk][2] = x2.lo; a_lo[kk][3] = x3.lo;
    }
    mbar_wait(&bars->v_full[st], ph);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < BN / 16; ++kk) {
      const uint64_t vd = desc_mnmajor<SW>(sv + st * Cfg::KV_BYTES, kk * 16, Cfg::KV_BOX);
      wgmma_rs<D, BF16, 1>(o, a_hi[kk], vd, 1);
      if constexpr (BF16) wgmma_rs<D, BF16, 1>(o, a_lo[kk], vd, 1);
    }
    wgmma_commit();
    wgmma_wait<0>();  // an MMA batch never stays in flight across the elementwise code (ptxas would serialise them)
    fence_regs(o);
    fence_regs(a_hi);
    fence_regs(a_lo);
    mbar_arrive(&bars->v_empty[st]);
    if (tid == 0 && i + NST < T) load_kv(i + NST);  // K and V of tile i are no longer read
    __syncwarp();
  }

  // ---------------- epilogue: O * 1/N -> global ----------------
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int qi = q_base + hh * 8;
    if (qi - m0 < mrows) {
      uint16_t* orow = reinterpret_cast<uint16_t*>(p.out) + (row0 + qi) * p.o_row_stride + (long long)h * p.o_head_stride;
#pragma unroll
      for (int nb = 0; nb < D / 8; ++nb) {
        const float a = o[nb * 4 + hh * 2] * p.inv_n, c = o[nb * 4 + hh * 2 + 1] * p.inv_n;
        *reinterpret_cast<uint32_t*>(orow + nb * 8 + 2 * t4) = BF16 ? pack_bf16x2(a, c) : pack_f16x2(a, c);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// host
// ------------------------------------------------------------------------------------------------
bool is_sm90() {
  static int cached = -1;
  if (cached < 0) {
    int dev = 0;
    cudaDeviceProp prop;
    cached = (cudaGetDevice(&dev) == cudaSuccess && cudaGetDeviceProperties(&prop, dev) == cudaSuccess && prop.major == 9) ? 1 : 0;
  }
  return cached == 1;
}

bool aligned_view(const void* ptr, long long row_stride, long long head_stride) {
  return (reinterpret_cast<uintptr_t>(ptr) & 15) == 0 && (row_stride % 8) == 0 && (head_stride % 8) == 0;
}

bool wgmma_fwd_supported(const hstu_attn_params& p) {
  if (p.dtype != HSTU_BF16 && p.dtype != HSTU_F16) return false;
  if (p.dqk != p.dv || (p.dqk != 32 && p.dqk != 64 && p.dqk != 128 && p.dqk != 256)) return false;
  if (p.delta_q_len != 0 || p.pos_w != nullptr || p.ts_w != nullptr) return false;
  if (p.total_rows >= (1ll << 31) - 256) return false;
  if (!aligned_view(p.q, p.q_row_stride, p.q_head_stride) || !aligned_view(p.k, p.k_row_stride, p.k_head_stride) ||
      !aligned_view(p.v, p.v_row_stride, p.v_head_stride) || !aligned_view(p.out, p.o_row_stride, p.o_head_stride))
    return false;
  return is_sm90();
}

template <int D, bool BF16>
static int launch_fwd_wgmma(const hstu_attn_params& p, cudaStream_t st) {
  using Cfg = FwdCfg<D>;
  FwdParams fp;
  memset(&fp, 0, sizeof(fp));
  if (int e = make_tmap_rows_heads(&fp.tmQ, p.q, p.total_rows, p.heads, D, p.q_row_stride, p.q_head_stride, Cfg::BOX_COLS, Cfg::BM)) return e;
  if (int e = make_tmap_rows_heads(&fp.tmK, p.k, p.total_rows, p.heads, D, p.k_row_stride, p.k_head_stride, Cfg::BOX_COLS, Cfg::BN)) return e;
  if (int e = make_tmap_rows_heads(&fp.tmV, p.v, p.total_rows, p.heads, D, p.v_row_stride, p.v_head_stride, Cfg::BOX_COLS, Cfg::BN)) return e;
  fp.seq_offsets = p.seq_offsets;
  fp.num_targets = p.num_targets;
  fp.out = p.out;
  fp.o_row_stride = p.o_row_stride;
  fp.o_head_stride = p.o_head_stride;
  fp.offsets_i64 = p.offsets_are_i64;
  fp.targets_i64 = p.num_targets_are_i64;
  fp.max_seq_len = p.max_seq_len;
  fp.win = p.max_attn_len;
  fp.min_full = p.min_full_attn_seq_len;
  fp.ctx = p.contextual_seq_len;
  fp.alpha_half = 0.5f * p.alpha;
  fp.inv_n = 1.0f / (float)p.max_seq_len;
  auto kern = attn_fwd_wgmma_kernel<D, BF16>;
  HSTU_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
  dim3 grid((p.max_seq_len + Cfg::BM - 1) / Cfg::BM, p.heads, p.batch);
  kern<<<grid, kFwdThreads, Cfg::SMEM_BYTES, st>>>(fp);
  HSTU_CUDA_OK(cudaGetLastError());
  return 0;
}

int attn_wgmma_fwd(const hstu_attn_params& p, cudaStream_t st) {
  const bool bf = p.dtype == HSTU_BF16;
  switch (p.dqk) {
    case 32: return bf ? launch_fwd_wgmma<32, true>(p, st) : launch_fwd_wgmma<32, false>(p, st);
    case 64: return bf ? launch_fwd_wgmma<64, true>(p, st) : launch_fwd_wgmma<64, false>(p, st);
    case 128: return bf ? launch_fwd_wgmma<128, true>(p, st) : launch_fwd_wgmma<128, false>(p, st);
    case 256: return bf ? launch_fwd_wgmma<256, true>(p, st) : launch_fwd_wgmma<256, false>(p, st);
  }
  set_error("wgmma forward: unsupported head dim %d", p.dqk);
  return HSTU_ERR_UNSUPPORTED;
}

}  // namespace hstu
