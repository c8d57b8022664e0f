// KV-cached (delta-q) HSTU attention forward with 16-bit (bf16 / fp16) queries and output over a float8 e4m3 K / V cache
// with per (sequence, head) descales, on the Hopper warpgroup tensor cores (DESIGN.md 3.8):
//
//   out = delta_attention(q, k * kd[b, h], v * vd[b, h])
//
// Geometry of the 16-bit delta-q kernel (attn_wgmma_fwd.cuh, kDelta): grid (sequence x head, 128-row query tile, key chunk),
// query row i of sequence b at position len - delta + i, the whole unclipped sequence as keys, an even split of the key tiles
// over the chunks, and with more than one chunk fp32 partials that delta_reduce_kernel sums unchanged.  What differs:
//   - TMA brings each 64-key tile of K and V in as e4m3 bytes, through a ring of byte stages (Cfg::STAGES) (one full barrier per
//     stage for both).  All 256 threads widen it into ONE 16-bit tile per operand, in the swizzled layout that the 16-bit
//     kernel's descriptors read (K K-major, V MN-major): bf16 for bf16 queries, fp16 for fp16 queries.  The widening is exact
//     (every e4m3 value is a normal fp16 and a bf16 value; NaN stays NaN; e4m3fn has no Inf).  Each writer fences
//     (fence.proxy.async) before the CTA barrier that precedes the MMAs reading the tile.
//   - One 16-bit buffer per operand: V_i is widened after S_i = Q K_i^T has completed, and K_{i+1} while O += P_i V_i runs
//     (after it for bf16 at dv <= 64).  Two CTA barriers per tile separate the uses.
//   - V rows past the sequence end are written as zeros by the widening itself (P = 0 does not neutralise a NaN in V); K rows
//     there only reach scores that the mask replaces by 0.
//   - S and P V are the 16-bit kernel's MMAs (bf16: hi / lo split of P; fp16: one fp16 P).  kd is folded into the score
//     scalars from the frexp mantissas and exponents, as in attn_fwd_e4m3_body: the tanh argument is alpha/2 kd S, and P is
//     formed as P' = 2^-e_k P (e_k the exponent of kd), so P' has the magnitude of the unscaled scores whatever kd is, and the
//     output scale (1/N) vd 2^e_k is applied as a normal mantissa and an exact power of two.  Partials carry vd 2^e_k.
// The warpgroup of padding rows (delta <= 64) issues no MMA; it widens its half of every tile.
#include "attn_wgmma_fwd.cuh"
#include "attn_wgmma_fwd_e4m3.cuh"

namespace hstu {
using namespace wg;

struct alignas(64) DeltaFp8KvParams {
  CUtensorMap tmQ, tmK, tmV;  // Q: the 16-bit queries; K, V: the e4m3 cache (bytes)
  SeqArgs seq;
  void* out;
  long long o_row_stride, o_head_stride;
  const float* descale[2];  // k, v: [B, H] fp32, or null (= 1)
  long long ds_batch[2], ds_head[2];
  float inv_n;  // 1 / max_seq_len
  int delta;
  float* part;  // with gridDim.z > 1 key chunks: the fp32 partials [chunks, B * delta, H, DV], multiplied by vd
};

template <int DQK, int DV>
struct DeltaFp8KvCfg {
  static constexpr int BM = 128, BN = 64;
  static constexpr int SW = swizzle_bytes(DQK), SWV = swizzle_bytes(DV);            // 16-bit Q / K and V tiles
  static constexpr int SWK8 = swizzle_bytes(DQK, 1), SWV8 = swizzle_bytes(DV, 1);  // e4m3 K and V boxes
  static constexpr int BOX_COLS = SW / 2;
  static constexpr int NBOX = DQK / BOX_COLS, NBOX_K8 = DQK / SWK8, NBOX_V8 = DV / SWV8;
  static constexpr int Q_BOX = BM * SW, K_BOX = BN * SW, V_BOX = BN * SWV, K8_BOX = BN * SWK8, V8_BOX = BN * SWV8;
  static constexpr int Q_BYTES = BM * DQK * 2, K_BYTES = BN * DQK * 2, V_BYTES = BN * DV * 2;
  static constexpr int K8_BYTES = BN * DQK, V8_BYTES = BN * DV, STAGE_BYTES = K8_BYTES + V8_BYTES;
  // byte stages: d = 256 takes 64 KB of Q + 64 KB of widened K / V + 3 x 32 KB = 224 KB; (128, 256) 32 + 48 + 4 x 24 = 176 KB
  static constexpr int STAGES = DQK == 256 ? 3 : 4;
  static constexpr int OFF_Q = 0;
  static constexpr int OFF_K = OFF_Q + Q_BYTES;
  static constexpr int OFF_V = OFF_K + K_BYTES;
  static constexpr int OFF_B = OFF_V + V_BYTES;
  static constexpr int OFF_BAR = OFF_B + STAGES * STAGE_BYTES;
  static constexpr int SMEM_BYTES = OFF_BAR + 64 + 1024;  // + barriers + alignment slack
  static_assert(SMEM_BYTES <= 232448, "shared memory budget");
  static_assert(OFF_K % 1024 == 0 && OFF_V % 1024 == 0 && OFF_B % 1024 == 0 && K8_BYTES % 1024 == 0 && V8_BYTES % 1024 == 0,
                "swizzle atom alignment");
  static_assert(DQK <= DV, "dqk > dv has no instantiation");
};

// Two e4m3 codes (the low 16 bits) -> two 16-bit values, exactly: e4m3 -> fp16 in hardware (a normal fp16 for every finite
// code, NaN -> NaN), and for bf16 fp16 -> fp32 -> bf16, exact as well (3 significand bits, exponents in [-9, 8])
template <bool BF16>
__device__ __forceinline__ uint32_t widen_e4m3x2(uint32_t codes) {
  uint32_t h2;
  asm("{\n.reg .b16 c;\ncvt.u16.u32 c, %1;\ncvt.rn.f16x2.e4m3x2 %0, c;\n}" : "=r"(h2) : "r"(codes));
  if constexpr (BF16) {
    float a, b;
    asm("{\n.reg .f16 x, y;\nmov.b32 {x, y}, %2;\ncvt.f32.f16 %0, x;\ncvt.f32.f16 %1, y;\n}" : "=f"(a), "=f"(b) : "r"(h2));
    return pack_bf16x2(a, b);
  } else {
    return h2;
  }
}

// The e4m3 [BN][D] tile at src (boxes of SW8 bytes per row) -> the 16-bit [BN][D] tile at dst (boxes of SW16 bytes per row),
// both swizzled; rows >= rows_valid are written as zeros.  All kAttnThreads threads, 8 elements (8 bytes in, 16 out) per
// step; consecutive threads take consecutive 8-column chunks of a row, so each quarter warp stores one 128-byte line and
// each half warp loads one.
template <int BN, int D, int SW8, int SW16, bool BF16>
__device__ __forceinline__ void widen_tile(const uint8_t* src, uint8_t* dst, int rows_valid) {
  constexpr int kPerRow = D / 8, kChunks = BN * kPerRow;
  static_assert(kChunks % kAttnThreads == 0, "whole steps");
#pragma unroll 1  // one step's values live at a time: the widening runs next to the O accumulator and P
  for (int k = 0; k < kChunks / kAttnThreads; ++k) {
    const int c = k * kAttnThreads + (int)threadIdx.x;
    const int r = c / kPerRow, col = (c % kPerRow) * 8;
    const uint8_t* s = src + (col / SW8) * (BN * SW8) + swizzled_chunk_offset<SW8>(r, (col % SW8) / 16) + (col % 16);
    uint8_t* d = dst + (col / (SW16 / 2)) * (BN * SW16) + swizzled_chunk_offset<SW16>(r, (col % (SW16 / 2)) / 8);
    uint4 w = make_uint4(0u, 0u, 0u, 0u);
    if (r < rows_valid) {
      const uint2 b = *reinterpret_cast<const uint2*>(s);
      w = make_uint4(widen_e4m3x2<BF16>(b.x), widen_e4m3x2<BF16>(b.x >> 16), widen_e4m3x2<BF16>(b.y), widen_e4m3x2<BF16>(b.y >> 16));
    }
    *reinterpret_cast<uint4*>(d) = w;
  }
}

template <int DQK, int DV, bool BF16>
__device__ __forceinline__ void attn_fwd_delta_fp8kv_body(const DeltaFp8KvParams& p) {
  using Cfg = DeltaFp8KvCfg<DQK, DV>;
  constexpr int SW = Cfg::SW, SWV = Cfg::SWV, BN = Cfg::BN, NST = Cfg::STAGES;
  // K_{i+1} is widened while O += P_i V_i runs, except for bf16 at dv <= 64, where the P hi / lo fragments in flight next to
  // it would spill within the 128 registers of two CTAs per SM
  constexpr bool kWidenUnderPV = !(BF16 && DV <= 64);
  const int b = (int)blockIdx.x / p.seq.heads, h = (int)blockIdx.x % p.seq.heads;
  const int m0 = (int)blockIdx.y * Cfg::BM;
  // the row of q / out, and of the partials of chunk blockIdx.z, of local query row 0 (recomputed where needed, so that
  // neither stays live through the key loop)
  auto out_row = [&]() { return (long long)b * p.delta + m0; };
  auto part_row = [&]() { return (long long)blockIdx.z * (gridDim.x / p.seq.heads) * p.delta + out_row(); };
  QTileSeq qs;
  seq_rows(p.seq, b, &qs);
  const int p0 = qs.len - p.delta + m0;  // sequence position of query row m0
  key_tiles<Cfg::BM, BN>(p.seq, b, p0, p.delta - m0, &qs);
  {  // chunk blockIdx.z of gridDim.z even shares of whole tiles; an empty share writes zeros
    const int per = (qs.T + (int)gridDim.z - 1) / (int)gridDim.z;
    qs.t0 += (int)blockIdx.z * per;
    qs.T = min(per, qs.T - (int)blockIdx.z * per);
    if (qs.T <= 0) {
      for (int idx = threadIdx.x; idx < qs.mrows * DV; idx += kAttnThreads) {
        if (gridDim.z > 1) p.part[((part_row() + idx / DV) * p.seq.heads + h) * DV + idx % DV] = 0.f;
        else reinterpret_cast<uint16_t*>(p.out)[(out_row() + idx / DV) * p.o_row_stride + (long long)h * p.o_head_stride + idx % DV] = 0;
      }
      return;
    }
  }

  uint8_t* smem = dyn_smem_1k();
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::OFF_BAR);  // [0]: Q; [1 + s]: byte stage s (K and V)
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (tid == 0) {
    mbar_init(&bars[0], 1);
    for (int s = 0; s < NST; ++s) mbar_init(&bars[1 + s], 1);
    fence_barrier_init();
  }
  __syncthreads();
  const int key_row0 = (int)(qs.row0 + (long long)qs.t0 * BN);  // rows < 2^31 - 256 (checked on the host)
  // (thread 0) key tile j into byte stage j % NST
  auto load_bytes = [&](int j) {
    const int st = j % NST;
    uint8_t* base = smem + Cfg::OFF_B + st * Cfg::STAGE_BYTES;
    mbar_arrive_expect_tx(&bars[1 + st], Cfg::STAGE_BYTES);
#pragma unroll
    for (int bx = 0; bx < Cfg::NBOX_K8; ++bx)
      tma_load_3d(base + bx * Cfg::K8_BOX, &p.tmK, &bars[1 + st], bx * Cfg::SWK8, h, key_row0 + j * BN);
#pragma unroll
    for (int bx = 0; bx < Cfg::NBOX_V8; ++bx)
      tma_load_3d(base + Cfg::K8_BYTES + bx * Cfg::V8_BOX, &p.tmV, &bars[1 + st], bx * Cfg::SWV8, h, key_row0 + j * BN);
  };
  if (tid == 0) {
    prefetch_tensormap(&p.tmQ);
    prefetch_tensormap(&p.tmK);
    prefetch_tensormap(&p.tmV);
    mbar_arrive_expect_tx(&bars[0], Cfg::Q_BYTES);
#pragma unroll
    for (int bx = 0; bx < Cfg::NBOX; ++bx)
      tma_load_3d(smem + Cfg::OFF_Q + bx * Cfg::Q_BOX, &p.tmQ, &bars[0], bx * Cfg::BOX_COLS, h, (int)out_row());
    for (int j = 0; j < min(qs.T, NST); ++j) load_bytes(j);
  }
  // widening of K_j (after waiting for its stage) and of V_j (whose stage the caller has waited for with K_j's)
  auto widen_k = [&](int j) {
    mbar_wait(&bars[1 + j % NST], (j / NST) & 1);
    widen_tile<BN, DQK, Cfg::SWK8, SW, BF16>(smem + Cfg::OFF_B + (j % NST) * Cfg::STAGE_BYTES, smem + Cfg::OFF_K, BN);
    fence_proxy_async_smem();  // generic-proxy writes -> the MMAs (async proxy), after the CTA barrier that follows
  };
  auto widen_v = [&](int j) {
    widen_tile<BN, DV, Cfg::SWV8, SWV, BF16>(smem + Cfg::OFF_B + (j % NST) * Cfg::STAGE_BYTES + Cfg::K8_BYTES,
                                              smem + Cfg::OFF_V, qs.len - (qs.t0 + j) * BN);
    fence_proxy_async_smem();
  };
  widen_k(0);
  __syncthreads();

  const int wgi = warp >> 2, w = warp & 3, g = lane >> 2, t4 = lane & 3;
  if (wgi * 64 >= qs.mrows) {
    // a warpgroup of padding rows only (delta <= 64): no MMA, no tanh, no output; it widens its half of every tile, between
    // the same two CTA barriers per tile as the MMA warpgroup
    for (int i = 0; i < qs.T; ++i) {
      widen_v(i);
      __syncthreads();
      if (i + 1 < qs.T) widen_k(i + 1);
      __syncthreads();
    }
    return;
  }
  const int q_base = p0 + wgi * 64 + w * 16 + g;  // query position of accumulator rows g (+ 8)
  const bool rows_idle = wgi * 64 + w * 16 >= qs.mrows;  // a warp whose 16 rows all lie past delta: P = 0
  // (not pinned: descriptors held in registers through the loop would spill at dv = 64 with bf16 queries)
  const uint64_t dq0 = desc_kmajor<SW>(smem_u32(smem + Cfg::OFF_Q) + wgi * 64 * SW, 0);
  const uint64_t dk0 = desc_kmajor<SW>(smem_u32(smem + Cfg::OFF_K), 0);
  const uint64_t dv0 = desc_mnmajor<SWV>(smem_u32(smem + Cfg::OFF_V), 0, Cfg::V_BOX);
  const bool fast = qs.msk.fast != 0;
  const int full_lim = full_valid_limit(qs.msk, p0);
  // c_s = alpha/2 kd scales the tanh argument; c_sp = alpha/2 kd 2^-e_k forms P' = 2^-e_k P (module comment)
  int ea, ek;
  const float m_s = frexpf(p.seq.alpha_half, &ea) * frexpf(load_descale(p.descale[0], p.ds_batch[0], p.ds_head[0], b, h), &ek);
  const float c_s = scalbnf(m_s, ea + ek), c_sp = scalbnf(m_s, ea);

  float o[DV / 2];
#pragma unroll
  for (int e = 0; e < DV / 2; ++e) o[e] = 0.f;
  uint32_t a_hi[BN / 16][4], a_lo[BN / 16][4];
  float s[BN / 2];
  mbar_wait(&bars[0], 0);
  for (int i = 0; i < qs.T; ++i) {
    const int n0 = (qs.t0 + i) * BN;
    // S_i = Q K_i^T, then the widening of V_i (widening under these MMAs crashes ptxas 12.9 at fp16, d = 32 and 64)
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < DQK / 16; ++ks) {
      const int kb = ks * 32, bx = kb / SW, off = kb % SW;
      wgmma_ss<BN, BF16, 0, 0>(s, desc_add(dq0, bx * Cfg::Q_BOX + off), desc_add(dk0, bx * Cfg::K_BOX + off), ks > 0);
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(s);
    widen_v(i);
    __syncthreads();  // V_i widened; K_i and byte stage i % NST read by everyone
    if (tid == 0 && i + NST < qs.T) load_bytes(i + NST);
    // P' = 2^-e_k silu(alpha kd S) * mask
    if (!rows_idle) {
      auto silu = [&](int n) {
        const float x = s[n] * c_s, xp = s[n] * c_sp;
        return __fmaf_rn(xp, tanh_approx(x), xp);  // silu(2x) = x (1 + tanh x)
      };
      mask_scores<BN>(qs.msk, fast, full_lim, qs.len, q_base, n0, t4, s, silu);
#pragma unroll
      for (int kk = 0; kk < BN / 16; ++kk) {
        const Operand<BF16> x0(s[8 * kk + 0], s[8 * kk + 1]), x1(s[8 * kk + 2], s[8 * kk + 3]);
        const Operand<BF16> x2(s[8 * kk + 4], s[8 * kk + 5]), x3(s[8 * kk + 6], s[8 * kk + 7]);
        a_hi[kk][0] = x0.hi; a_hi[kk][1] = x1.hi; a_hi[kk][2] = x2.hi; a_hi[kk][3] = x3.hi;
        a_lo[kk][0] = x0.lo; a_lo[kk][1] = x1.lo; a_lo[kk][2] = x2.lo; a_lo[kk][3] = x3.lo;
      }
    } else {
#pragma unroll
      for (int kk = 0; kk < BN / 16; ++kk)
#pragma unroll
        for (int r = 0; r < 4; ++r) a_hi[kk][r] = a_lo[kk][r] = 0u;
    }
    // O += P'_i V_i (kWidenUnderPV: under the widening of K_{i+1})
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < BN / 16; ++kk) {
      wgmma_rs<DV, BF16, 1>(o, a_hi[kk], desc_add(dv0, kk * 16 * SWV), 1);
      if constexpr (BF16) wgmma_rs<DV, BF16, 1>(o, a_lo[kk], desc_add(dv0, kk * 16 * SWV), 1);
    }
    wgmma_commit();
    if (kWidenUnderPV && i + 1 < qs.T) widen_k(i + 1);
    wgmma_wait<0>();
    fence_regs(o);
    fence_regs(a_hi);
    fence_regs(a_lo);
    if (!kWidenUnderPV && i + 1 < qs.T) widen_k(i + 1);
    __syncthreads();  // K_{i+1} widened; V_i read by everyone
  }

  // ---------------- epilogue: O' (1/N) vd 2^e_k -> out, or O' vd 2^e_k -> the fp32 partials ----------------
  int ev, ek2;  // (e_k again: reloaded rather than kept live through the loop)
  const float m_v = frexpf(load_descale(p.descale[1], p.ds_batch[1], p.ds_head[1], b, h), &ev);
  frexpf(load_descale(p.descale[0], p.ds_batch[0], p.ds_head[0], b, h), &ek2);
  const int e_o = ev + ek2;
  const float c_o = gridDim.z > 1 ? m_v : p.inv_n * m_v;
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int lr = wgi * 64 + w * 16 + g + hh * 8;
    if (lr >= qs.mrows) continue;
    if (gridDim.z > 1) {
      float* prow = p.part + ((part_row() + lr) * p.seq.heads + h) * DV;
#pragma unroll
      for (int nb = 0; nb < DV / 8; ++nb)
        *reinterpret_cast<float2*>(prow + nb * 8 + 2 * t4) =
            make_float2(scalbnf(o[nb * 4 + hh * 2] * c_o, e_o), scalbnf(o[nb * 4 + hh * 2 + 1] * c_o, e_o));
    } else {
      uint16_t* orow = reinterpret_cast<uint16_t*>(p.out) + (out_row() + lr) * p.o_row_stride + (long long)h * p.o_head_stride;
#pragma unroll
      for (int nb = 0; nb < DV / 8; ++nb) {
        const float x = scalbnf(o[nb * 4 + hh * 2] * c_o, e_o), y = scalbnf(o[nb * 4 + hh * 2 + 1] * c_o, e_o);
        *reinterpret_cast<uint32_t*>(orow + nb * 8 + 2 * t4) = BF16 ? pack_bf16x2(x, y) : pack_f16x2(x, y);
      }
    }
  }
}

// Two CTAs per SM (<= 128 registers per thread) where the 16-bit delta kernel has them, dv <= 64, except bf16 at dv = 64:
// there the P hi / lo fragments next to the O accumulator, the scores and the widening's state spill 4-12 bytes within 128
// registers, so it runs one CTA per SM without spills (ptxas -v, DESIGN.md 3.8)
template <int DV, bool BF16> constexpr int kFp8KvMinBlocks = (DV == 32 || (DV == 64 && !BF16)) ? 2 : 1;
template <int DQK, int DV, bool BF16>
__global__ void __launch_bounds__(kAttnThreads, kFp8KvMinBlocks<DV, BF16>)
    attn_fwd_delta_e4m3kv_wgmma_kernel(const __grid_constant__ DeltaFp8KvParams p) {
  attn_fwd_delta_fp8kv_body<DQK, DV, BF16>(p);
}

// ------------------------------------------------------------------------------------------------
// host
// ------------------------------------------------------------------------------------------------
int delta_fp8_kv_check(const hstu_attn_params& p) {
  if (p.dtype != HSTU_BF16 && p.dtype != HSTU_F16) {
    set_error("delta-q attention on an fp8 K / V cache: q and out must be bf16 or fp16 (got dtype %d)", p.dtype);
    return HSTU_ERR_UNSUPPORTED;
  }
  if (p.delta_q_len <= 0) {
    set_error("delta-q attention on an fp8 K / V cache: delta_q_len must be > 0 (got %d)", p.delta_q_len);
    return HSTU_ERR_UNSUPPORTED;
  }
  if (p.pos_w != nullptr || p.ts_w != nullptr) {
    set_error("delta-q attention on an fp8 K / V cache: the relative bias is not supported");
    return HSTU_ERR_UNSUPPORTED;
  }
  if (p.impl == HSTU_IMPL_GENERIC) {
    set_error("delta-q attention on an fp8 K / V cache runs on the wgmma kernels only: the generic kernels take no fp8 input");
    return HSTU_ERR_UNSUPPORTED;
  }
  if (!wgmma_dims(p.dqk, p.dv)) {
    set_error("delta-q attention on an fp8 K / V cache: dqk == dv or dqk < dv, both in {32, 64, 128, 256}, only (dqk=%d, dv=%d)",
              p.dqk, p.dv);
    return HSTU_ERR_UNSUPPORTED;
  }
  if (p.total_rows >= (1ll << 31) - 256 || (long long)p.batch * p.delta_q_len >= (1ll << 31) - 256) {
    set_error("delta-q attention on an fp8 K / V cache: at most 2^31 - 257 rows of k / v and of q");
    return HSTU_ERR_UNSUPPORTED;
  }
  if (!aligned_view(p.q, p.q_row_stride, p.q_head_stride) || !aligned_view(p.out, p.o_row_stride, p.o_head_stride)) {
    set_error("delta-q attention on an fp8 K / V cache: q and out need 16-byte aligned bases and row / head strides that are "
              "multiples of 8 elements");
    return HSTU_ERR_UNSUPPORTED;
  }
  if (!e4m3_view(p.k, p.k_row_stride, p.k_head_stride) || !e4m3_view(p.v, p.v_row_stride, p.v_head_stride)) {
    set_error("delta-q attention on an fp8 K / V cache: k and v need 16-byte aligned bases and row / head strides that are "
              "multiples of 16 elements");
    return HSTU_ERR_UNSUPPORTED;
  }
  return 0;
}

template <int DQK, int DV, bool BF16>
static int launch_delta_fp8kv(const hstu_attn_params& p, const hstu_attn_descales& ds, cudaStream_t st) {
  using Cfg = DeltaFp8KvCfg<DQK, DV>;
  DeltaFp8KvParams fp;
  memset(&fp, 0, sizeof(fp));
  const int chunks = delta_chunks(p);  // the rule of the 16-bit delta kernel: sizes only, whatever the K / V type
  if (chunks > 1) {
    const size_t need = wgmma_delta_workspace_bytes(p);
    if (p.workspace == nullptr || p.workspace_bytes < need) {
      set_error("hstu_attn_fwd_delta_fp8_kv: workspace of %zu bytes required (got %zu)", need, p.workspace_bytes);
      return HSTU_ERR_WORKSPACE;
    }
    fp.part = reinterpret_cast<float*>(p.workspace);
  }
  const long long q_rows = (long long)p.batch * p.delta_q_len;
  if (int e = make_tmap_rows_heads(&fp.tmQ, p.q, q_rows, p.heads, DQK, p.q_row_stride, p.q_head_stride, Cfg::BOX_COLS, Cfg::BM))
    return e;
  if (int e = make_tmap_rows_heads(&fp.tmK, p.k, p.total_rows, p.heads, DQK, p.k_row_stride, p.k_head_stride, Cfg::SWK8, Cfg::BN, 1))
    return e;
  if (int e = make_tmap_rows_heads(&fp.tmV, p.v, p.total_rows, p.heads, DV, p.v_row_stride, p.v_head_stride, Cfg::SWV8, Cfg::BN, 1))
    return e;
  fp.seq = seq_args(p);
  fp.out = p.out;
  fp.o_row_stride = p.o_row_stride;
  fp.o_head_stride = p.o_head_stride;
  fp.descale[0] = ds.k, fp.ds_batch[0] = ds.k_batch_stride, fp.ds_head[0] = ds.k_head_stride;
  fp.descale[1] = ds.v, fp.ds_batch[1] = ds.v_batch_stride, fp.ds_head[1] = ds.v_head_stride;
  fp.inv_n = 1.0f / (float)p.max_seq_len;
  fp.delta = p.delta_q_len;
  auto kern = attn_fwd_delta_e4m3kv_wgmma_kernel<DQK, DV, BF16>;
  HSTU_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
  const dim3 grid(p.batch * p.heads, (p.delta_q_len + Cfg::BM - 1) / Cfg::BM, chunks);
  kern<<<grid, kAttnThreads, Cfg::SMEM_BYTES, st>>>(fp);
  HSTU_CUDA_OK(cudaGetLastError());
  if (chunks > 1)
    return launch_delta_reduce(BF16, fp.part, p.out, q_rows, p.heads, DV, chunks, p.o_row_stride, p.o_head_stride, fp.inv_n, st);
  return 0;
}

int attn_wgmma_fwd_delta_fp8_kv(const hstu_attn_params& p, const hstu_attn_descales& ds, cudaStream_t st) {
  if (p.dqk != p.dv)
    return dispatch_dims(MixedDims{}, p, "delta-q attention on an fp8 K / V cache",
                         [&]<int DQK, int DV, bool BF16>() { return launch_delta_fp8kv<DQK, DV, BF16>(p, ds, st); });
  return dispatch_dims(SquareDims{}, p, "delta-q attention on an fp8 K / V cache",
                       [&]<int DQK, int DV, bool BF16>() { return launch_delta_fp8kv<DQK, DV, BF16>(p, ds, st); });
}

}  // namespace hstu
