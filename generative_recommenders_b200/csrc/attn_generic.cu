// Generic jagged HSTU attention (forward + backward) on CUDA cores, fp32 accumulate.
//
// Role: the fully general path of libhstu_b200 -- any dtype (fp32/bf16/fp16), any head dims <= 256 with
// dqk != dv, every mask option of the reference (targets, max_attn_len, min_full_attn_seq_len, contextual prefix),
// the delta-q (cached) forward and the research-path relative bias.  The wgmma/TMA kernels (attn_wgmma_*.cu)
// take over for bf16/fp16 at the tensor-core-friendly head dims; this file is what they are validated against
// on-device at sizes the CPU oracle cannot reach, and what runs fp32 and odd head dims (25, 50, 8 ...).
//
// Math (SURVEY.md appendix A; reference ops/pytorch/pt_hstu_attention.py:130-171):
//   S = alpha Q K^T (+ bias), P = silu(S)/N * mask, O = P V
//   dV = P^T dO, dP = dO V^T, dS = dP * sig(S) * (1 + S (1 - sig(S))) / N * mask, dQ = alpha dS K, dK = alpha dS^T Q
//
// Layout: one CTA of 256 threads per (64- or 32-row tile, head, sequence); operand tiles staged in shared memory
// as fp32 (row pitch d+1 -> conflict-free column access); each thread owns an (R x R) micro-tile of the score
// tile and an (R x d/16) slice of the output tile.  Backward is split into a key-stationary kernel (dK, dV) and a
// query-stationary kernel (dQ, dpos_w, dts_w) so that no atomics are needed on dQ/dK/dV (deterministic).
// Every kernel exists for the causal mask and, with `bidir` in its name, for the non-causal one (common.cuh: ranges and
// mask_valid_bidir; kBidir of the bodies); the non-causal kernels take no delta-q call and no relative bias.
#include "common.cuh"

namespace hstu {

template <bool kBidir>
__device__ __forceinline__ bool pair_valid(const SeqMask& m, int i, int j) {
  return kBidir ? mask_valid_bidir(m, i, j) : mask_valid(m, i, j);
}
template <bool kBidir>
__device__ __forceinline__ void key_range(const SeqMask& m, int m0, int m1, int* lo, int* hi) {
  if (kBidir) kv_range_for_q_rows_bidir(m, m0, m1, lo, hi);
  else kv_range_for_q_rows(m, m0, m1, lo, hi);
}

struct GenericArgs {
  hstu_attn_params p;
};

template <typename T>
__device__ __forceinline__ void load_tile(float* dst, int pitch, const T* src, long long row_stride, int rows_valid,
                                          int tile_rows, int d, int tid) {
  // dst[r][c] = src[r * row_stride + c] for r < rows_valid else 0
  for (int idx = tid; idx < tile_rows * d; idx += 256) {
    int r = idx / d, c = idx - r * d;
    float v = 0.f;
    if (r < rows_valid) v = Cvt<T>::to_f(src[(long long)r * row_stride + c]);
    dst[r * pitch + c] = v;
  }
}

struct SeqGeom {
  long long kv_row0;  // first memory row of this sequence in k/v
  long long q_row0;   // first memory row of this sequence's query rows in q/out
  int len;            // number of key positions (clipped to max_seq_len)
  int len_true;       // unclipped length (rows [len, len_true) of a full-attention call are zero-filled)
  int q_pos0;         // sequence position of the first query row
  int nq;             // number of query rows
  int n_tgt;          // -1 if none
};

__device__ __forceinline__ SeqGeom seq_geom(const hstu_attn_params& p, int b) {
  SeqGeom g;
  long long s = load_index(p.seq_offsets, p.offsets_are_i64, b);
  long long e = load_index(p.seq_offsets, p.offsets_are_i64, b + 1);
  int len = (int)(e - s);
  g.kv_row0 = s;
  g.len_true = len;
  g.n_tgt = p.num_targets ? (int)load_index(p.num_targets, p.num_targets_are_i64, b) : -1;
  if (p.delta_q_len > 0) {
    // pytorch_cached_hstu_mha (pt_hstu_attention.py:175-235): queries are the last delta rows; keys are not clipped
    g.len = len;
    g.nq = p.delta_q_len;
    g.q_pos0 = len - p.delta_q_len;
    g.q_row0 = (long long)b * p.delta_q_len;
  } else {
    g.len = len < p.max_seq_len ? len : p.max_seq_len;  // jagged_to_padded_dense truncates at N
    g.nq = g.len;
    g.q_pos0 = 0;
    g.q_row0 = s;
  }
  return g;
}

__device__ __forceinline__ float warp_sum_f(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ float bias_at(const hstu_attn_params& p, int b, int i, int j) {
  // research/modeling/sequential/hstu.py:124-143
  float bias = 0.f;
  int n = p.max_seq_len;
  if (p.pos_w) bias += p.pos_w[n - 1 + j - i];
  if (p.ts_w) {
    const long long* ts = reinterpret_cast<const long long*>(p.timestamps) + (long long)b * n;
    int i1 = i + 1 < n ? i + 1 : n - 1;
    bias += p.ts_w[ts_bucket(ts[i1] - ts[j], p.num_ts_buckets)];
  }
  return bias;
}

// ------------------------------------------------------------------------------------------------
// forward
// ------------------------------------------------------------------------------------------------
template <typename T, int TILE, int DMAX, bool kBidir>
__device__ __forceinline__ void attn_fwd_generic_body(const GenericArgs args) {
  const hstu_attn_params& p = args.p;
  constexpr int R = TILE / 16;
  constexpr int NC = DMAX / 16;
  const int b = blockIdx.z, h = blockIdx.y;
  const SeqGeom g = seq_geom(p, b);
  const int mt = gridDim.x - 1 - blockIdx.x;  // heavy (late) tiles first
  const int m0 = mt * TILE;
  if (blockIdx.x == 0 && p.delta_q_len == 0 && g.len_true > g.len)
    zero_rows(p.out, sizeof(T), p.o_row_stride, (long long)h * p.o_head_stride, p.dv, g.kv_row0 + g.len, g.kv_row0 + g.len_true);
  if (m0 >= g.nq) return;
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  const int dqk = p.dqk, dv = p.dv;
  const int pq = dqk + 1, pv = dv + 1, pp = TILE + 1;
  extern __shared__ float smem[];
  float* sQ = smem;
  float* sK = sQ + TILE * pq;
  float* sV = sK + TILE * pq;
  float* sP = sV + TILE * pv;

  const SeqMask msk = make_seq_mask(g.len, g.n_tgt, p.max_attn_len, p.min_full_attn_seq_len, p.contextual_seq_len);
  const T* qp = reinterpret_cast<const T*>(p.q) + (g.q_row0 + m0) * p.q_row_stride + (long long)h * p.q_head_stride;
  const int mrows = min(TILE, g.nq - m0);
  load_tile<T>(sQ, pq, qp, p.q_row_stride, mrows, TILE, dqk, tid);

  float acc[R][NC];
#pragma unroll
  for (int r = 0; r < R; ++r)
#pragma unroll
    for (int c = 0; c < NC; ++c) acc[r][c] = 0.f;

  int lo, hi;
  key_range<kBidir>(msk, g.q_pos0 + m0, g.q_pos0 + m0 + mrows, &lo, &hi);
  const bool has_bias = p.pos_w != nullptr || p.ts_w != nullptr;
  for (int n0 = (lo / TILE) * TILE; n0 < hi; n0 += TILE) {
    const int nrows = min(TILE, g.len - n0);
    __syncthreads();  // previous iteration done with sK/sV/sP (and sQ visible on the first)
    load_tile<T>(sK, pq, reinterpret_cast<const T*>(p.k) + (g.kv_row0 + n0) * p.k_row_stride + (long long)h * p.k_head_stride,
                 p.k_row_stride, nrows, TILE, dqk, tid);
    load_tile<T>(sV, pv, reinterpret_cast<const T*>(p.v) + (g.kv_row0 + n0) * p.v_row_stride + (long long)h * p.v_head_stride,
                 p.v_row_stride, nrows, TILE, dv, tid);
    __syncthreads();
    float s[R][R];
#pragma unroll
    for (int r = 0; r < R; ++r)
#pragma unroll
      for (int c = 0; c < R; ++c) s[r][c] = 0.f;
    for (int d = 0; d < dqk; ++d) {
      float qv[R], kv[R];
#pragma unroll
      for (int r = 0; r < R; ++r) qv[r] = sQ[(ty * R + r) * pq + d];
#pragma unroll
      for (int c = 0; c < R; ++c) kv[c] = sK[(tx + 16 * c) * pq + d];
#pragma unroll
      for (int r = 0; r < R; ++r)
#pragma unroll
        for (int c = 0; c < R; ++c) s[r][c] = fmaf(qv[r], kv[c], s[r][c]);
    }
#pragma unroll
    for (int r = 0; r < R; ++r)
#pragma unroll
      for (int c = 0; c < R; ++c) {
        const int il = ty * R + r, jl = tx + 16 * c;
        const int i = g.q_pos0 + m0 + il, j = n0 + jl;
        float pval = 0.f;
        if (il < mrows && jl < nrows && pair_valid<kBidir>(msk, i, j)) {
          float x = s[r][c] * p.alpha;
          if (has_bias) x += bias_at(p, b, i, j);
          pval = silu_f(x);
        }
        sP[il * pp + jl] = pval;
      }
    __syncthreads();
    for (int j = 0; j < nrows; ++j) {
      float pr[R];
#pragma unroll
      for (int r = 0; r < R; ++r) pr[r] = sP[(ty * R + r) * pp + j];
#pragma unroll
      for (int c = 0; c < NC; ++c) {
        const int col = tx + 16 * c;
        if (col < dv) {
          const float vv = sV[j * pv + col];
#pragma unroll
          for (int r = 0; r < R; ++r) acc[r][c] = fmaf(pr[r], vv, acc[r][c]);
        }
      }
    }
  }
  const float inv_n = 1.0f / (float)p.max_seq_len;
  T* op = reinterpret_cast<T*>(p.out) + (g.q_row0 + m0) * p.o_row_stride + (long long)h * p.o_head_stride;
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const int il = ty * R + r;
    if (il < mrows) {
#pragma unroll
      for (int c = 0; c < NC; ++c) {
        const int col = tx + 16 * c;
        if (col < dv) op[(long long)il * p.o_row_stride + col] = Cvt<T>::from_f(acc[r][c] * inv_n);
      }
    }
  }
}

template <typename T, int TILE, int DMAX>
__global__ void __launch_bounds__(256) attn_fwd_generic_kernel(const GenericArgs args) {
  attn_fwd_generic_body<T, TILE, DMAX, false>(args);
}
template <typename T, int TILE, int DMAX>
__global__ void __launch_bounds__(256) attn_fwd_bidir_generic_kernel(const GenericArgs args) {
  attn_fwd_generic_body<T, TILE, DMAX, true>(args);
}

// ------------------------------------------------------------------------------------------------
// backward, key-stationary: dK, dV
// ------------------------------------------------------------------------------------------------
template <typename T, int TILE, int DMAX, bool kBidir>
__device__ __forceinline__ void attn_bwd_kv_generic_body(const GenericArgs args) {
  const hstu_attn_params& p = args.p;
  constexpr int R = TILE / 16;
  constexpr int NC = DMAX / 16;
  const int b = blockIdx.z, h = blockIdx.y;
  const SeqGeom g = seq_geom(p, b);
  const int n0 = blockIdx.x * TILE;  // early key tiles are the heavy ones and come first
  if (blockIdx.x == 0 && g.len_true > g.len) {
    zero_rows(p.dk, sizeof(T), p.dk_row_stride, (long long)h * p.dk_head_stride, p.dqk, g.kv_row0 + g.len, g.kv_row0 + g.len_true);
    zero_rows(p.dv_out, sizeof(T), p.dv_row_stride, (long long)h * p.dv_head_stride, p.dv, g.kv_row0 + g.len, g.kv_row0 + g.len_true);
  }
  if (n0 >= g.len) return;
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  const int dqk = p.dqk, dv = p.dv;
  const int pq = dqk + 1, pv = dv + 1, pp = TILE + 1;
  extern __shared__ float smem[];
  float* sK = smem;                 // [TILE][pq]
  float* sV = sK + TILE * pq;       // [TILE][pv]
  float* sQ = sV + TILE * pv;       // [TILE][pq]
  float* sDO = sQ + TILE * pq;      // [TILE][pv]
  float* sP = sDO + TILE * pv;      // [TILE(q)][pp]  P   (row = query, col = key)
  float* sDS = sP + TILE * pp;      // [TILE(q)][pp]  dS

  const SeqMask msk = make_seq_mask(g.len, g.n_tgt, p.max_attn_len, p.min_full_attn_seq_len, p.contextual_seq_len);
  const int nrows = min(TILE, g.len - n0);
  load_tile<T>(sK, pq, reinterpret_cast<const T*>(p.k) + (g.kv_row0 + n0) * p.k_row_stride + (long long)h * p.k_head_stride,
               p.k_row_stride, nrows, TILE, dqk, tid);
  load_tile<T>(sV, pv, reinterpret_cast<const T*>(p.v) + (g.kv_row0 + n0) * p.v_row_stride + (long long)h * p.v_head_stride,
               p.v_row_stride, nrows, TILE, dv, tid);

  float adk[R][NC], adv[R][NC];  // this thread: key rows ty*R+r, feature cols tx+16c
#pragma unroll
  for (int r = 0; r < R; ++r)
#pragma unroll
    for (int c = 0; c < NC; ++c) adk[r][c] = adv[r][c] = 0.f;

  int lo, hi, ctx_hi;
  if (kBidir) q_range_for_kv_rows_bidir(msk, n0, n0 + nrows, &lo, &hi, &ctx_hi);
  else q_range_for_kv_rows(msk, n0, n0 + nrows, &lo, &hi, &ctx_hi);
  const bool has_bias = p.pos_w != nullptr || p.ts_w != nullptr;
  const float inv_n = 1.0f / (float)p.max_seq_len;
  // query tiles: the contextual prefix rows [0, ctx_hi) that lie before the main range, then the main range [lo, hi)
  const int main_start = (lo / TILE) * TILE;
  for (int pass = 0; pass < 2; ++pass) {
    const int q_lo = pass == 0 ? 0 : main_start;
    const int q_hi = pass == 0 ? min(ctx_hi, main_start) : hi;
    for (int m0 = q_lo; m0 < q_hi; m0 += TILE) {
      const int mrows = min(TILE, g.len - m0);
      __syncthreads();
      load_tile<T>(sQ, pq, reinterpret_cast<const T*>(p.q) + (g.q_row0 + m0) * p.q_row_stride + (long long)h * p.q_head_stride,
                   p.q_row_stride, mrows, TILE, dqk, tid);
      load_tile<T>(sDO, pv, reinterpret_cast<const T*>(p.dout) + (g.q_row0 + m0) * p.do_row_stride + (long long)h * p.do_head_stride,
                   p.do_row_stride, mrows, TILE, dv, tid);
      __syncthreads();
      // S[q][k] and dP[q][k] micro tiles: query rows ty*R+r, key cols tx+16c
      float s[R][R], dp[R][R];
#pragma unroll
      for (int r = 0; r < R; ++r)
#pragma unroll
        for (int c = 0; c < R; ++c) s[r][c] = dp[r][c] = 0.f;
      for (int d = 0; d < dqk; ++d) {
        float qv[R], kv[R];
#pragma unroll
        for (int r = 0; r < R; ++r) qv[r] = sQ[(ty * R + r) * pq + d];
#pragma unroll
        for (int c = 0; c < R; ++c) kv[c] = sK[(tx + 16 * c) * pq + d];
#pragma unroll
        for (int r = 0; r < R; ++r)
#pragma unroll
          for (int c = 0; c < R; ++c) s[r][c] = fmaf(qv[r], kv[c], s[r][c]);
      }
      for (int d = 0; d < dv; ++d) {
        float ov[R], vv[R];
#pragma unroll
        for (int r = 0; r < R; ++r) ov[r] = sDO[(ty * R + r) * pv + d];
#pragma unroll
        for (int c = 0; c < R; ++c) vv[c] = sV[(tx + 16 * c) * pv + d];
#pragma unroll
        for (int r = 0; r < R; ++r)
#pragma unroll
          for (int c = 0; c < R; ++c) dp[r][c] = fmaf(ov[r], vv[c], dp[r][c]);
      }
#pragma unroll
      for (int r = 0; r < R; ++r)
#pragma unroll
        for (int c = 0; c < R; ++c) {
          const int il = ty * R + r, jl = tx + 16 * c;
          const int i = m0 + il, j = n0 + jl;
          float pval = 0.f, ds = 0.f;
          if (il < mrows && jl < nrows && pair_valid<kBidir>(msk, i, j)) {
            float x = s[r][c] * p.alpha;
            if (has_bias) x += bias_at(p, b, i, j);
            const float sg = sigmoid_f(x);
            pval = x * sg * inv_n;
            ds = dp[r][c] * sg * (1.f + x * (1.f - sg)) * inv_n;
          }
          sP[il * pp + jl] = pval;
          sDS[il * pp + jl] = ds;
        }
      __syncthreads();
      // dV[k][c] += sum_q P[q][k] dO[q][c];  dK[k][c] += sum_q dS[q][k] Q[q][c]
      for (int qi = 0; qi < mrows; ++qi) {
        float pr[R], dsr[R];
#pragma unroll
        for (int r = 0; r < R; ++r) {
          pr[r] = sP[qi * pp + ty * R + r];
          dsr[r] = sDS[qi * pp + ty * R + r];
        }
#pragma unroll
        for (int c = 0; c < NC; ++c) {
          const int col = tx + 16 * c;
          if (col < dv) {
            const float o = sDO[qi * pv + col];
#pragma unroll
            for (int r = 0; r < R; ++r) adv[r][c] = fmaf(pr[r], o, adv[r][c]);
          }
          if (col < dqk) {
            const float qq = sQ[qi * pq + col];
#pragma unroll
            for (int r = 0; r < R; ++r) adk[r][c] = fmaf(dsr[r], qq, adk[r][c]);
          }
        }
      }
    }
  }
  T* dkp = reinterpret_cast<T*>(p.dk) + (g.kv_row0 + n0) * p.dk_row_stride + (long long)h * p.dk_head_stride;
  T* dvp = reinterpret_cast<T*>(p.dv_out) + (g.kv_row0 + n0) * p.dv_row_stride + (long long)h * p.dv_head_stride;
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const int jl = ty * R + r;
    if (jl < nrows) {
#pragma unroll
      for (int c = 0; c < NC; ++c) {
        const int col = tx + 16 * c;
        if (col < dv) dvp[(long long)jl * p.dv_row_stride + col] = Cvt<T>::from_f(adv[r][c]);
        if (col < dqk) dkp[(long long)jl * p.dk_row_stride + col] = Cvt<T>::from_f(adk[r][c] * p.alpha);
      }
    }
  }
}

template <typename T, int TILE, int DMAX>
__global__ void __launch_bounds__(256) attn_bwd_kv_generic_kernel(const GenericArgs args) {
  attn_bwd_kv_generic_body<T, TILE, DMAX, false>(args);
}
template <typename T, int TILE, int DMAX>
__global__ void __launch_bounds__(256) attn_bwd_kv_bidir_generic_kernel(const GenericArgs args) {
  attn_bwd_kv_generic_body<T, TILE, DMAX, true>(args);
}

// ------------------------------------------------------------------------------------------------
// backward, query-stationary: dQ (+ dpos_w, dts_w of the research bias)
// ------------------------------------------------------------------------------------------------
template <typename T, int TILE, int DMAX, bool kBidir>
__device__ __forceinline__ void attn_bwd_q_generic_body(const GenericArgs args) {
  const hstu_attn_params& p = args.p;
  constexpr int R = TILE / 16;
  constexpr int NC = DMAX / 16;
  const int b = blockIdx.z, h = blockIdx.y;
  const SeqGeom g = seq_geom(p, b);
  const int mt = gridDim.x - 1 - blockIdx.x;
  const int m0 = mt * TILE;
  if (blockIdx.x == 0 && g.len_true > g.len)
    zero_rows(p.dq, sizeof(T), p.dq_row_stride, (long long)h * p.dq_head_stride, p.dqk, g.kv_row0 + g.len, g.kv_row0 + g.len_true);
  if (m0 >= g.len) return;
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  const int dqk = p.dqk, dv = p.dv;
  const int pq = dqk + 1, pv = dv + 1, pp = TILE + 1;
  extern __shared__ float smem[];
  float* sQ = smem;
  float* sDO = sQ + TILE * pq;
  float* sK = sDO + TILE * pv;
  float* sV = sK + TILE * pq;
  float* sDS = sV + TILE * pv;
  float* hpos = sDS + TILE * pp;   // [2 TILE - 1] position-bias gradient of the current tile pair
  float* hts = hpos + 2 * TILE;    // [num_ts_buckets + 1] time-bias gradient of this CTA
  if (p.dpos_w || p.dts_w) {
    for (int t = tid; t < 2 * TILE + (p.dts_w ? p.num_ts_buckets + 1 : 0); t += 256) hpos[t] = 0.f;
  }

  const SeqMask msk = make_seq_mask(g.len, g.n_tgt, p.max_attn_len, p.min_full_attn_seq_len, p.contextual_seq_len);
  const int mrows = min(TILE, g.len - m0);
  load_tile<T>(sQ, pq, reinterpret_cast<const T*>(p.q) + (g.q_row0 + m0) * p.q_row_stride + (long long)h * p.q_head_stride,
               p.q_row_stride, mrows, TILE, dqk, tid);
  load_tile<T>(sDO, pv, reinterpret_cast<const T*>(p.dout) + (g.q_row0 + m0) * p.do_row_stride + (long long)h * p.do_head_stride,
               p.do_row_stride, mrows, TILE, dv, tid);
  float adq[R][NC];
#pragma unroll
  for (int r = 0; r < R; ++r)
#pragma unroll
    for (int c = 0; c < NC; ++c) adq[r][c] = 0.f;
  int lo, hi;
  key_range<kBidir>(msk, m0, m0 + mrows, &lo, &hi);
  const bool has_bias = p.pos_w != nullptr || p.ts_w != nullptr;
  const float inv_n = 1.0f / (float)p.max_seq_len;
  for (int n0 = (lo / TILE) * TILE; n0 < hi; n0 += TILE) {
    const int nrows = min(TILE, g.len - n0);
    __syncthreads();
    load_tile<T>(sK, pq, reinterpret_cast<const T*>(p.k) + (g.kv_row0 + n0) * p.k_row_stride + (long long)h * p.k_head_stride,
                 p.k_row_stride, nrows, TILE, dqk, tid);
    load_tile<T>(sV, pv, reinterpret_cast<const T*>(p.v) + (g.kv_row0 + n0) * p.v_row_stride + (long long)h * p.v_head_stride,
                 p.v_row_stride, nrows, TILE, dv, tid);
    __syncthreads();
    float s[R][R], dp[R][R];
#pragma unroll
    for (int r = 0; r < R; ++r)
#pragma unroll
      for (int c = 0; c < R; ++c) s[r][c] = dp[r][c] = 0.f;
    for (int d = 0; d < dqk; ++d) {
      float qv[R], kv[R];
#pragma unroll
      for (int r = 0; r < R; ++r) qv[r] = sQ[(ty * R + r) * pq + d];
#pragma unroll
      for (int c = 0; c < R; ++c) kv[c] = sK[(tx + 16 * c) * pq + d];
#pragma unroll
      for (int r = 0; r < R; ++r)
#pragma unroll
        for (int c = 0; c < R; ++c) s[r][c] = fmaf(qv[r], kv[c], s[r][c]);
    }
    for (int d = 0; d < dv; ++d) {
      float ov[R], vv[R];
#pragma unroll
      for (int r = 0; r < R; ++r) ov[r] = sDO[(ty * R + r) * pv + d];
#pragma unroll
      for (int c = 0; c < R; ++c) vv[c] = sV[(tx + 16 * c) * pv + d];
#pragma unroll
      for (int r = 0; r < R; ++r)
#pragma unroll
        for (int c = 0; c < R; ++c) dp[r][c] = fmaf(ov[r], vv[c], dp[r][c]);
    }
#pragma unroll
    for (int r = 0; r < R; ++r)
#pragma unroll
      for (int c = 0; c < R; ++c) {
        const int il = ty * R + r, jl = tx + 16 * c;
        const int i = m0 + il, j = n0 + jl;
        float ds = 0.f;
        int bk = -1;
        if (il < mrows && jl < nrows && pair_valid<kBidir>(msk, i, j)) {
          float x = s[r][c] * p.alpha;
          if (has_bias) {
            const int n = p.max_seq_len;
            if (p.pos_w) x += p.pos_w[n - 1 + j - i];
            if (p.ts_w) {
              const long long* ts = reinterpret_cast<const long long*>(p.timestamps) + (long long)b * n;
              const int i1 = i + 1 < n ? i + 1 : n - 1;
              bk = ts_bucket(ts[i1] - ts[j], p.num_ts_buckets);
              x += p.ts_w[bk];
            }
          }
          const float sg = sigmoid_f(x);
          ds = dp[r][c] * sg * (1.f + x * (1.f - sg)) * inv_n;
        }
        if (has_bias) {  // CTA-uniform
          // The bias parameters are shared by every (sequence, head, i, j): one global atomic per score serialises on a few
          // hundred addresses (10.8 ms per call at the ML-20M shape).  Gradients are first accumulated in shared memory --
          // position bias: the 2 TILE - 1 diagonals of this tile pair (<= 2 lanes of a warp share one); time bias: lanes of
          // a warp mostly hit ONE bucket, so the warp sums first -- and flushed with one global atomic per bin.
          if (p.dpos_w && ds != 0.f) atomicAdd(hpos + (jl - il + TILE - 1), ds);
          if (p.dts_w) {
            int same;
            __match_all_sync(0xffffffffu, bk, &same);
            if (same) {
              const float t = warp_sum_f(ds);
              if ((tid & 31) == 0 && bk >= 0 && t != 0.f) atomicAdd(hts + bk, t);
            } else if (bk >= 0 && ds != 0.f) {
              atomicAdd(hts + bk, ds);
            }
          }
        }
        sDS[il * pp + jl] = ds;
      }
    __syncthreads();
    if (has_bias && p.dpos_w && tid < 2 * TILE - 1) {
      const float v = hpos[tid];
      hpos[tid] = 0.f;  // the next tile pair accumulates after two more barriers
      if (v != 0.f) atomicAdd(p.dpos_w + (p.max_seq_len - 1 + (n0 - m0) + tid - (TILE - 1)), v);
    }
    for (int j = 0; j < nrows; ++j) {
      float dsr[R];
#pragma unroll
      for (int r = 0; r < R; ++r) dsr[r] = sDS[(ty * R + r) * pp + j];
#pragma unroll
      for (int c = 0; c < NC; ++c) {
        const int col = tx + 16 * c;
        if (col < dqk) {
          const float kk = sK[j * pq + col];
#pragma unroll
          for (int r = 0; r < R; ++r) adq[r][c] = fmaf(dsr[r], kk, adq[r][c]);
        }
      }
    }
  }
  if (p.dts_w) {
    __syncthreads();
    for (int t = tid; t <= p.num_ts_buckets; t += 256) {
      const float v = hts[t];
      if (v != 0.f) atomicAdd(p.dts_w + t, v);
    }
  }
  T* dqp = reinterpret_cast<T*>(p.dq) + (g.q_row0 + m0) * p.dq_row_stride + (long long)h * p.dq_head_stride;
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const int il = ty * R + r;
    if (il < mrows) {
#pragma unroll
      for (int c = 0; c < NC; ++c) {
        const int col = tx + 16 * c;
        if (col < dqk) dqp[(long long)il * p.dq_row_stride + col] = Cvt<T>::from_f(adq[r][c] * p.alpha);
      }
    }
  }
}

template <typename T, int TILE, int DMAX>
__global__ void __launch_bounds__(256) attn_bwd_q_generic_kernel(const GenericArgs args) {
  attn_bwd_q_generic_body<T, TILE, DMAX, false>(args);
}
template <typename T, int TILE, int DMAX>
__global__ void __launch_bounds__(256) attn_bwd_q_bidir_generic_kernel(const GenericArgs args) {
  attn_bwd_q_generic_body<T, TILE, DMAX, true>(args);
}

// ------------------------------------------------------------------------------------------------
// host launchers
// ------------------------------------------------------------------------------------------------
template <typename K>
static int set_smem(K kernel, size_t bytes) {
  HSTU_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
  return 0;
}

template <typename T, int TILE, int DMAX>
static int launch_fwd(const hstu_attn_params& p, cudaStream_t st, bool bidir) {
  const int nq_max = p.delta_q_len > 0 ? p.delta_q_len : p.max_seq_len;
  dim3 grid((nq_max + TILE - 1) / TILE, p.heads, p.batch);
  size_t smem = sizeof(float) * (size_t)(2 * TILE * (p.dqk + 1) + TILE * (p.dv + 1) + TILE * (TILE + 1));
  auto kern = bidir ? attn_fwd_bidir_generic_kernel<T, TILE, DMAX> : attn_fwd_generic_kernel<T, TILE, DMAX>;
  if (int e = set_smem(kern, smem)) return e;
  GenericArgs a{p};
  kern<<<grid, 256, smem, st>>>(a);
  HSTU_CUDA_OK(cudaGetLastError());
  return 0;
}

template <typename T, int TILE, int DMAX>
static int launch_bwd(const hstu_attn_params& p, cudaStream_t st, bool bidir) {
  dim3 grid((p.max_seq_len + TILE - 1) / TILE, p.heads, p.batch);
  GenericArgs a{p};
  {
    size_t smem = sizeof(float) * (size_t)(2 * TILE * (p.dqk + 1) + 2 * TILE * (p.dv + 1) + 2 * TILE * (TILE + 1));
    auto kern = bidir ? attn_bwd_kv_bidir_generic_kernel<T, TILE, DMAX> : attn_bwd_kv_generic_kernel<T, TILE, DMAX>;
    if (int e = set_smem(kern, smem)) return e;
    kern<<<grid, 256, smem, st>>>(a);
    HSTU_CUDA_OK(cudaGetLastError());
  }
  {
    size_t smem = sizeof(float) * (size_t)(2 * TILE * (p.dqk + 1) + 2 * TILE * (p.dv + 1) + TILE * (TILE + 1) + 2 * TILE +
                                           (p.dts_w ? p.num_ts_buckets + 1 : 0));
    auto kern = bidir ? attn_bwd_q_bidir_generic_kernel<T, TILE, DMAX> : attn_bwd_q_generic_kernel<T, TILE, DMAX>;
    if (int e = set_smem(kern, smem)) return e;
    kern<<<grid, 256, smem, st>>>(a);
    HSTU_CUDA_OK(cudaGetLastError());
  }
  return 0;
}

template <typename T>
static int dispatch_fwd(const hstu_attn_params& p, cudaStream_t st, bool bidir) {
  const int dm = p.dqk > p.dv ? p.dqk : p.dv;
  if (dm <= 64) return launch_fwd<T, 64, 64>(p, st, bidir);
  if (dm <= 128) return launch_fwd<T, 64, 128>(p, st, bidir);
  return launch_fwd<T, 64, 256>(p, st, bidir);
}
template <typename T>
static int dispatch_bwd(const hstu_attn_params& p, cudaStream_t st, bool bidir) {
  const int dm = p.dqk > p.dv ? p.dqk : p.dv;
  if (dm <= 64) return launch_bwd<T, 64, 64>(p, st, bidir);
  if (dm <= 128) return launch_bwd<T, 64, 128>(p, st, bidir);
  return launch_bwd<T, 32, 256>(p, st, bidir);
}

int attn_generic_fwd(const hstu_attn_params& p, cudaStream_t st, bool bidir) {
  switch (p.dtype) {
    case HSTU_F32: return dispatch_fwd<float>(p, st, bidir);
    case HSTU_BF16: return dispatch_fwd<__nv_bfloat16>(p, st, bidir);
    case HSTU_F16: return dispatch_fwd<__half>(p, st, bidir);
  }
  set_error("unsupported dtype %d", p.dtype);
  return HSTU_ERR_UNSUPPORTED;
}

int attn_generic_bwd(const hstu_attn_params& p, cudaStream_t st, bool bidir) {
  switch (p.dtype) {
    case HSTU_F32: return dispatch_bwd<float>(p, st, bidir);
    case HSTU_BF16: return dispatch_bwd<__nv_bfloat16>(p, st, bidir);
    case HSTU_F16: return dispatch_bwd<__half>(p, st, bidir);
  }
  set_error("unsupported dtype %d", p.dtype);
  return HSTU_ERR_UNSUPPORTED;
}

}  // namespace hstu
