// Timestamp + position embedding add in front of the STU stack (SURVEY.md section 8 row f2).
//
//   out[r, :] = cast(seq[r, :] * alpha) + cast(pos_w[pos_ind(r), :] + ts_w[ts_bucket(r), :])
//
// Reference: ops/position.py:43-96 (facade, `seq_embeddings * alpha` first), ops/pytorch/pt_position.py:39-134 (eager):
//   pos_ind: n = position of row r in its sequence b; high = len_b - num_targets_b * (interleave ? 2 : 1) (len_b without targets);
//            with targets  c = high - min(n, high),  else  c = len_b - n;   c += max_contextual_seq_len;
//            c = min(c, max_pos_ind - 1);   c = n  if n < max_contextual_seq_len                     (pt_position.py:39-72)
//   ts_bucket: dt = ts[last row of b] - ts[r]; x = max(dt, 1e-6) / 60; y = log(x) | sqrt(x); bucket = clamp((int)max(y, 0), 0, nb)
//            with nb = ts_w.size(1) - 1 exactly as the eager code has it (pt_position.py:98; the host passes it in)
//   the sum of the two table rows is formed in fp32, cast to the activation dtype, then added to the (already rounded) scaled
//   activation (pt_position.py:124-133): the same three roundings are reproduced here so that bf16 results match bit for bit.
// Backward: d_seq = dout * alpha; d_pos_w / d_ts_w are scatter-adds of dout (fp32 atomics).  Rows are walked in order by a
// CTA; consecutive rows of a sequence fall into the same time bucket for long runs, so the bucket gradient is accumulated in
// registers and flushed only when the bucket changes (the run-length trick the reference's Triton backward needs a sort for,
// ops/triton/triton_position.py:170-435).
//
// HBM-bound row-wise kernel: one warp per row, 128-bit accesses along the row when D allows.
#include "common.cuh"
#include "internal.h"

namespace hstu {

__device__ __forceinline__ int find_batch(const void* off, int is_i64, int B, long long row) {
  int lo = 0, hi = B;  // largest b with off[b] <= row
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (load_index(off, is_i64, mid) <= row) lo = mid;
    else hi = mid;
  }
  return lo;
}

template <typename T>
__global__ void __launch_bounds__(256) position_fwd_kernel(const PosArgs a) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * 8 + warp;
  if (row >= a.L) return;
  const int b = find_batch(a.seq_offsets, a.offsets_i64, a.B, row);
  const long long s = load_index(a.seq_offsets, a.offsets_i64, b), e = load_index(a.seq_offsets, a.offsets_i64, b + 1);
  const long long n = row - s;
  const long long len = load_index(a.seq_lengths, a.lengths_i64, b);
  long long c;
  if (a.num_targets) {
    const long long nt = load_index(a.num_targets, a.targets_i64, b);
    const long long high = len - nt * (a.interleave ? 2 : 1);
    c = high - (n < high ? n : high);
  } else {
    c = len - n;
  }
  c += a.max_contextual;
  c = c < a.max_pos_ind - 1 ? c : a.max_pos_ind - 1;
  if (n < a.max_contextual) c = n;
  // query time = timestamp of the last row of the sequence (index clamp(len - 1, 0) of the padded row, pt_position.py:108-110)
  long long qi = len - 1;
  qi = qi < 0 ? 0 : qi;
  const long long qt = (s + qi < e) ? a.timestamps[s + qi] : 0;  // padded positions hold 0
  const float dt = (float)(qt - a.timestamps[row]);               // int64 -> fp32, as torch's clamp(min=1e-6) promotes
  float x = fmaxf(dt, 1e-6f) / 60.0f;
  x = a.log_bucket ? logf(x) : sqrtf(x);
  x = fmaxf(x, 0.0f);
  int bucket = (int)x;
  bucket = bucket < 0 ? 0 : (bucket > a.num_time_buckets ? a.num_time_buckets : bucket);
  if (lane == 0) {
    if (a.pos_inds) a.pos_inds[row] = (int)c;
    if (a.ts_inds) a.ts_inds[row] = bucket;
  }
  const T* src = reinterpret_cast<const T*>(a.seq) + row * a.D;
  T* dst = reinterpret_cast<T*>(a.out) + row * a.D;
  const float* pw = a.pos_w + (long long)c * a.D;
  const float* tw = a.ts_w + (long long)bucket * a.D;
  if (sizeof(T) == 2 && (a.D & 7) == 0 && a.vec_ok) {
    // 8 elements per lane and step: one 128-bit load of the activation, two of each fp32 table row, one 128-bit store
    for (int col = lane * 8; col < a.D; col += 256) {
      const uint4 xv = *reinterpret_cast<const uint4*>(src + col);
      const float4 p0 = *reinterpret_cast<const float4*>(pw + col), p1 = *reinterpret_cast<const float4*>(pw + col + 4);
      const float4 t0 = *reinterpret_cast<const float4*>(tw + col), t1 = *reinterpret_cast<const float4*>(tw + col + 4);
      const float pe[8] = {t0.x + p0.x, t0.y + p0.y, t0.z + p0.z, t0.w + p0.w, t1.x + p1.x, t1.y + p1.y, t1.z + p1.z, t1.w + p1.w};
      const T* xe = reinterpret_cast<const T*>(&xv);
      uint4 ov;
      T* oe = reinterpret_cast<T*>(&ov);
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const T scaled = Cvt<T>::from_f(__fmul_rn(Cvt<T>::to_f(xe[k]), a.alpha));
        const T emb = Cvt<T>::from_f(pe[k]);
        oe[k] = Cvt<T>::from_f(__fadd_rn(Cvt<T>::to_f(scaled), Cvt<T>::to_f(emb)));
      }
      *reinterpret_cast<uint4*>(dst + col) = ov;
    }
    return;
  }
  for (int col = lane; col < a.D; col += 32) {
    // separate roundings, as the eager path has them: no contraction of the scale and the add into one FMA (fp32 would differ)
    const T scaled = Cvt<T>::from_f(__fmul_rn(Cvt<T>::to_f(src[col]), a.alpha));
    const T emb = Cvt<T>::from_f(__fadd_rn(tw[col], pw[col]));
    dst[col] = Cvt<T>::from_f(__fadd_rn(Cvt<T>::to_f(scaled), Cvt<T>::to_f(emb)));
  }
}

// One CTA walks ROWS consecutive rows; thread t owns columns t, t + blockDim.x, ... (NCOL of them, D <= NCOL * blockDim.x).
template <typename T, int NCOL>
__global__ void __launch_bounds__(256) position_bwd_kernel(const T* __restrict__ dout, T* __restrict__ dseq,
                                                            float* __restrict__ dpos, float* __restrict__ dts,
                                                            const int* __restrict__ pos_inds, const int* __restrict__ ts_inds,
                                                            long long L, int D, float alpha, int rows_per_cta) {
  const long long r0 = (long long)blockIdx.x * rows_per_cta;
  long long r1 = r0 + rows_per_cta;
  r1 = r1 < L ? r1 : L;
  float acc[NCOL];
#pragma unroll
  for (int k = 0; k < NCOL; ++k) acc[k] = 0.f;
  int cur = -1;
  for (long long r = r0; r < r1; ++r) {
    const int pi = pos_inds[r], ti = ts_inds[r];
    if (ti != cur) {
      if (cur >= 0) {
#pragma unroll
        for (int k = 0; k < NCOL; ++k) {
          const int col = threadIdx.x + k * blockDim.x;
          if (col < D) atomicAdd(dts + (long long)cur * D + col, acc[k]);
          acc[k] = 0.f;
        }
      }
      cur = ti;
    }
#pragma unroll
    for (int k = 0; k < NCOL; ++k) {
      const int col = threadIdx.x + k * blockDim.x;
      if (col < D) {
        const float g = Cvt<T>::to_f(dout[r * D + col]);
        dseq[r * D + col] = Cvt<T>::from_f(__fmul_rn(g, alpha));
        acc[k] += g;
        atomicAdd(dpos + (long long)pi * D + col, g);
      }
    }
  }
  if (cur >= 0) {
#pragma unroll
    for (int k = 0; k < NCOL; ++k) {
      const int col = threadIdx.x + k * blockDim.x;
      if (col < D) atomicAdd(dts + (long long)cur * D + col, acc[k]);
    }
  }
}

int position_fwd(const PosArgs& a, int dtype, cudaStream_t st) {
  if (a.L == 0) return 0;
  const unsigned blocks = (unsigned)((a.L + 7) / 8);
  switch (dtype) {
    case HSTU_F32: position_fwd_kernel<float><<<blocks, 256, 0, st>>>(a); break;
    case HSTU_BF16: position_fwd_kernel<__nv_bfloat16><<<blocks, 256, 0, st>>>(a); break;
    case HSTU_F16: position_fwd_kernel<__half><<<blocks, 256, 0, st>>>(a); break;
    default: set_error("position_fwd: bad dtype %d", dtype); return HSTU_ERR_INVALID_ARGUMENT;
  }
  HSTU_CUDA_OK(cudaGetLastError());
  return 0;
}

template <typename T>
static int position_bwd_t(const void* dout, void* dseq, float* dpos, float* dts, const int* pi, const int* ti, long long L, int D,
                          float alpha, cudaStream_t st) {
  // ~8 CTAs per SM in flight; at least 32 rows per CTA so that the time-bucket runs are worth keeping in registers
  long long rows = (L + 132 * 8 - 1) / (132 * 8);
  rows = rows < 32 ? 32 : rows;
  const unsigned blocks = (unsigned)((L + rows - 1) / rows);
  const T* d = reinterpret_cast<const T*>(dout);
  T* s = reinterpret_cast<T*>(dseq);
  if (D <= 256) position_bwd_kernel<T, 1><<<blocks, 256, 0, st>>>(d, s, dpos, dts, pi, ti, L, D, alpha, (int)rows);
  else if (D <= 512) position_bwd_kernel<T, 2><<<blocks, 256, 0, st>>>(d, s, dpos, dts, pi, ti, L, D, alpha, (int)rows);
  else if (D <= 1024) position_bwd_kernel<T, 4><<<blocks, 256, 0, st>>>(d, s, dpos, dts, pi, ti, L, D, alpha, (int)rows);
  else {
    set_error("position_bwd: embedding dim %d > 1024 is not supported", D);
    return HSTU_ERR_UNSUPPORTED;
  }
  HSTU_CUDA_OK(cudaGetLastError());
  return 0;
}

int position_bwd(const void* dout, void* dseq, float* dpos, float* dts, const int* pi, const int* ti, long long L, int D,
                 float alpha, int dtype, cudaStream_t st) {
  if (L == 0) return 0;
  switch (dtype) {
    case HSTU_F32: return position_bwd_t<float>(dout, dseq, dpos, dts, pi, ti, L, D, alpha, st);
    case HSTU_BF16: return position_bwd_t<__nv_bfloat16>(dout, dseq, dpos, dts, pi, ti, L, D, alpha, st);
    case HSTU_F16: return position_bwd_t<__half>(dout, dseq, dpos, dts, pi, ti, L, D, alpha, st);
  }
  set_error("position_bwd: bad dtype %d", dtype);
  return HSTU_ERR_INVALID_ARGUMENT;
}

}  // namespace hstu
