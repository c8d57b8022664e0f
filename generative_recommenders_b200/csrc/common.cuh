// Shared device/host helpers for libhstu_b200 (sm_90a).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/hstu_b200.h"

namespace hstu {

void set_error(const char* fmt, ...);

#define HSTU_CHECK_ARG(cond, ...)            \
  do {                                       \
    if (!(cond)) {                           \
      ::hstu::set_error(__VA_ARGS__);        \
      return HSTU_ERR_INVALID_ARGUMENT;      \
    }                                        \
  } while (0)

#define HSTU_CUDA_OK(expr)                                                              \
  do {                                                                                  \
    cudaError_t _e = (expr);                                                            \
    if (_e != cudaSuccess) {                                                            \
      ::hstu::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return HSTU_ERR_CUDA;                                                             \
    }                                                                                   \
  } while (0)

// ------------------------------------------------------------------------------------------------
// dtype helpers
// ------------------------------------------------------------------------------------------------
template <typename T>
struct Cvt;
template <>
struct Cvt<float> {
  static __device__ __forceinline__ float to_f(float x) { return x; }
  static __device__ __forceinline__ float from_f(float x) { return x; }
};
template <>
struct Cvt<__nv_bfloat16> {
  static __device__ __forceinline__ float to_f(__nv_bfloat16 x) { return __bfloat162float(x); }
  static __device__ __forceinline__ __nv_bfloat16 from_f(float x) { return __float2bfloat16_rn(x); }
};
template <>
struct Cvt<__half> {
  static __device__ __forceinline__ float to_f(__half x) { return __half2float(x); }
  static __device__ __forceinline__ __half from_f(float x) { return __float2half_rn(x); }
};

static inline int dtype_bytes(int dt) { return dt == HSTU_F32 ? 4 : 2; }

// ------------------------------------------------------------------------------------------------
// Attention mask -- restates ops/pytorch/pt_hstu_attention.py:33-84 for the real positions of ONE sequence.
// ------------------------------------------------------------------------------------------------
struct SeqMask {
  int len;        // sequence length (already clipped to max_seq_len)
  int max_id;     // max_ids of the reference after contextual / target adjustment
  int ctx;        // contextual_seq_len
  int win;        // max_attn_len (0 = none)
  int min_full;   // min_full_attn_seq_len
  int has_tgt;    // num_targets given
  int fast;       // 1: plain causal(+targets): valid = (j < min(i, max_id)) | (j == i)
};

__host__ __device__ inline SeqMask make_seq_mask(int len, int n_tgt /* <0: none */, int win, int min_full, int ctx) {
  SeqMask m;
  m.len = len;
  m.ctx = ctx;
  m.win = win;
  m.min_full = min_full;
  m.has_tgt = n_tgt >= 0;
  int max_id = len;
  if (ctx > 0) max_id = max_id - ctx + 1;
  if (n_tgt >= 0) max_id -= n_tgt;
  m.max_id = max_id;
  m.fast = (ctx == 0 && win == 0);
  return m;
}

__host__ __device__ inline int seq_id(const SeqMask& m, int p) {
  int id = p;
  if (m.ctx > 0) {
    id = p - m.ctx + 1;
    id = id < 0 ? 0 : id;
  }
  if (m.has_tgt) id = id < m.max_id ? id : m.max_id;
  return id;
}

__host__ __device__ inline bool mask_valid(const SeqMask& m, int i, int j) {
  if (m.fast) {
    // ids are positions clamped to max_id: (id_i - id_j > 0) <=> j < min(i, max_id) when targets are present,
    // j < i otherwise (max_id == len then).
    int lim = m.has_tgt ? (i < m.max_id ? i : m.max_id) : i;
    return (j < lim) | (j == i);
  }
  int idi = seq_id(m, i), idj = seq_id(m, j);
  int d = idi - idj;
  bool valid = (i == j) | (d > 0);
  if (m.win > 0) {
    if (m.min_full > 0)
      valid = valid & ((d <= m.win) | (idi >= m.max_id - m.min_full));
    else
      valid = valid & (d <= m.win);
  }
  if (m.ctx > 0) valid = valid | ((idi == 0) & (idj < m.max_id));
  return valid;
}

// Conservative key range [lo, hi) attended by query rows [m0, m1) (m1 <= len).
__host__ __device__ inline void kv_range_for_q_rows(const SeqMask& m, int m0, int m1, int* lo, int* hi) {
  int h = m1;                                  // causal: j <= i
  if (m.ctx > 0 && m0 < m.ctx) h = m.len;      // contextual rows (id 0) see every key with id < max_id
  if (h > m.len) h = m.len;
  int l = 0;
  if (m.win > 0) {
    int id0 = seq_id(m, m0);
    bool full_rows = false;
    if (m.min_full > 0) {
      int idlast = seq_id(m, m1 - 1);
      full_rows = idlast >= m.max_id - m.min_full;
    }
    if (!full_rows && id0 - m.win > 0) {
      int first_id = id0 - m.win;              // keys need id_j >= first_id (>= 1)
      l = first_id + (m.ctx > 0 ? m.ctx - 1 : 0);
      if (l > m0) l = m0;                      // the diagonal is always valid
    }
  }
  *lo = l;
  *hi = h;
}

// Conservative query range [lo, hi) attending keys [n0, n1) (n1 <= len), plus the contextual prefix rows [0, ctx_hi).
__host__ __device__ inline void q_range_for_kv_rows(const SeqMask& m, int n0, int n1, int* lo, int* hi, int* ctx_hi) {
  int l = n0;  // causal: i >= j
  int h = m.len;
  if (m.win > 0 && m.min_full == 0) {
    int idl = seq_id(m, n1 - 1);
    if (!(m.has_tgt && idl + m.win >= m.max_id)) {
      long long last = (long long)idl + m.win + (m.ctx > 0 ? m.ctx - 1 : 0) + 1;
      if (last < h) h = (int)last;
    }
    if (h < n1) h = n1 < m.len ? n1 : m.len;  // diagonal rows
  }
  int c = 0;
  if (m.ctx > 0) {
    c = m.ctx < l ? m.ctx : l;  // rows [0, c) are before `lo`; rows >= lo are covered by the main range
    if (c > m.len) c = m.len;
  }
  *lo = l;
  *hi = h;
  *ctx_hi = c;
}

// ------------------------------------------------------------------------------------------------
// Per-sequence geometry read from device arrays
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ long long load_index(const void* p, int is_i64, int idx) {
  return is_i64 ? (long long)reinterpret_cast<const long long*>(p)[idx] : (long long)reinterpret_cast<const int*>(p)[idx];
}

// Rows [r0, r1) of head `head_off` (element offset) of a [rows, heads, d] tensor := 0, by all threads of the CTA.  Used for the
// rows of a sequence at positions >= max_seq_len: the reference drops them on the way in (jagged_to_padded_dense truncates)
// and returns zeros for them (dense_to_jagged of the padded result), pt_hstu_attention.py:97-167.  Rare path: plain stores.
__device__ __forceinline__ void zero_rows(void* base, int elem_bytes, long long row_stride, long long head_off, int d,
                                          long long r0, long long r1) {
  const long long n = (r1 - r0) * d;
  for (long long idx = threadIdx.x; idx < n; idx += blockDim.x) {
    const long long r = r0 + idx / d, c = idx % d;
    const long long off = r * row_stride + head_off + c;
    if (elem_bytes == 2) reinterpret_cast<uint16_t*>(base)[off] = 0;
    else reinterpret_cast<uint32_t*>(base)[off] = 0u;
  }
}

// MUFU.EX2 + MUFU.RCP (2 ulp): the IEEE division `1.0f / x` compiles to ~15 instructions with a slow-path call, which made the
// SiLU kernels issue-bound (26 instructions per element)
__device__ __forceinline__ float sigmoid_f(float x) { return __fdividef(1.0f, 1.0f + __expf(-x)); }
__device__ __forceinline__ float silu_f(float x) { return x * sigmoid_f(x); }

// time-bucket of the research relative bias: clamp(floor(log(max(|d|,1))/0.301), 0, nb)  (hstu.py:604-612)
__device__ __forceinline__ int ts_bucket(long long d, int nb) {
  long long a = d < 0 ? -d : d;
  if (a < 1) a = 1;
  int bkt = (int)(logf((float)a) / 0.301f);
  bkt = bkt < 0 ? 0 : bkt;
  return bkt > nb ? nb : bkt;
}

}  // namespace hstu
