// jagged x dense batched matmul with a broadcast bias (SURVEY.md section 8 rows a9 / f4):
//     out[r, :] = jagged[r, :] @ dense[b] + bias[b]        for the rows r of sequence b
// Reference: ops/jagged_tensors.py:210-253 (facade), ops/pytorch/pt_jagged.py:77-98 (eager: operands promoted to fp32, result
// cast back to the dtype of `jagged`), ops/triton/triton_jagged.py:56-347 (kernels + backward).
// Here: fp32-accumulate tiles on the CUDA cores (64 x 64 outputs per CTA, 4 x 4 per thread, K in steps of 16): the only caller
// (modules/contextualize_mlps.py:136) runs it once per batch outside the STU stack with K, N = a few hundred.
// Rows at positions >= max_seq_len of a sequence are written as exact zeros (the eager path truncates the padded operand at
// max_seq_len and dense_to_jagged pads those rows with 0); so they pass no gradient to jagged either (the d_jagged pass is the
// same kernel), and the wgrad kernel reads no row past max_seq_len.  The grid has ceil(max_seq_len / 64) row tiles per
// sequence, as the reference's; a CTA strides over its sequence's tiles by that count, so every row of a longer sequence is
// written without the host learning the longest length.
//   forward / d_jagged:  C[r, n] = sum_k A[r, k] * B[b][k, n]   (TRANS_B: B[b][n, k])   (+ bias[b, n])
//   d_dense / d_bias:    dW[b][k, n] = sum_{r in b} A[r, k] * G[r, n];   dbias[b, n] = sum_{r in b} G[r, n]
#include "common.cuh"
#include "internal.h"

namespace hstu {

template <typename T, bool TRANS_B>
__global__ void __launch_bounds__(256) jagged_bmm_kernel(const T* __restrict__ A, const T* __restrict__ Bm,
                                                          const T* __restrict__ bias, T* __restrict__ C,
                                                          const void* __restrict__ offsets, int off_i64, int K, int N,
                                                          int max_seq_len) {
  __shared__ float sA[16][64 + 1];
  __shared__ float sB[16][64 + 1];
  const int b = blockIdx.z;
  const long long r0 = load_index(offsets, off_i64, b);
  long long len = load_index(offsets, off_i64, b + 1) - r0;
  const int n0 = blockIdx.y * 64;
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  const T* Bb = Bm + (long long)b * K * N;
  // m0 and len are uniform across the CTA, so the barriers below are too
  for (long long m0 = (long long)blockIdx.x * 64; m0 < len; m0 += (long long)gridDim.x * 64) {
    const bool live = m0 < max_seq_len;  // tiles at or past max_seq_len only store zeros
    float acc[4][4] = {};
    if (live) {
      for (int k0 = 0; k0 < K; k0 += 16) {
        for (int idx = tid; idx < 64 * 16; idx += 256) {
          const int r = idx >> 4, k = idx & 15;   // A tile: 64 rows x 16 k
          const long long row = m0 + r;
          float v = 0.f;
          if (row < len && row < max_seq_len && k0 + k < K) v = Cvt<T>::to_f(A[(r0 + row) * K + k0 + k]);
          sA[k][r] = v;
        }
        for (int idx = tid; idx < 64 * 16; idx += 256) {
          int k, n;
          if (TRANS_B) { n = idx >> 4; k = idx & 15; } else { k = idx >> 6; n = idx & 63; }
          float v = 0.f;
          if (k0 + k < K && n0 + n < N)
            v = Cvt<T>::to_f(TRANS_B ? Bb[(long long)(n0 + n) * K + k0 + k] : Bb[(long long)(k0 + k) * N + n0 + n]);
          sB[k][n] = v;
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < 16; ++k) {
          float a[4], bb[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) a[i] = sA[k][ty * 4 + i];
#pragma unroll
          for (int j = 0; j < 4; ++j) bb[j] = sB[k][tx * 4 + j];
#pragma unroll
          for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[i][j] += a[i] * bb[j];
        }
        __syncthreads();
      }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const long long row = m0 + ty * 4 + i;
      if (row >= len) continue;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int n = n0 + tx * 4 + j;
        if (n >= N) continue;
        float v = 0.f;
        if (row < max_seq_len) v = acc[i][j] + (bias ? Cvt<T>::to_f(bias[(long long)b * N + n]) : 0.f);
        C[(r0 + row) * N + n] = Cvt<T>::from_f(v);
      }
    }
  }
}

// dW[b][k, n] = sum_r A[r, k] G[r, n]; dbias[b, n] = sum_r G[r, n].  CTA = (64 k, 64 n) tile of one batch entry, rows in steps of 16.
template <typename T>
__global__ void __launch_bounds__(256) jagged_bmm_wgrad_kernel(const T* __restrict__ A, const T* __restrict__ G,
                                                                T* __restrict__ dW, T* __restrict__ dbias,
                                                                const void* __restrict__ offsets, int off_i64, int K, int N,
                                                                int max_seq_len) {
  __shared__ float sA[16][64 + 1];
  __shared__ float sG[16][64 + 1];
  const int b = blockIdx.z;
  const long long r0 = load_index(offsets, off_i64, b);
  long long len = load_index(offsets, off_i64, b + 1) - r0;
  len = len < max_seq_len ? len : max_seq_len;
  const int k0 = blockIdx.x * 64, n0 = blockIdx.y * 64;
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  float acc[4][4] = {};
  float bsum[4] = {};
  for (long long rr = 0; rr < len; rr += 16) {
    for (int idx = tid; idx < 16 * 64; idx += 256) {
      const int r = idx >> 6, c = idx & 63;
      const bool ok = rr + r < len;
      sA[r][c] = (ok && k0 + c < K) ? Cvt<T>::to_f(A[(r0 + rr + r) * K + k0 + c]) : 0.f;
      sG[r][c] = (ok && n0 + c < N) ? Cvt<T>::to_f(G[(r0 + rr + r) * N + n0 + c]) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < 16; ++r) {
      float a[4], g[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = sA[r][ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) g[j] = sG[r][tx * 4 + j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] += a[i] * g[j];
      if (ty == 0)
#pragma unroll
        for (int j = 0; j < 4; ++j) bsum[j] += g[j];
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int k = k0 + ty * 4 + i;
    if (k >= K) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n < N) dW[((long long)b * K + k) * N + n] = Cvt<T>::from_f(acc[i][j]);
    }
  }
  if (dbias && blockIdx.x == 0 && ty == 0)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n < N) dbias[(long long)b * N + n] = Cvt<T>::from_f(bsum[j]);
    }
}

template <typename T>
static int bmm_t(const void* A, const void* Bm, const void* bias, void* C, const void* off, int off_i64, int batch, int K, int N,
                 int max_seq_len, bool trans_b, cudaStream_t st) {
  dim3 grid((max_seq_len + 63) / 64, (N + 63) / 64, batch);
  if (trans_b)
    jagged_bmm_kernel<T, true><<<grid, 256, 0, st>>>((const T*)A, (const T*)Bm, (const T*)bias, (T*)C, off, off_i64, K, N, max_seq_len);
  else
    jagged_bmm_kernel<T, false><<<grid, 256, 0, st>>>((const T*)A, (const T*)Bm, (const T*)bias, (T*)C, off, off_i64, K, N, max_seq_len);
  HSTU_CUDA_OK(cudaGetLastError());
  return 0;
}

int jagged_bmm(const void* A, const void* Bm, const void* bias, void* C, const void* off, int off_i64, int batch, int K, int N,
               int max_seq_len, bool trans_b, int dtype, cudaStream_t st) {
  if (batch == 0) return 0;
  switch (dtype) {
    case HSTU_F32: return bmm_t<float>(A, Bm, bias, C, off, off_i64, batch, K, N, max_seq_len, trans_b, st);
    case HSTU_BF16: return bmm_t<__nv_bfloat16>(A, Bm, bias, C, off, off_i64, batch, K, N, max_seq_len, trans_b, st);
    case HSTU_F16: return bmm_t<__half>(A, Bm, bias, C, off, off_i64, batch, K, N, max_seq_len, trans_b, st);
  }
  set_error("jagged_bmm: bad dtype %d", dtype);
  return HSTU_ERR_INVALID_ARGUMENT;
}

template <typename T>
static int wgrad_t(const void* A, const void* G, void* dW, void* dbias, const void* off, int off_i64, int batch, int K, int N,
                   int max_seq_len, cudaStream_t st) {
  dim3 grid((K + 63) / 64, (N + 63) / 64, batch);
  jagged_bmm_wgrad_kernel<T><<<grid, 256, 0, st>>>((const T*)A, (const T*)G, (T*)dW, (T*)dbias, off, off_i64, K, N, max_seq_len);
  HSTU_CUDA_OK(cudaGetLastError());
  return 0;
}

int jagged_bmm_wgrad(const void* A, const void* G, void* dW, void* dbias, const void* off, int off_i64, int batch, int K, int N,
                     int max_seq_len, int dtype, cudaStream_t st) {
  if (batch == 0) return 0;
  switch (dtype) {
    case HSTU_F32: return wgrad_t<float>(A, G, dW, dbias, off, off_i64, batch, K, N, max_seq_len, st);
    case HSTU_BF16: return wgrad_t<__nv_bfloat16>(A, G, dW, dbias, off, off_i64, batch, K, N, max_seq_len, st);
    case HSTU_F16: return wgrad_t<__half>(A, G, dW, dbias, off, off_i64, batch, K, N, max_seq_len, st);
  }
  set_error("jagged_bmm_wgrad: bad dtype %d", dtype);
  return HSTU_ERR_INVALID_ARGUMENT;
}

}  // namespace hstu
