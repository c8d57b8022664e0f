// Row-wise normalisation kernels of the HSTU block (HBM-bound): LayerNorm / SwishLayerNorm / RMSNorm forward and
// backward, the fused output stage  y = u * Norm(attn)  [+ concat(u, attn, y)] [+ dropout]  forward and backward,
// and SiLU on a strided column block (the `u` quarter of uvqk).
//
// Reference semantics: ops/pytorch/pt_layer_norm.py:24-61, ops/layer_norm.py:138-158, ops/pytorch/pt_hstu_linear.py:23-66.
// Design: one warp per normalised vector (a row, or a (row, head) pair for group norm); the vector is read once with
// 128-bit loads into registers (<= 1024 elements), statistics via warp shuffles in fp32, written once.  Parameter
// gradients use per-lane register accumulators -> per-CTA shared-memory reduction -> `partial` rows -> one
// column-reduce kernel (two-stage, no atomics, deterministic).
#include "common.cuh"

namespace hstu {

// norm_fast.cu: the same kernels specialised for 16-bit elements and a normalised length of 256 (no predicates, packed math)
bool norm_fast_applicable(int dtype, int len);
int layer_norm_fwd_fast(const void* x, const void* w, const void* b, void* y, float* mean, float* rstd, long long n, long long xs,
                        long long ys, float eps, int dtype, cudaStream_t st);
int layer_norm_bwd_fast(const void* dy, const void* x, const void* w, const float* mean, const float* rstd, void* dx, float* partial,
                        long long n, long long xs, long long dys, long long dxs, int dtype, int* grid_out, cudaStream_t st);
int norm_mul_dropout_fwd_fast(const void* attn, const void* u, const void* w, const void* b, void* out, float* mean, float* rstd,
                              long long n, long long as, long long us, float eps, float p, unsigned long long seed, int dtype,
                              int silu_u, int concat, cudaStream_t st);
int norm_mul_dropout_bwd_fast(const void* dout, const void* attn, const void* u, const void* w, const void* b, const float* mean,
                              const float* rstd, void* dattn, void* du, float* partial, long long n, long long as, long long us,
                              long long das, long long dus, float p, unsigned long long seed, int dtype, int silu_u, int concat,
                              int* grid_out, cudaStream_t st);

constexpr int kNormThreads = 256;
constexpr int kNormWarps = kNormThreads / 32;
constexpr int kMaxPerLane = 32;     // 32 lanes * 32 = 1024 elements per normalised vector
constexpr int kPartialRows = 528;   // backward: 132 SMs * 4 CTAs (each CTA emits one partial row of dw/db)
constexpr int kFwdGridCap = 2112;   // forward: 132 SMs * 16 CTAs

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// element c of a vector of length D is owned by lane (c / VEC) % 32, slot ((c / VEC) / 32) * VEC + c % VEC
template <typename T, int VEC, int PL>
struct RowIO {
  static __device__ __forceinline__ void load(const T* row, int D, int lane, float (&v)[PL]) {
#pragma unroll
    for (int k = 0; k < PL / VEC; ++k) {
      const int c = (k * 32 + lane) * VEC;
      if (c < D) {
        if constexpr (VEC == 1) {
          v[k] = Cvt<T>::to_f(row[c]);
        } else {
          uint4 raw = *reinterpret_cast<const uint4*>(row + c);
          const T* e = reinterpret_cast<const T*>(&raw);
#pragma unroll
          for (int i = 0; i < VEC; ++i) v[k * VEC + i] = Cvt<T>::to_f(e[i]);
        }
      } else {
#pragma unroll
        for (int i = 0; i < VEC; ++i) v[k * VEC + i] = 0.f;
      }
    }
  }
  // L2 prefetch of the lane's part of a row (the row a warp will process in its NEXT iteration): a warp works on one row at a
  // time, so without it only one row of loads per warp is in flight and the kernels are bound by HBM latency, not bandwidth
  static __device__ __forceinline__ void prefetch(const T* row, int D, int lane) {
#ifdef HSTU_NORM_NO_PREFETCH
    return;
#endif
    if constexpr (VEC > 1) {
#pragma unroll
      for (int k = 0; k < PL / VEC; ++k) {
        const int c = (k * 32 + lane) * VEC;
        if (c < D) asm volatile("prefetch.global.L2 [%0];" ::"l"(row + c));
      }
    }
  }
  static __device__ __forceinline__ void store(T* row, int D, int lane, const float (&v)[PL]) {
#pragma unroll
    for (int k = 0; k < PL / VEC; ++k) {
      const int c = (k * 32 + lane) * VEC;
      if (c < D) {
        if constexpr (VEC == 1) {
          row[c] = Cvt<T>::from_f(v[k]);
        } else {
          uint4 raw;
          T* e = reinterpret_cast<T*>(&raw);
#pragma unroll
          for (int i = 0; i < VEC; ++i) e[i] = Cvt<T>::from_f(v[k * VEC + i]);
          *reinterpret_cast<uint4*>(row + c) = raw;
        }
      }
    }
  }
};

#define FOR_OWNED(VEC, D, lane, k, i, c)                  \
  _Pragma("unroll") for (int k = 0; k < PL / VEC; ++k) \
  _Pragma("unroll") for (int i = 0; i < VEC; ++i)         \
    if (int c = (k * 32 + lane) * VEC + i; c < D)

// Dropout decisions: counter-based, one splitmix64 finaliser of (seed, index / 4) yields the four 16-bit uniforms of four
// consecutive elements (keep iff r16 >= round(p * 65536)).  Forward and backward -- and the vectorised and scalar paths --
// evaluate the same function of the element index, so the masks always agree.  (One hash per element made the output
// stage ALU-bound: ~90 integer instructions per element against ~10 for the rest of the kernel.)
__device__ __forceinline__ unsigned long long dropout_hash4(unsigned long long seed, unsigned long long idx4) {
  unsigned long long z = seed + 0x9E3779B97F4A7C15ull * (idx4 + 1);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
__device__ __forceinline__ uint32_t dropout_threshold(float p) {
  const float t = p * 65536.0f + 0.5f;
  return t >= 65536.f ? 65536u : (uint32_t)t;  // p = 1 drops everything
}
__device__ __forceinline__ bool dropout_keep(unsigned long long seed, unsigned long long idx, uint32_t thr) {
  const unsigned long long z = dropout_hash4(seed, idx >> 2);
  return (uint32_t)((z >> (16 * (idx & 3))) & 0xffffu) >= thr;
}
// v[] holds the lane's elements of one vector (RowIO layout) whose first element has flat index `base`
template <int VEC, int PL>
__device__ __forceinline__ void apply_dropout(float (&v)[PL], int len, int lane, unsigned long long base,
                                              unsigned long long seed, uint32_t thr, float keep_scale) {
  if constexpr (VEC % 4 == 0) {
    // vector path: base and every chunk start are multiples of 4 (len % VEC == 0 is a precondition of this path)
#pragma unroll
    for (int k = 0; k < PL / VEC; ++k) {
      const int c0 = (k * 32 + lane) * VEC;
      if (c0 < len) {
#pragma unroll
        for (int g = 0; g < VEC / 4; ++g) {
          const unsigned long long z = dropout_hash4(seed, (base + c0 + g * 4) >> 2);
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const bool keep = (uint32_t)((z >> (16 * e)) & 0xffffu) >= thr;
            v[k * VEC + g * 4 + e] = keep ? v[k * VEC + g * 4 + e] * keep_scale : 0.f;
          }
        }
      }
    }
  } else {
#pragma unroll
    for (int k = 0; k < PL / VEC; ++k)
#pragma unroll
      for (int i = 0; i < VEC; ++i) {
        const int c = (k * 32 + lane) * VEC + i;
        if (c < len) v[k * VEC + i] = dropout_keep(seed, base + c, thr) ? v[k * VEC + i] * keep_scale : 0.f;
      }
  }
}

// ------------------------------------------------------------------------------------------------
// LayerNorm / SwishLayerNorm / RMSNorm forward
// ------------------------------------------------------------------------------------------------
template <typename T, int VEC, int PL, bool RMS>
__global__ void __launch_bounds__(kNormThreads) ln_fwd_kernel(const T* __restrict__ x, const T* __restrict__ w,
                                                               const T* __restrict__ b, T* __restrict__ y,
                                                               float* __restrict__ mean_out, float* __restrict__ rstd_out,
                                                               long long n_rows, int D, long long xs, long long ys,
                                                               float eps, int swish) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float wv[PL], bv[PL];
  if (w) RowIO<T, VEC, PL>::load(w, D, lane, wv);
  if (b) RowIO<T, VEC, PL>::load(b, D, lane, bv);
  const float inv_d = 1.0f / (float)D;
  const long long rstep = (long long)gridDim.x * kNormWarps;
  for (long long r = (long long)blockIdx.x * kNormWarps + warp; r < n_rows; r += rstep) {
    float v[PL];
    if (r + rstep < n_rows) RowIO<T, VEC, PL>::prefetch(x + (r + rstep) * xs, D, lane);
    RowIO<T, VEC, PL>::load(x + r * xs, D, lane, v);
    float mean = 0.f;
    if constexpr (!RMS) {
      float s = 0.f;
#pragma unroll
      for (int i = 0; i < PL; ++i) s += v[i];
      mean = warp_sum(s) * inv_d;
    }
    float s2 = 0.f;
    FOR_OWNED(VEC, D, lane, k, i, c) {
      const float dlt = v[k * VEC + i] - mean;
      s2 += dlt * dlt;
    }
    const float rstd = rsqrtf(warp_sum(s2) * inv_d + eps);
    float o[PL];
#pragma unroll
    for (int i = 0; i < PL; ++i) {
      float z = (v[i] - mean) * rstd;
      if (w) z *= wv[i];
      if (b) z += bv[i];
      o[i] = swish ? v[i] * sigmoid_f(z) : z;
    }
    RowIO<T, VEC, PL>::store(y + r * ys, D, lane, o);
    if (lane == 0) {
      if (mean_out) mean_out[r] = mean;
      if (rstd_out) rstd_out[r] = rstd;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// LayerNorm / SwishLayerNorm / RMSNorm backward (dx + partial dw/db)
// ------------------------------------------------------------------------------------------------
template <typename T, int VEC, int PL, bool RMS>
__global__ void __launch_bounds__(kNormThreads) ln_bwd_kernel(const T* __restrict__ dy, const T* __restrict__ x,
                                                               const T* __restrict__ w, const T* __restrict__ b,
                                                               const float* __restrict__ mean_in,
                                                               const float* __restrict__ rstd_in, T* __restrict__ dx,
                                                               float* __restrict__ partial, long long n_rows, int D,
                                                               long long xs, long long dys, long long dxs, int swish) {
  extern __shared__ float red[];  // [kNormWarps][2][D]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float wv[PL], bv[PL];
  if (w) RowIO<T, VEC, PL>::load(w, D, lane, wv);
  if (b) RowIO<T, VEC, PL>::load(b, D, lane, bv);
  float aw[PL], ab[PL];
#pragma unroll
  for (int i = 0; i < PL; ++i) aw[i] = ab[i] = 0.f;
  const float inv_d = 1.0f / (float)D;
  const long long rstep = (long long)gridDim.x * kNormWarps;
  for (long long r = (long long)blockIdx.x * kNormWarps + warp; r < n_rows; r += rstep) {
    float xv[PL], g[PL];
    if (r + rstep < n_rows) {
      RowIO<T, VEC, PL>::prefetch(x + (r + rstep) * xs, D, lane);
      RowIO<T, VEC, PL>::prefetch(dy + (r + rstep) * dys, D, lane);
    }
    RowIO<T, VEC, PL>::load(x + r * xs, D, lane, xv);
    RowIO<T, VEC, PL>::load(dy + r * dys, D, lane, g);
    const float mean = RMS ? 0.f : mean_in[r];
    const float rstd = rstd_in[r];
    float direct[PL];
    float c1 = 0.f, c2 = 0.f;
#pragma unroll
    for (int i = 0; i < PL; ++i) {
      const float xhat = (xv[i] - mean) * rstd;
      float dz = g[i];
      direct[i] = 0.f;
      if (swish) {  // y = x * sig(z), z = xhat*w+b
        float z = xhat;
        if (w) z *= wv[i];
        if (b) z += bv[i];
        const float sg = sigmoid_f(z);
        direct[i] = g[i] * sg;
        dz = g[i] * xv[i] * sg * (1.f - sg);
      }
      aw[i] += dz * xhat;
      ab[i] += dz;
      const float wdy = w ? dz * wv[i] : dz;
      g[i] = wdy;
      c1 += xhat * wdy;
      c2 += wdy;
      xv[i] = xhat;
    }
    c1 = warp_sum(c1) * inv_d;
    c2 = RMS ? 0.f : warp_sum(c2) * inv_d;
    float o[PL];
#pragma unroll
    for (int i = 0; i < PL; ++i) o[i] = (g[i] - (xv[i] * c1 + c2)) * rstd + direct[i];
    RowIO<T, VEC, PL>::store(dx + r * dxs, D, lane, o);
  }
  if (partial == nullptr) return;
  FOR_OWNED(VEC, D, lane, k, i, c) {
    red[(warp * 2 + 0) * D + c] = aw[k * VEC + i];
    red[(warp * 2 + 1) * D + c] = ab[k * VEC + i];
  }
  __syncthreads();
  for (int c = threadIdx.x; c < 2 * D; c += kNormThreads) {
    float s = 0.f;
#pragma unroll
    for (int wp = 0; wp < kNormWarps; ++wp) s += red[wp * 2 * D + c];
    partial[(long long)blockIdx.x * 2 * D + c] = s;
  }
}

// out[c] = sum_r partial[r][c]   (c < ncols); out0 = first `split` columns, out1 = the rest (either nullable).
// One CTA per 32 columns: 32 row groups x 32 columns, every thread adds rows g, g + 32, ... (independent 128-byte coalesced
// loads), then the 32 group sums of a column are added in a fixed order -> deterministic.  (A thread per column walking all
// rows alone took 40 us for 592 x 512 -- as long as the layer-norm backward kernel it follows.)
constexpr int kColsumGroups = 32;
__global__ void __launch_bounds__(32 * kColsumGroups) colsum_kernel(const float* __restrict__ partial, int rows, int ncols,
                                                                    int split, float* out0, float* out1) {
  __shared__ float red[kColsumGroups][33];
  const int lane = threadIdx.x & 31, g = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + lane;
  float s = 0.f;
  if (c < ncols) {
#pragma unroll 4
    for (int r = g; r < rows; r += kColsumGroups) s += partial[(long long)r * ncols + c];
  }
  red[g][lane] = s;
  __syncthreads();
  if (g == 0 && c < ncols) {
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < kColsumGroups; ++k) t += red[k][lane];
    if (c < split) {
      if (out0) out0[c] = t;
    } else {
      if (out1) out1[c - split] = t;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Output stage: y = u' * Norm(attn); out = dropout([u' | attn | y]) or dropout(y)
// A "vector" is a full row (layer norm: G = 1, len = H*dv) or one head of a row (group norm: G = H, len = dv).
// ------------------------------------------------------------------------------------------------
template <typename T, int VEC, int PL>
__global__ void __launch_bounds__(kNormThreads) nmd_fwd_kernel(const T* __restrict__ attn, const T* __restrict__ u,
                                                                const T* __restrict__ w, const T* __restrict__ b,
                                                                T* __restrict__ out, float* __restrict__ mean_out,
                                                                float* __restrict__ rstd_out, long long n_rows, int G,
                                                                int len, long long as, long long us, float eps, float p,
                                                                unsigned long long seed, int silu_u, int concat,
                                                                int group_norm) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int width = G * len;
  const long long os = (long long)(concat ? 3 : 1) * width;
  float wv[PL], bv[PL];
  if (!group_norm) {
    RowIO<T, VEC, PL>::load(w, len, lane, wv);
    RowIO<T, VEC, PL>::load(b, len, lane, bv);
  }
  const float inv_d = 1.0f / (float)len;
  const float keep_scale = p > 0.f ? 1.0f / (1.0f - p) : 1.0f;
  const uint32_t thr = dropout_threshold(p);
  const long long n_vec = n_rows * G;
  const long long vstep = (long long)gridDim.x * kNormWarps;
  for (long long vi = (long long)blockIdx.x * kNormWarps + warp; vi < n_vec; vi += vstep) {
    const long long r = vi / G;
    const int gidx = (int)(vi - r * G);
    float a[PL], uu[PL];
    if (vi + vstep < n_vec) {
      const long long r2 = (vi + vstep) / G;
      const int g2 = (int)(vi + vstep - r2 * G);
      RowIO<T, VEC, PL>::prefetch(attn + r2 * as + g2 * len, len, lane);
      RowIO<T, VEC, PL>::prefetch(u + r2 * us + g2 * len, len, lane);
    }
    RowIO<T, VEC, PL>::load(attn + r * as + gidx * len, len, lane, a);
    RowIO<T, VEC, PL>::load(u + r * us + gidx * len, len, lane, uu);
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < PL; ++i) s += a[i];
    const float mean = warp_sum(s) * inv_d;
    float s2 = 0.f;
    FOR_OWNED(VEC, len, lane, k, i, c) {
      const float dlt = a[k * VEC + i] - mean;
      s2 += dlt * dlt;
    }
    const float rstd = rsqrtf(warp_sum(s2) * inv_d + eps);
    float gw = 1.f, gb = 0.f;
    if (group_norm) {
      gw = Cvt<T>::to_f(w[gidx]);
      gb = Cvt<T>::to_f(b[gidx]);
    }
    float y[PL];
#pragma unroll
    for (int i = 0; i < PL; ++i) {
      if (silu_u) uu[i] = silu_f(uu[i]);
      const float xhat = (a[i] - mean) * rstd;
      const float nrm = group_norm ? xhat * gw + gb : xhat * wv[i] + bv[i];
      y[i] = uu[i] * nrm;
      if (concat == 2) a[i] = nrm;  // concat_ua (research block): the middle part is Norm(attn), not attn
    }
    T* orow = out + r * os + gidx * len;
    if (p > 0.f) {
      const unsigned long long base = (unsigned long long)r * os + gidx * len;
      if (concat) {
        apply_dropout<VEC, PL>(uu, len, lane, base, seed, thr, keep_scale);
        apply_dropout<VEC, PL>(a, len, lane, base + width, seed, thr, keep_scale);
        apply_dropout<VEC, PL>(y, len, lane, base + 2 * width, seed, thr, keep_scale);
      } else {
        apply_dropout<VEC, PL>(y, len, lane, base, seed, thr, keep_scale);
      }
    }
    if (concat) {
      RowIO<T, VEC, PL>::store(orow, len, lane, uu);
      RowIO<T, VEC, PL>::store(orow + width, len, lane, a);
      RowIO<T, VEC, PL>::store(orow + 2 * width, len, lane, y);
    } else {
      RowIO<T, VEC, PL>::store(orow, len, lane, y);
    }
    if (lane == 0) {
      if (mean_out) mean_out[vi] = mean;
      if (rstd_out) rstd_out[vi] = rstd;
    }
  }
}

template <typename T, int VEC, int PL>
__global__ void __launch_bounds__(kNormThreads) nmd_bwd_kernel(
    const T* __restrict__ dout, const T* __restrict__ attn, const T* __restrict__ u, const T* __restrict__ w,
    const T* __restrict__ b, const float* __restrict__ mean_in, const float* __restrict__ rstd_in, T* __restrict__ dattn,
    T* __restrict__ du, float* __restrict__ partial, long long n_rows, int G, int len, long long as, long long us,
    long long das, long long dus, float p, unsigned long long seed, int silu_u, int concat, int group_norm) {
  extern __shared__ float red[];  // LN: [kNormWarps][2][len]; GN: [kNormWarps][2][G]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int width = G * len;
  const long long os = (long long)(concat ? 3 : 1) * width;
  float wv[PL], bv[PL];
  float aw[PL], ab[PL];
#pragma unroll
  for (int i = 0; i < PL; ++i) aw[i] = ab[i] = 0.f;
  if (!group_norm) {
    RowIO<T, VEC, PL>::load(w, len, lane, wv);
    RowIO<T, VEC, PL>::load(b, len, lane, bv);
  } else {
    for (int c = threadIdx.x; c < kNormWarps * 2 * G; c += kNormThreads) red[c] = 0.f;
    __syncthreads();
  }
  const float inv_d = 1.0f / (float)len;
  const float keep_scale = p > 0.f ? 1.0f / (1.0f - p) : 1.0f;
  const uint32_t thr = dropout_threshold(p);
  const long long n_vec = n_rows * G;
  const long long vstep = (long long)gridDim.x * kNormWarps;
  for (long long vi = (long long)blockIdx.x * kNormWarps + warp; vi < n_vec; vi += vstep) {
    const long long r = vi / G;
    const int gidx = (int)(vi - r * G);
    float a[PL], uu[PL], gy[PL], gu[PL], ga[PL];
    if (vi + vstep < n_vec) {
      const long long r2 = (vi + vstep) / G;
      const int g2 = (int)(vi + vstep - r2 * G);
      RowIO<T, VEC, PL>::prefetch(attn + r2 * as + g2 * len, len, lane);
      RowIO<T, VEC, PL>::prefetch(u + r2 * us + g2 * len, len, lane);
      const T* d2 = dout + r2 * os + g2 * len;
      RowIO<T, VEC, PL>::prefetch(d2, len, lane);
      if (concat) {
        RowIO<T, VEC, PL>::prefetch(d2 + width, len, lane);
        RowIO<T, VEC, PL>::prefetch(d2 + 2 * width, len, lane);
      }
    }
    RowIO<T, VEC, PL>::load(attn + r * as + gidx * len, len, lane, a);
    RowIO<T, VEC, PL>::load(u + r * us + gidx * len, len, lane, uu);
    const T* drow = dout + r * os + gidx * len;
    if (concat) {
      RowIO<T, VEC, PL>::load(drow, len, lane, gu);
      RowIO<T, VEC, PL>::load(drow + width, len, lane, ga);
      RowIO<T, VEC, PL>::load(drow + 2 * width, len, lane, gy);
    } else {
      RowIO<T, VEC, PL>::load(drow, len, lane, gy);
#pragma unroll
      for (int i = 0; i < PL; ++i) gu[i] = ga[i] = 0.f;
    }
    if (p > 0.f) {
      const unsigned long long base = (unsigned long long)r * os + gidx * len;
      if (concat) {
        apply_dropout<VEC, PL>(gu, len, lane, base, seed, thr, keep_scale);
        apply_dropout<VEC, PL>(ga, len, lane, base + width, seed, thr, keep_scale);
        apply_dropout<VEC, PL>(gy, len, lane, base + 2 * width, seed, thr, keep_scale);
      } else {
        apply_dropout<VEC, PL>(gy, len, lane, base, seed, thr, keep_scale);
      }
    }
    const float mean = mean_in[vi], rstd = rstd_in[vi];
    float gw = 1.f, gb = 0.f;
    if (group_norm) {
      gw = Cvt<T>::to_f(w[gidx]);
      gb = Cvt<T>::to_f(b[gidx]);
    }
    float c1 = 0.f, c2 = 0.f, sgw = 0.f, sgb = 0.f;
#pragma unroll
    for (int i = 0; i < PL; ++i) {
      // concat_ua: the gradient of the middle part belongs to Norm(attn) and flows through the normalisation
      const float g_mid = concat == 2 ? ga[i] : 0.f;
      if (concat == 2) ga[i] = 0.f;
      const float upre = uu[i];
      float sg = 0.f;
      float ua = upre;
      if (silu_u) {
        sg = sigmoid_f(upre);
        ua = upre * sg;
      }
      const float xhat = (a[i] - mean) * rstd;
      const float wi = group_norm ? gw : wv[i];
      const float nrm = xhat * wi + (group_norm ? gb : bv[i]);
      float dua = gy[i] * nrm + gu[i];        // d/d u'
      const float dn = gy[i] * ua + g_mid;   // d/d Norm(attn)
      if (silu_u) dua *= sg * (1.f + upre * (1.f - sg));
      gu[i] = dua;
      if (group_norm) {
        sgw += dn * xhat;
        sgb += dn;
      } else {
        aw[i] += dn * xhat;
        ab[i] += dn;
      }
      const float wdy = dn * wi;
      gy[i] = wdy;
      c1 += xhat * wdy;
      c2 += wdy;
      a[i] = xhat;
    }
    c1 = warp_sum(c1) * inv_d;
    c2 = warp_sum(c2) * inv_d;
#pragma unroll
    for (int i = 0; i < PL; ++i) ga[i] += (gy[i] - (a[i] * c1 + c2)) * rstd;
    RowIO<T, VEC, PL>::store(dattn + r * das + gidx * len, len, lane, ga);
    RowIO<T, VEC, PL>::store(du + r * dus + gidx * len, len, lane, gu);
    if (group_norm) {
      sgw = warp_sum(sgw);
      sgb = warp_sum(sgb);
      if (lane == 0) {
        red[(warp * 2 + 0) * G + gidx] += sgw;
        red[(warp * 2 + 1) * G + gidx] += sgb;
      }
    }
  }
  if (partial == nullptr) return;
  const int np = group_norm ? G : len;
  if (!group_norm) {
    FOR_OWNED(VEC, len, lane, k, i, c) {
      red[(warp * 2 + 0) * len + c] = aw[k * VEC + i];
      red[(warp * 2 + 1) * len + c] = ab[k * VEC + i];
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < 2 * np; c += kNormThreads) {
    float s = 0.f;
#pragma unroll
    for (int wp = 0; wp < kNormWarps; ++wp) s += red[wp * 2 * np + c];
    partial[(long long)blockIdx.x * 2 * np + c] = s;
  }
}

// ------------------------------------------------------------------------------------------------
// SiLU on a strided [n_rows, n_cols] block
// ------------------------------------------------------------------------------------------------
template <typename T, int VEC, bool BWD>
__global__ void silu_kernel(const T* __restrict__ x, const T* __restrict__ dy, T* __restrict__ out, long long n_rows,
                            int n_cols, long long xs, long long dys, long long os) {
  // U independent 16-byte vectors per thread and iteration: all loads are issued before the first use, so that a thread has
  // U (forward) or 2 U (backward) requests in flight -- with one, 64 resident warps cover only half of the bandwidth-delay product
  constexpr int U = (VEC == 1 || BWD) ? 1 : 4;  // measured: the backward (two input streams) is fastest with one vector per thread
  const int vec_per_row = n_cols / VEC;
  const long long total = n_rows * vec_per_row;
  // a CTA works on contiguous chunks of U * blockDim vectors (thread t: vectors t, t + blockDim, ...): the U requests of a thread
  // stay within a few KB of each other (DRAM page locality) instead of a whole grid stride apart
  const long long stride = blockDim.x;
  const long long chunk = (long long)blockDim.x * U;
  for (long long idx0 = (long long)blockIdx.x * chunk + threadIdx.x; idx0 - threadIdx.x < total; idx0 += (long long)gridDim.x * chunk) {
    T xv[U][VEC], gv[U][VEC];
    long long xo[U], oo[U];
#pragma unroll
    for (int k = 0; k < U; ++k) {
      const long long idx = idx0 + k * stride;
      if (idx < total) {
        const long long r = idx / vec_per_row;
        const int c = (int)(idx - r * vec_per_row) * VEC;
        xo[k] = r * xs + c;
        oo[k] = r * os + c;
        if constexpr (VEC == 1) {
          xv[k][0] = x[xo[k]];
          if (BWD) gv[k][0] = dy[r * dys + c];
        } else {
          *reinterpret_cast<uint4*>(xv[k]) = *reinterpret_cast<const uint4*>(x + xo[k]);
          if (BWD) *reinterpret_cast<uint4*>(gv[k]) = *reinterpret_cast<const uint4*>(dy + r * dys + c);
        }
      }
    }
#pragma unroll
    for (int k = 0; k < U; ++k) {
      if (idx0 + k * stride < total) {
        T ov[VEC];
#pragma unroll
        for (int i = 0; i < VEC; ++i) {
          const float xf = Cvt<T>::to_f(xv[k][i]);
          const float sg = sigmoid_f(xf);
          float o = xf * sg;
          if (BWD) o = Cvt<T>::to_f(gv[k][i]) * sg * (1.f + xf * (1.f - sg));
          ov[i] = Cvt<T>::from_f(o);
        }
        if constexpr (VEC == 1) {
          out[oo[k]] = ov[0];
        } else {
          *reinterpret_cast<uint4*>(out + oo[k]) = *reinterpret_cast<const uint4*>(ov);
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
static inline bool aligned16(const void* p) { return p == nullptr || (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

static inline int norm_grid(long long n_vec, bool fwd = false) {
  long long need = (n_vec + kNormWarps - 1) / kNormWarps;
  if (need < 1) need = 1;
  const int cap = fwd ? kFwdGridCap : kPartialRows;
  return (int)(need < cap ? need : cap);
}

// 16-bit elements: every pointer 16-byte aligned, every row stride a multiple of 8 elements
static bool fast_layout(std::initializer_list<const void*> ptrs, std::initializer_list<long long> strides) {
#ifdef HSTU_NORM_NO_FAST
  return false;
#endif
  for (const void* p : ptrs)
    if (p == nullptr || !aligned16(p)) return false;
  for (long long s : strides)
    if (s % 8) return false;
  return true;
}

template <typename T>
static bool can_vec(int D, std::initializer_list<const void*> ptrs, std::initializer_list<long long> strides) {
  constexpr int VEC = 16 / sizeof(T);
  if (D % VEC) return false;
  for (const void* p : ptrs)
    if (!aligned16(p)) return false;
  for (long long s : strides)
    if (s % VEC) return false;
  return true;
}

// Calls F.template operator()<VEC, PL>() with the vector width / per-lane capacity that fit (D, alignment).
template <typename T, typename F>
static int dispatch_shape(int D, bool vec, F&& f) {
  constexpr int V = 16 / sizeof(T);
  if (D <= 256) return vec ? f.template operator()<V, 8>() : f.template operator()<1, 8>();
  if (D <= 512) return vec ? f.template operator()<V, 16>() : f.template operator()<1, 16>();
  return vec ? f.template operator()<V, 32>() : f.template operator()<1, 32>();
}

template <typename T>
static int ln_fwd_t(const void* x, const void* w, const void* b, void* y, float* mean, float* rstd, long long n, int D,
                    long long xs, long long ys, float eps, int swish, bool rms, cudaStream_t st) {
  const bool v = can_vec<T>(D, {x, w, b, y}, {xs, ys});
  const int grid = norm_grid(n, true);
  return dispatch_shape<T>(D, v, [&]<int VV, int PL>() -> int {
    if (rms)
      ln_fwd_kernel<T, VV, PL, true><<<grid, kNormThreads, 0, st>>>((const T*)x, (const T*)w, (const T*)b, (T*)y, mean,
                                                                    rstd, n, D, xs, ys, eps, swish);
    else
      ln_fwd_kernel<T, VV, PL, false><<<grid, kNormThreads, 0, st>>>((const T*)x, (const T*)w, (const T*)b, (T*)y, mean,
                                                                     rstd, n, D, xs, ys, eps, swish);
    HSTU_CUDA_OK(cudaGetLastError());
    return 0;
  });
}

template <typename T>
static int ln_bwd_t(const void* dy, const void* x, const void* w, const void* b, const float* mean, const float* rstd,
                    void* dx, float* dw, float* db, float* partial, long long n, int D, long long xs, long long dys,
                    long long dxs, int swish, bool rms, cudaStream_t st) {
  const bool v = can_vec<T>(D, {dy, x, w, b, dx}, {xs, dys, dxs});
  const int grid = norm_grid(n);
  const bool want_param = (dw != nullptr || db != nullptr);
  if (want_param && partial == nullptr) {
    set_error("layer_norm_bwd: dw/db requested but no partial scratch given");
    return HSTU_ERR_WORKSPACE;
  }
  float* part = want_param ? partial : nullptr;
  const size_t smem = sizeof(float) * kNormWarps * 2 * (size_t)D;
  int rc = dispatch_shape<T>(D, v, [&]<int VV, int PL>() -> int {
    if (rms) {
      HSTU_CUDA_OK(cudaFuncSetAttribute(ln_bwd_kernel<T, VV, PL, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      ln_bwd_kernel<T, VV, PL, true><<<grid, kNormThreads, smem, st>>>((const T*)dy, (const T*)x, (const T*)w, (const T*)b,
                                                                       mean, rstd, (T*)dx, part, n, D, xs, dys, dxs, swish);
    } else {
      HSTU_CUDA_OK(cudaFuncSetAttribute(ln_bwd_kernel<T, VV, PL, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      ln_bwd_kernel<T, VV, PL, false><<<grid, kNormThreads, smem, st>>>((const T*)dy, (const T*)x, (const T*)w, (const T*)b,
                                                                        mean, rstd, (T*)dx, part, n, D, xs, dys, dxs, swish);
    }
    HSTU_CUDA_OK(cudaGetLastError());
    return 0;
  });
  if (rc) return rc;
  if (want_param) {
    colsum_kernel<<<(2 * D + 31) / 32, 32 * kColsumGroups, 0, st>>>(part, grid, 2 * D, D, dw, db);
    HSTU_CUDA_OK(cudaGetLastError());
  }
  return 0;
}

#define DISPATCH_DTYPE(dt, CALL)                              \
  switch (dt) {                                               \
    case HSTU_F32: { using T = float; return CALL; }          \
    case HSTU_BF16: { using T = __nv_bfloat16; return CALL; } \
    case HSTU_F16: { using T = __half; return CALL; }         \
    default: set_error("unsupported dtype %d", dt); return HSTU_ERR_UNSUPPORTED; \
  }

int layer_norm_fwd(const void* x, const void* w, const void* b, void* y, float* mean, float* rstd, long long n, int D,
                   long long xs, long long ys, float eps, int dtype, int swish, bool rms, cudaStream_t st) {
  if (n == 0) return 0;
  if (D < 1 || D > 32 * kMaxPerLane) {
    set_error("layer_norm: D=%d outside the supported range [1, %d]", D, 32 * kMaxPerLane);
    return HSTU_ERR_UNSUPPORTED;
  }
  if (norm_fast_applicable(dtype, D) && !swish && !rms && fast_layout({x, w, b, y}, {xs, ys}))
    return layer_norm_fwd_fast(x, w, b, y, mean, rstd, n, xs, ys, eps, dtype, st);
  DISPATCH_DTYPE(dtype, (ln_fwd_t<T>(x, w, b, y, mean, rstd, n, D, xs, ys, eps, swish, rms, st)));
}

int layer_norm_bwd(const void* dy, const void* x, const void* w, const void* b, const float* mean, const float* rstd,
                   void* dx, float* dw, float* db, float* partial, long long n, int D, long long xs, long long dys,
                   long long dxs, int dtype, int swish, bool rms, cudaStream_t st) {
  if (D < 1 || D > 32 * kMaxPerLane) {
    set_error("layer_norm: D=%d outside the supported range [1, %d]", D, 32 * kMaxPerLane);
    return HSTU_ERR_UNSUPPORTED;
  }
  if (n == 0) {
    if (dw) HSTU_CUDA_OK(cudaMemsetAsync(dw, 0, sizeof(float) * D, st));
    if (db) HSTU_CUDA_OK(cudaMemsetAsync(db, 0, sizeof(float) * D, st));
    return 0;
  }
  if (norm_fast_applicable(dtype, D) && !swish && !rms && fast_layout({dy, x, w, b, dx}, {xs, dys, dxs})) {
    const bool want_param = (dw != nullptr || db != nullptr);
    if (want_param && partial == nullptr) {
      set_error("layer_norm_bwd: dw/db requested but no partial scratch given");
      return HSTU_ERR_WORKSPACE;
    }
    int grid = 0;
    if (int rc = layer_norm_bwd_fast(dy, x, w, mean, rstd, dx, want_param ? partial : nullptr, n, xs, dys, dxs, dtype, &grid, st))
      return rc;
    if (want_param) {
      colsum_kernel<<<(2 * D + 31) / 32, 32 * kColsumGroups, 0, st>>>(partial, grid, 2 * D, D, dw, db);
      HSTU_CUDA_OK(cudaGetLastError());
    }
    return 0;
  }
  DISPATCH_DTYPE(dtype, (ln_bwd_t<T>(dy, x, w, b, mean, rstd, dx, dw, db, partial, n, D, xs, dys, dxs, swish, rms, st)));
}

template <typename T>
static int nmd_fwd_t(const void* attn, const void* u, const void* w, const void* b, void* out, float* mean, float* rstd,
                     long long n, int H, int dv, long long as, long long us, float eps, float p, unsigned long long seed,
                     int silu_u, int concat, int gn, cudaStream_t st) {
  const int G = gn ? H : 1, len = gn ? dv : H * dv;
  // group norm: vectors start at head offsets g*len, and out rows at multiples of width -> need len % VEC == 0 (checked)
  const bool v = can_vec<T>(len, {attn, u, gn ? nullptr : w, gn ? nullptr : b, out}, {as, us});
  const int grid = norm_grid(n * G, true);
  return dispatch_shape<T>(len, v, [&]<int VV, int PL>() -> int {
    nmd_fwd_kernel<T, VV, PL><<<grid, kNormThreads, 0, st>>>((const T*)attn, (const T*)u, (const T*)w, (const T*)b,
                                                             (T*)out, mean, rstd, n, G, len, as, us, eps, p, seed, silu_u,
                                                             concat, gn);
    HSTU_CUDA_OK(cudaGetLastError());
    return 0;
  });
}

template <typename T>
static int nmd_bwd_t(const void* dout, const void* attn, const void* u, const void* w, const void* b, const float* mean,
                     const float* rstd, void* dattn, void* du, float* dw, float* db, float* partial, long long n, int H,
                     int dv, long long as, long long us, long long das, long long dus, float p, unsigned long long seed,
                     int silu_u, int concat, int gn, cudaStream_t st) {
  const int G = gn ? H : 1, len = gn ? dv : H * dv;
  const bool v = can_vec<T>(len, {dout, attn, u, gn ? nullptr : w, gn ? nullptr : b, dattn, du}, {as, us, das, dus});
  const int grid = norm_grid(n * G);
  const bool want_param = (dw != nullptr || db != nullptr);
  if (want_param && partial == nullptr) {
    set_error("norm_mul_dropout_bwd: dw/db requested but no partial scratch given");
    return HSTU_ERR_WORKSPACE;
  }
  float* part = want_param ? partial : nullptr;
  const int np = gn ? G : len;
  const size_t smem = sizeof(float) * kNormWarps * 2 * (size_t)np;
  int rc = dispatch_shape<T>(len, v, [&]<int VV, int PL>() -> int {
    HSTU_CUDA_OK(cudaFuncSetAttribute(nmd_bwd_kernel<T, VV, PL>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    nmd_bwd_kernel<T, VV, PL><<<grid, kNormThreads, smem, st>>>((const T*)dout, (const T*)attn, (const T*)u, (const T*)w,
                                                                (const T*)b, mean, rstd, (T*)dattn, (T*)du, part, n, G,
                                                                len, as, us, das, dus, p, seed, silu_u, concat, gn);
    HSTU_CUDA_OK(cudaGetLastError());
    return 0;
  });
  if (rc) return rc;
  if (want_param) {
    colsum_kernel<<<(2 * np + 31) / 32, 32 * kColsumGroups, 0, st>>>(part, grid, 2 * np, np, dw, db);
    HSTU_CUDA_OK(cudaGetLastError());
  }
  return 0;
}

int norm_mul_dropout_fwd(const void* attn, const void* u, const void* w, const void* b, void* out, float* mean,
                         float* rstd, long long n, int H, int dv, long long as, long long us, float eps, float p,
                         unsigned long long seed, int dtype, int silu_u, int concat, int gn, cudaStream_t st) {
  if (n == 0) return 0;
  const int len = gn ? dv : H * dv;
  if (len < 1 || len > 32 * kMaxPerLane) {
    set_error("norm_mul_dropout: normalised length %d outside [1, %d]", len, 32 * kMaxPerLane);
    return HSTU_ERR_UNSUPPORTED;
  }
  if (!gn && norm_fast_applicable(dtype, len) && fast_layout({attn, u, w, b, out}, {as, us}))
    return norm_mul_dropout_fwd_fast(attn, u, w, b, out, mean, rstd, n, as, us, eps, p, seed, dtype, silu_u, concat, st);
  DISPATCH_DTYPE(dtype, (nmd_fwd_t<T>(attn, u, w, b, out, mean, rstd, n, H, dv, as, us, eps, p, seed, silu_u, concat, gn, st)));
}

int norm_mul_dropout_bwd(const void* dout, const void* attn, const void* u, const void* w, const void* b,
                         const float* mean, const float* rstd, void* dattn, void* du, float* dw, float* db,
                         float* partial, long long n, int H, int dv, long long as, long long us, long long das,
                         long long dus, float p, unsigned long long seed, int dtype, int silu_u, int concat, int gn,
                         cudaStream_t st) {
  const int len = gn ? dv : H * dv;
  const int np = gn ? H : len;
  if (len < 1 || len > 32 * kMaxPerLane) {
    set_error("norm_mul_dropout: normalised length %d outside [1, %d]", len, 32 * kMaxPerLane);
    return HSTU_ERR_UNSUPPORTED;
  }
  if (n == 0) {
    if (dw) HSTU_CUDA_OK(cudaMemsetAsync(dw, 0, sizeof(float) * np, st));
    if (db) HSTU_CUDA_OK(cudaMemsetAsync(db, 0, sizeof(float) * np, st));
    return 0;
  }
  if (!gn && norm_fast_applicable(dtype, len) && fast_layout({dout, attn, u, w, b, dattn, du}, {as, us, das, dus})) {
    const bool want_param = (dw != nullptr || db != nullptr);
    if (want_param && partial == nullptr) {
      set_error("norm_mul_dropout_bwd: dw/db requested but no partial scratch given");
      return HSTU_ERR_WORKSPACE;
    }
    int grid = 0;
    if (int rc = norm_mul_dropout_bwd_fast(dout, attn, u, w, b, mean, rstd, dattn, du, want_param ? partial : nullptr, n, as, us,
                                           das, dus, p, seed, dtype, silu_u, concat, &grid, st))
      return rc;
    if (want_param) {
      colsum_kernel<<<(2 * len + 31) / 32, 32 * kColsumGroups, 0, st>>>(partial, grid, 2 * len, len, dw, db);
      HSTU_CUDA_OK(cudaGetLastError());
    }
    return 0;
  }
  DISPATCH_DTYPE(dtype, (nmd_bwd_t<T>(dout, attn, u, w, b, mean, rstd, dattn, du, dw, db, partial, n, H, dv, as, us, das,
                                      dus, p, seed, silu_u, concat, gn, st)));
}

template <typename T>
static int silu_t(const void* x, const void* dy, void* out, long long n, int cols, long long xs, long long dys,
                  long long os, bool bwd, cudaStream_t st) {
  constexpr int VEC = 16 / sizeof(T);
  const bool v = can_vec<T>(cols, {x, dy, out}, {xs, dys, os});
  const long long total = n * (cols / (v ? VEC : 1));
  const int per_thread = (v && !bwd) ? 4 : 1;  // the kernel's U
  long long blocks = (total + 256 * per_thread - 1) / (256 * per_thread);
  const long long cap = bwd ? 132 * 16 : 132 * 8;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
#define LAUNCH(VV, BB) silu_kernel<T, VV, BB><<<(int)blocks, 256, 0, st>>>((const T*)x, (const T*)dy, (T*)out, n, cols, xs, dys, os)
  if (bwd) {
    if (v) LAUNCH(VEC, true); else LAUNCH(1, true);
  } else {
    if (v) LAUNCH(VEC, false); else LAUNCH(1, false);
  }
#undef LAUNCH
  HSTU_CUDA_OK(cudaGetLastError());
  return 0;
}

int silu_fwd_bwd(const void* x, const void* dy, void* out, long long n, int cols, long long xs, long long dys,
                 long long os, int dtype, bool bwd, cudaStream_t st) {
  if (n == 0 || cols == 0) return 0;
  DISPATCH_DTYPE(dtype, (silu_t<T>(x, dy, out, n, cols, xs, dys, os, bwd, st)));
}

int norm_partial_rows() { return kPartialRows; }

}  // namespace hstu
