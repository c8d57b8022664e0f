// Row-wise kernels of the HSTU block, specialised for the shape every reference configuration of the hot path uses:
// 16-bit elements (bf16 / fp16), normalised length 256 (D = H * dv = 256), affine LayerNorm.  Same math and the same dropout
// function as the general kernels in norm.cu (which remain the path for every other shape); what changes is the instruction count.
//
// Why: at the bench shape the general kernels spend their instructions on per-element bounds predicates, scalar conversions and
// 64-bit index arithmetic rather than on the data they move.  Here one lane owns exactly
// one 16-byte vector of a row (no predicates), the math works on fp32 pairs, conversions work on pairs, a
// warp keeps TWO rows in flight and the next rows are prefetched into L2.
#include "common.cuh"

namespace hstu {

namespace {

// fp32 pair arithmetic, lane by lane with round-to-nearest (sm_90 has no packed fp32x2 instructions)
__device__ __forceinline__ float2 f2_mul(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 f2_add(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 f2_fma(float2 a, float2 b, float2 c) {
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}

constexpr int kFastThreads = 256;
constexpr int kFastWarps = kFastThreads / 32;
constexpr int kLen = 256;           // normalised length: 32 lanes x 8 elements
constexpr int kPartialRowsFast = 528;  // same as norm.cu: 132 SMs x 4 CTAs, one partial row of (dw | db) per CTA
constexpr int kFwdGridCapFast = 132 * 8;

template <typename T>
struct Pair16;
template <>
struct Pair16<__nv_bfloat16> {
  static __device__ __forceinline__ float2 up(uint32_t r) {
    return make_float2(__uint_as_float(r << 16), __uint_as_float(r & 0xffff0000u));
  }
  static __device__ __forceinline__ uint32_t pk(float2 v) {
    __nv_bfloat162 h = __floats2bfloat162_rn(v.x, v.y);
    return *reinterpret_cast<uint32_t*>(&h);
  }
};
template <>
struct Pair16<__half> {
  static __device__ __forceinline__ float2 up(uint32_t r) {
    __half2 h = *reinterpret_cast<__half2*>(&r);
    return __half22float2(h);
  }
  static __device__ __forceinline__ uint32_t pk(float2 v) {
    __half2 h = __floats2half2_rn(v.x, v.y);
    return *reinterpret_cast<uint32_t*>(&h);
  }
};

template <typename T>
__device__ __forceinline__ void unpack8(const uint4& raw, float2 (&v)[4]) {
  v[0] = Pair16<T>::up(raw.x);
  v[1] = Pair16<T>::up(raw.y);
  v[2] = Pair16<T>::up(raw.z);
  v[3] = Pair16<T>::up(raw.w);
}
template <typename T>
__device__ __forceinline__ uint4 pack8(const float2 (&v)[4]) {
  return make_uint4(Pair16<T>::pk(v[0]), Pair16<T>::pk(v[1]), Pair16<T>::pk(v[2]), Pair16<T>::pk(v[3]));
}
__device__ __forceinline__ uint4 ld16(const void* p) { return *reinterpret_cast<const uint4*>(p); }
__device__ __forceinline__ void st16(void* p, const uint4& v) { *reinterpret_cast<uint4*>(p) = v; }
__device__ __forceinline__ void pf_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
__device__ __forceinline__ float2 splat(float x) { return make_float2(x, x); }
__device__ __forceinline__ float hsum(float2 v) { return v.x + v.y; }

// butterfly sums of N independent values at once (the shuffles of different values overlap)
template <int N>
__device__ __forceinline__ void warp_sum_n(float (&v)[N]) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    float t[N];
#pragma unroll
    for (int i = 0; i < N; ++i) t[i] = __shfl_xor_sync(0xffffffffu, v[i], o);
#pragma unroll
    for (int i = 0; i < N; ++i) v[i] += t[i];
  }
}

__device__ __forceinline__ float fast_sigmoid(float x) { return __fdividef(1.0f, 1.0f + __expf(-x)); }

// the dropout function of norm.cu (dropout_hash4 / 16-bit fields), applied to the lane's 8 consecutive elements whose first has
// flat index `first` (a multiple of 8): two hashes, eight decisions
__device__ __forceinline__ unsigned long long hash4(unsigned long long seed, unsigned long long idx4) {
  unsigned long long z = seed + 0x9E3779B97F4A7C15ull * (idx4 + 1);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
__device__ __forceinline__ void dropout8(float2 (&v)[4], unsigned long long first, unsigned long long seed, uint32_t thr,
                                         float keep_scale) {
#pragma unroll
  for (int g = 0; g < 2; ++g) {
    const unsigned long long z = hash4(seed, (first >> 2) + g);
    const uint32_t lo = (uint32_t)z, hi = (uint32_t)(z >> 32);
    const float s0 = (lo & 0xffffu) >= thr ? keep_scale : 0.f;
    const float s1 = (lo >> 16) >= thr ? keep_scale : 0.f;
    const float s2 = (hi & 0xffffu) >= thr ? keep_scale : 0.f;
    const float s3 = (hi >> 16) >= thr ? keep_scale : 0.f;
    v[2 * g] = f2_mul(v[2 * g], make_float2(s0, s1));
    v[2 * g + 1] = f2_mul(v[2 * g + 1], make_float2(s2, s3));
  }
}
__device__ __forceinline__ uint32_t drop_threshold(float p) {
  const float t = p * 65536.0f + 0.5f;
  return t >= 65536.f ? 65536u : (uint32_t)t;
}

// ------------------------------------------------------------------------------------------------
// LayerNorm forward: y = (x - mean) rstd w + b
// ------------------------------------------------------------------------------------------------
template <typename T, int ROWS>
__global__ void __launch_bounds__(kFastThreads) ln_fwd_fast_kernel(const T* __restrict__ x, const T* __restrict__ w,
                                                                    const T* __restrict__ b, T* __restrict__ y,
                                                                    float* __restrict__ mean_out, float* __restrict__ rstd_out,
                                                                    long long n_rows, long long xs, long long ys, float eps) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int col = lane * 8;
  float2 wv[4], bv[4];
  unpack8<T>(ld16(w + col), wv);
  unpack8<T>(ld16(b + col), bv);
  const long long rstep = (long long)gridDim.x * kFastWarps;
  constexpr float inv_d = 1.0f / kLen;
  for (long long r0 = (long long)blockIdx.x * kFastWarps + warp; r0 < n_rows; r0 += ROWS * rstep) {
    uint4 raw[ROWS];
    bool ok[ROWS];
#pragma unroll
    for (int k = 0; k < ROWS; ++k) {
      const long long r = r0 + k * rstep;
      ok[k] = r < n_rows;
      raw[k] = ok[k] ? ld16(x + r * xs + col) : make_uint4(0, 0, 0, 0);
    }
#pragma unroll
    for (int k = 0; k < ROWS; ++k) {
      const long long r = r0 + (ROWS + k) * rstep;
      if (r < n_rows) pf_l2(x + r * xs + col);
    }
    float2 v[ROWS][4];
    float s[ROWS];
#pragma unroll
    for (int k = 0; k < ROWS; ++k) {
      unpack8<T>(raw[k], v[k]);
      s[k] = hsum(f2_add(f2_add(v[k][0], v[k][1]), f2_add(v[k][2], v[k][3])));
    }
    warp_sum_n<ROWS>(s);
    float mean[ROWS], q[ROWS];
#pragma unroll
    for (int k = 0; k < ROWS; ++k) {
      mean[k] = s[k] * inv_d;
      const float2 nm = splat(-mean[k]);
      float2 acc = make_float2(0.f, 0.f);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        v[k][i] = f2_add(v[k][i], nm);
        acc = f2_fma(v[k][i], v[k][i], acc);
      }
      q[k] = hsum(acc);
    }
    warp_sum_n<ROWS>(q);
#pragma unroll
    for (int k = 0; k < ROWS; ++k) {
      const float rstd = rsqrtf(q[k] * inv_d + eps);
      const float2 r2 = splat(rstd);
      float2 o[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) o[i] = f2_fma(f2_mul(v[k][i], r2), wv[i], bv[i]);
      const long long r = r0 + k * rstep;
      if (ok[k]) {
        st16(y + r * ys + col, pack8<T>(o));
        if (lane == 0) {
          if (mean_out) mean_out[r] = mean[k];
          if (rstd_out) rstd_out[r] = rstd;
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// LayerNorm backward: dx, partial (dw | db) per CTA
// ------------------------------------------------------------------------------------------------
template <typename T, int ROWS>
__global__ void __launch_bounds__(kFastThreads) ln_bwd_fast_kernel(const T* __restrict__ dy, const T* __restrict__ x,
                                                                    const T* __restrict__ w, const float* __restrict__ mean_in,
                                                                    const float* __restrict__ rstd_in, T* __restrict__ dx,
                                                                    float* __restrict__ partial, long long n_rows, long long xs,
                                                                    long long dys, long long dxs) {
  __shared__ float red[kFastWarps][2 * kLen];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int col = lane * 8;
  float2 wv[4], aw[4], ab[4];
  unpack8<T>(ld16(w + col), wv);
#pragma unroll
  for (int i = 0; i < 4; ++i) aw[i] = ab[i] = make_float2(0.f, 0.f);
  const long long rstep = (long long)gridDim.x * kFastWarps;
  constexpr float inv_d = 1.0f / kLen;
  for (long long r0 = (long long)blockIdx.x * kFastWarps + warp; r0 < n_rows; r0 += ROWS * rstep) {
    uint4 xr[ROWS], gr[ROWS];
    float mean[ROWS], rstd[ROWS];
    bool ok[ROWS];
#pragma unroll
    for (int k = 0; k < ROWS; ++k) {
      const long long r = r0 + k * rstep;
      ok[k] = r < n_rows;
      xr[k] = gr[k] = make_uint4(0, 0, 0, 0);  // a missing row contributes zeros everywhere
      mean[k] = 0.f;
      rstd[k] = 0.f;
      if (ok[k]) {
        xr[k] = ld16(x + r * xs + col);
        gr[k] = ld16(dy + r * dys + col);
        mean[k] = mean_in[r];
        rstd[k] = rstd_in[r];
      }
    }
#pragma unroll
    for (int k = 0; k < ROWS; ++k) {
      const long long r = r0 + (ROWS + k) * rstep;
      if (r < n_rows) {
        pf_l2(x + r * xs + col);
        pf_l2(dy + r * dys + col);
      }
    }
    float2 xh[ROWS][4], wd[ROWS][4];
    float c[2 * ROWS];
#pragma unroll
    for (int k = 0; k < ROWS; ++k) {
      float2 g[4];
      unpack8<T>(xr[k], xh[k]);
      unpack8<T>(gr[k], g);
      const float2 r2 = splat(rstd[k]), nm = splat(-mean[k] * rstd[k]);
      float2 c1 = make_float2(0.f, 0.f), c2 = make_float2(0.f, 0.f);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        xh[k][i] = f2_fma(xh[k][i], r2, nm);
        aw[i] = f2_fma(g[i], xh[k][i], aw[i]);
        ab[i] = f2_add(ab[i], g[i]);
        wd[k][i] = f2_mul(g[i], wv[i]);
        c1 = f2_fma(xh[k][i], wd[k][i], c1);
        c2 = f2_add(c2, wd[k][i]);
      }
      c[2 * k] = hsum(c1);
      c[2 * k + 1] = hsum(c2);
    }
    warp_sum_n<2 * ROWS>(c);
#pragma unroll
    for (int k = 0; k < ROWS; ++k) {
      const float2 c1 = splat(-c[2 * k] * inv_d), c2 = splat(-c[2 * k + 1] * inv_d), r2 = splat(rstd[k]);
      float2 o[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) o[i] = f2_mul(f2_add(wd[k][i], f2_fma(xh[k][i], c1, c2)), r2);
      if (ok[k]) st16(dx + (r0 + k * rstep) * dxs + col, pack8<T>(o));
    }
  }
  if (partial == nullptr) return;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    red[warp][col + 2 * i] = aw[i].x;
    red[warp][col + 2 * i + 1] = aw[i].y;
    red[warp][kLen + col + 2 * i] = ab[i].x;
    red[warp][kLen + col + 2 * i + 1] = ab[i].y;
  }
  __syncthreads();
  for (int cidx = threadIdx.x; cidx < 2 * kLen; cidx += kFastThreads) {
    float s = 0.f;
#pragma unroll
    for (int wp = 0; wp < kFastWarps; ++wp) s += red[wp][cidx];
    partial[(long long)blockIdx.x * 2 * kLen + cidx] = s;
  }
}

// ------------------------------------------------------------------------------------------------
// Output stage forward: y = u' * LN(attn); out = dropout(y) or dropout([u' | attn or LN(attn) | y])
// ------------------------------------------------------------------------------------------------
template <typename T, int CONCAT, int ROWS>
__global__ void __launch_bounds__(kFastThreads) nmd_fwd_fast_kernel(const T* __restrict__ attn, const T* __restrict__ u,
                                                                     const T* __restrict__ w, const T* __restrict__ b,
                                                                     T* __restrict__ out, float* __restrict__ mean_out,
                                                                     float* __restrict__ rstd_out, long long n_rows, long long as,
                                                                     long long us, float eps, float p, unsigned long long seed,
                                                                     int silu_u) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int col = lane * 8;
  constexpr long long os = (CONCAT ? 3 : 1) * kLen;
  float2 wv[4], bv[4];
  unpack8<T>(ld16(w + col), wv);
  unpack8<T>(ld16(b + col), bv);
  const float keep_scale = p > 0.f ? 1.0f / (1.0f - p) : 1.0f;
  const uint32_t thr = drop_threshold(p);
  const long long rstep = (long long)gridDim.x * kFastWarps;
  constexpr float inv_d = 1.0f / kLen;
  for (long long r0 = (long long)blockIdx.x * kFastWarps + warp; r0 < n_rows; r0 += ROWS * rstep) {
    uint4 ar[ROWS], ur[ROWS];
    bool ok[ROWS];
#pragma unroll
    for (int k = 0; k < ROWS; ++k) {
      const long long r = r0 + k * rstep;
      ok[k] = r < n_rows;
      ar[k] = ur[k] = make_uint4(0, 0, 0, 0);
      if (ok[k]) {
        ar[k] = ld16(attn + r * as + col);
        ur[k] = ld16(u + r * us + col);
      }
    }
#pragma unroll
    for (int k = 0; k < ROWS; ++k) {
      const long long r = r0 + (ROWS + k) * rstep;
      if (r < n_rows) {
        pf_l2(attn + r * as + col);
        pf_l2(u + r * us + col);
      }
    }
    float2 a[ROWS][4], d[ROWS][4];
    float s[ROWS], q[ROWS], mean[ROWS];
#pragma unroll
    for (int k = 0; k < ROWS; ++k) {
      unpack8<T>(ar[k], a[k]);
      s[k] = hsum(f2_add(f2_add(a[k][0], a[k][1]), f2_add(a[k][2], a[k][3])));
    }
    warp_sum_n<ROWS>(s);
#pragma unroll
    for (int k = 0; k < ROWS; ++k) {
      mean[k] = s[k] * inv_d;
      const float2 nm = splat(-mean[k]);
      float2 acc = make_float2(0.f, 0.f);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        d[k][i] = f2_add(a[k][i], nm);
        acc = f2_fma(d[k][i], d[k][i], acc);
      }
      q[k] = hsum(acc);
    }
    warp_sum_n<ROWS>(q);
#pragma unroll
    for (int k = 0; k < ROWS; ++k) {
      const long long r = r0 + k * rstep;
      const float rstd = rsqrtf(q[k] * inv_d + eps);
      const float2 r2 = splat(rstd);
      float2 uu[4], y[4];
      unpack8<T>(ur[k], uu);
      if (silu_u) {
#pragma unroll
        for (int i = 0; i < 4; ++i) uu[i] = make_float2(uu[i].x * fast_sigmoid(uu[i].x), uu[i].y * fast_sigmoid(uu[i].y));
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 nrm = f2_fma(f2_mul(d[k][i], r2), wv[i], bv[i]);
        y[i] = f2_mul(uu[i], nrm);
        if (CONCAT == 2) a[k][i] = nrm;  // concat_ua: the middle part is LN(attn)
      }
      if (!ok[k]) continue;
      T* orow = out + r * os + col;
      const unsigned long long first = (unsigned long long)r * os + col;
      if (CONCAT) {
        if (p > 0.f) {
          dropout8(uu, first, seed, thr, keep_scale);
          dropout8(a[k], first + kLen, seed, thr, keep_scale);
          dropout8(y, first + 2 * kLen, seed, thr, keep_scale);
        }
        st16(orow, pack8<T>(uu));
        st16(orow + kLen, pack8<T>(a[k]));
        st16(orow + 2 * kLen, pack8<T>(y));
      } else {
        if (p > 0.f) dropout8(y, first, seed, thr, keep_scale);
        st16(orow, pack8<T>(y));
      }
      if (lane == 0) {
        if (mean_out) mean_out[r] = mean[k];
        if (rstd_out) rstd_out[r] = rstd;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Output stage backward: dattn, du, partial (dw | db) per CTA
// ------------------------------------------------------------------------------------------------
template <typename T, int CONCAT>
__global__ void __launch_bounds__(kFastThreads, 2) nmd_bwd_fast_kernel(
    const T* __restrict__ dout, const T* __restrict__ attn, const T* __restrict__ u, const T* __restrict__ w,
    const T* __restrict__ b, const float* __restrict__ mean_in, const float* __restrict__ rstd_in, T* __restrict__ dattn,
    T* __restrict__ du, float* __restrict__ partial, long long n_rows, long long as, long long us, long long das, long long dus,
    float p, unsigned long long seed, int silu_u) {
  __shared__ float red[kFastWarps][2 * kLen];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int col = lane * 8;
  constexpr long long os = (CONCAT ? 3 : 1) * kLen;
  float2 wv[4], bv[4], aw[4], ab[4];
  unpack8<T>(ld16(w + col), wv);
  unpack8<T>(ld16(b + col), bv);
#pragma unroll
  for (int i = 0; i < 4; ++i) aw[i] = ab[i] = make_float2(0.f, 0.f);
  const float keep_scale = p > 0.f ? 1.0f / (1.0f - p) : 1.0f;
  const uint32_t thr = drop_threshold(p);
  const long long rstep = (long long)gridDim.x * kFastWarps;
  constexpr float inv_d = 1.0f / kLen;
  for (long long r = (long long)blockIdx.x * kFastWarps + warp; r < n_rows; r += rstep) {
    const T* drow = dout + r * os + col;
    const uint4 ar = ld16(attn + r * as + col), ur = ld16(u + r * us + col);
    uint4 g0 = ld16(drow), g1 = make_uint4(0, 0, 0, 0), g2 = make_uint4(0, 0, 0, 0);
    if (CONCAT) {
      g1 = ld16(drow + kLen);
      g2 = ld16(drow + 2 * kLen);
    }
    const float mean = mean_in[r], rstd = rstd_in[r];
    if (r + rstep < n_rows) {
      const long long rn = r + rstep;
      pf_l2(attn + rn * as + col);
      pf_l2(u + rn * us + col);
      pf_l2(dout + rn * os + col);
      if (CONCAT) {
        pf_l2(dout + rn * os + col + kLen);
        pf_l2(dout + rn * os + col + 2 * kLen);
      }
    }
    float2 a[4], uu[4], gy[4], gu[4], ga[4];
    unpack8<T>(ar, a);
    unpack8<T>(ur, uu);
    if (CONCAT) {
      unpack8<T>(g0, gu);
      unpack8<T>(g1, ga);
      unpack8<T>(g2, gy);
    } else {
      unpack8<T>(g0, gy);
#pragma unroll
      for (int i = 0; i < 4; ++i) gu[i] = ga[i] = make_float2(0.f, 0.f);
    }
    if (p > 0.f) {
      const unsigned long long first = (unsigned long long)r * os + col;
      if (CONCAT) {
        dropout8(gu, first, seed, thr, keep_scale);
        dropout8(ga, first + kLen, seed, thr, keep_scale);
        dropout8(gy, first + 2 * kLen, seed, thr, keep_scale);
      } else {
        dropout8(gy, first, seed, thr, keep_scale);
      }
    }
    const float2 r2 = splat(rstd), nm = splat(-mean * rstd);
    float2 c1 = make_float2(0.f, 0.f), c2 = make_float2(0.f, 0.f);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 xhat = f2_fma(a[i], r2, nm);
      const float2 nrm = f2_fma(xhat, wv[i], bv[i]);
      float2 ua = uu[i];
      float2 dsil = make_float2(1.f, 1.f);
      if (silu_u) {
        const float sx = fast_sigmoid(uu[i].x), sy = fast_sigmoid(uu[i].y);
        ua = make_float2(uu[i].x * sx, uu[i].y * sy);
        dsil = make_float2(sx * (1.f + uu[i].x * (1.f - sx)), sy * (1.f + uu[i].y * (1.f - sy)));
      }
      float2 dua = f2_fma(gy[i], nrm, gu[i]);                       // d / d u'
      // concat_ua: the gradient of the middle part belongs to LN(attn) and flows through the normalisation
      const float2 dn = CONCAT == 2 ? f2_fma(gy[i], ua, ga[i]) : f2_mul(gy[i], ua);  // d / d LN(attn)
      if (silu_u) dua = f2_mul(dua, dsil);
      gu[i] = dua;
      aw[i] = f2_fma(dn, xhat, aw[i]);
      ab[i] = f2_add(ab[i], dn);
      const float2 wdy = f2_mul(dn, wv[i]);
      c1 = f2_fma(xhat, wdy, c1);
      c2 = f2_add(c2, wdy);
      gy[i] = wdy;
      a[i] = xhat;
    }
    float c[2] = {hsum(c1), hsum(c2)};
    warp_sum_n<2>(c);
    const float2 k1 = splat(-c[0] * inv_d), k2 = splat(-c[1] * inv_d);
    float2 o[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      o[i] = f2_mul(f2_add(gy[i], f2_fma(a[i], k1, k2)), r2);
      if (CONCAT == 1) o[i] = f2_add(o[i], ga[i]);  // concat_ux: the middle part is attn itself
    }
    st16(dattn + r * das + col, pack8<T>(o));
    st16(du + r * dus + col, pack8<T>(gu));
  }
  if (partial == nullptr) return;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    red[warp][col + 2 * i] = aw[i].x;
    red[warp][col + 2 * i + 1] = aw[i].y;
    red[warp][kLen + col + 2 * i] = ab[i].x;
    red[warp][kLen + col + 2 * i + 1] = ab[i].y;
  }
  __syncthreads();
  for (int cidx = threadIdx.x; cidx < 2 * kLen; cidx += kFastThreads) {
    float s = 0.f;
#pragma unroll
    for (int wp = 0; wp < kFastWarps; ++wp) s += red[wp][cidx];
    partial[(long long)blockIdx.x * 2 * kLen + cidx] = s;
  }
}

inline int grid_for(long long n_rows, int rows_per_iter, int cap) {
  long long need = (n_rows + (long long)kFastWarps * rows_per_iter - 1) / ((long long)kFastWarps * rows_per_iter);
  if (need < 1) need = 1;
  return (int)(need < cap ? need : cap);
}

}  // namespace

// Each launcher returns -1 when the shape is not the specialised one (the caller then uses the general kernel), 0 on success.
bool norm_fast_applicable(int dtype, int len) { return (dtype == HSTU_BF16 || dtype == HSTU_F16) && len == kLen; }

template <typename T>
static int ln_fwd_fast_t(const void* x, const void* w, const void* b, void* y, float* mean, float* rstd, long long n, long long xs,
                         long long ys, float eps, cudaStream_t st) {
  constexpr int ROWS = 2;
  ln_fwd_fast_kernel<T, ROWS><<<grid_for(n, ROWS, kFwdGridCapFast), kFastThreads, 0, st>>>(
      (const T*)x, (const T*)w, (const T*)b, (T*)y, mean, rstd, n, xs, ys, eps);
  HSTU_CUDA_OK(cudaGetLastError());
  return 0;
}
int layer_norm_fwd_fast(const void* x, const void* w, const void* b, void* y, float* mean, float* rstd, long long n, long long xs,
                        long long ys, float eps, int dtype, cudaStream_t st) {
  return dtype == HSTU_BF16 ? ln_fwd_fast_t<__nv_bfloat16>(x, w, b, y, mean, rstd, n, xs, ys, eps, st)
                            : ln_fwd_fast_t<__half>(x, w, b, y, mean, rstd, n, xs, ys, eps, st);
}

template <typename T>
static int ln_bwd_fast_t(const void* dy, const void* x, const void* w, const float* mean, const float* rstd, void* dx,
                         float* partial, long long n, long long xs, long long dys, long long dxs, int* grid_out, cudaStream_t st) {
  constexpr int ROWS = 2;
  const int grid = grid_for(n, ROWS, kPartialRowsFast);
  *grid_out = grid;
  ln_bwd_fast_kernel<T, ROWS><<<grid, kFastThreads, 0, st>>>((const T*)dy, (const T*)x, (const T*)w, mean, rstd, (T*)dx, partial, n,
                                                             xs, dys, dxs);
  HSTU_CUDA_OK(cudaGetLastError());
  return 0;
}
int layer_norm_bwd_fast(const void* dy, const void* x, const void* w, const float* mean, const float* rstd, void* dx, float* partial,
                        long long n, long long xs, long long dys, long long dxs, int dtype, int* grid_out, cudaStream_t st) {
  return dtype == HSTU_BF16 ? ln_bwd_fast_t<__nv_bfloat16>(dy, x, w, mean, rstd, dx, partial, n, xs, dys, dxs, grid_out, st)
                            : ln_bwd_fast_t<__half>(dy, x, w, mean, rstd, dx, partial, n, xs, dys, dxs, grid_out, st);
}

template <typename T>
static int nmd_fwd_fast_t(const void* attn, const void* u, const void* w, const void* b, void* out, float* mean, float* rstd,
                          long long n, long long as, long long us, float eps, float p, unsigned long long seed, int silu_u, int concat,
                          cudaStream_t st) {
  constexpr int ROWS = 2;
  const int grid = grid_for(n, ROWS, kFwdGridCapFast);
#define HSTU_NMD_FWD(C)                                                                                                          \
  nmd_fwd_fast_kernel<T, C, ROWS><<<grid, kFastThreads, 0, st>>>((const T*)attn, (const T*)u, (const T*)w, (const T*)b, (T*)out, \
                                                                 mean, rstd, n, as, us, eps, p, seed, silu_u)
  if (concat == 0) HSTU_NMD_FWD(0);
  else if (concat == 1) HSTU_NMD_FWD(1);
  else HSTU_NMD_FWD(2);
#undef HSTU_NMD_FWD
  HSTU_CUDA_OK(cudaGetLastError());
  return 0;
}
int norm_mul_dropout_fwd_fast(const void* attn, const void* u, const void* w, const void* b, void* out, float* mean, float* rstd,
                              long long n, long long as, long long us, float eps, float p, unsigned long long seed, int dtype,
                              int silu_u, int concat, cudaStream_t st) {
  return dtype == HSTU_BF16
             ? nmd_fwd_fast_t<__nv_bfloat16>(attn, u, w, b, out, mean, rstd, n, as, us, eps, p, seed, silu_u, concat, st)
             : nmd_fwd_fast_t<__half>(attn, u, w, b, out, mean, rstd, n, as, us, eps, p, seed, silu_u, concat, st);
}

template <typename T>
static int nmd_bwd_fast_t(const void* dout, const void* attn, const void* u, const void* w, const void* b, const float* mean,
                          const float* rstd, void* dattn, void* du, float* partial, long long n, long long as, long long us,
                          long long das, long long dus, float p, unsigned long long seed, int silu_u, int concat, int* grid_out,
                          cudaStream_t st) {
  const int grid = grid_for(n, 1, kPartialRowsFast);
  *grid_out = grid;
#define HSTU_NMD_BWD(C)                                                                                                       \
  nmd_bwd_fast_kernel<T, C><<<grid, kFastThreads, 0, st>>>((const T*)dout, (const T*)attn, (const T*)u, (const T*)w, (const T*)b, \
                                                           mean, rstd, (T*)dattn, (T*)du, partial, n, as, us, das, dus, p, seed, \
                                                           silu_u)
  if (concat == 0) HSTU_NMD_BWD(0);
  else if (concat == 1) HSTU_NMD_BWD(1);
  else HSTU_NMD_BWD(2);
#undef HSTU_NMD_BWD
  HSTU_CUDA_OK(cudaGetLastError());
  return 0;
}
int norm_mul_dropout_bwd_fast(const void* dout, const void* attn, const void* u, const void* w, const void* b, const float* mean,
                              const float* rstd, void* dattn, void* du, float* partial, long long n, long long as, long long us,
                              long long das, long long dus, float p, unsigned long long seed, int dtype, int silu_u, int concat,
                              int* grid_out, cudaStream_t st) {
  return dtype == HSTU_BF16 ? nmd_bwd_fast_t<__nv_bfloat16>(dout, attn, u, w, b, mean, rstd, dattn, du, partial, n, as, us, das, dus,
                                                            p, seed, silu_u, concat, grid_out, st)
                            : nmd_bwd_fast_t<__half>(dout, attn, u, w, b, mean, rstd, dattn, du, partial, n, as, us, das, dus, p, seed,
                                                     silu_u, concat, grid_out, st);
}

}  // namespace hstu
