// TEST INFRASTRUCTURE (libhstu_b200_selftest.so, include/hstu_b200_selftest.h): on-device self test of the sm_90a building
// blocks the attention kernels are made of, on the same helpers (wgmma.cuh, tmap.cu):
//   TMA load of swizzled boxes (64B and 128B swizzle) completing on an mbarrier,
//   S = A B^T   wgmma with both operands K-major in shared memory          (score GEMMs of both kernels)
//   O = S V     wgmma with A = S from registers (hi + lo bf16), B MN-major   (P V, dV, dK)
//   E = W V     wgmma with A MN-major written by threads through swizzled_chunk_offset, B MN-major   (dQ = dS K)
//   S = A B^T   on e4m3 operands (m64n64k32, both K-major, byte TMA with 32B / 64B / 128B swizzle)  (scores of the fp8 forward)
// Inputs are multiples of 1/8 in [-1, 1] (of 1/4 for e4m3): every product and sum is exact in fp32 (and S fits the 16 bits of
// hi + lo), so the device results must equal the host reference exactly.
#include <stdarg.h>
#include <string.h>

#include <string>
#include <vector>

#include "common.cuh"
#include "wgmma.cuh"

namespace hstu {

static char g_selftest_err[512] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_selftest_err, sizeof(g_selftest_err), fmt, ap);
  va_end(ap);
}

using namespace wg;

// one warpgroup; A, B, V: [64 rows][D] bf16 loaded by TMA (swizzle 2D bytes); W: [64][64] bf16 in global memory
template <int D>
__global__ void __launch_bounds__(128) selftest_kernel(const __grid_constant__ CUtensorMap tA, const __grid_constant__ CUtensorMap tB,
                                                       const __grid_constant__ CUtensorMap tV, const uint16_t* W, float* S, float* O,
                                                       float* E) {
  constexpr int SW = D * 2, TILE = 64 * SW, WBYTES = 64 * 128;
  extern __shared__ uint8_t raw[];
  uint8_t* sm = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(raw) + 1023) & ~uintptr_t(1023));
  uint8_t *sA = sm, *sB = sm + TILE, *sV = sm + 2 * TILE, *sW = sm + 3 * TILE;
  uint64_t* bar = reinterpret_cast<uint64_t*>(sW + WBYTES);
  const int tid = threadIdx.x, w = tid >> 5, g = (tid & 31) >> 2, t4 = tid & 3;
  if (tid == 0) {
    mbar_init(bar, 1);
    fence_barrier_init();
  }
  // W as an MN-major operand: row k of the box holds W[0..63][k] (the layout of the backward's dS^T boxes)
  for (int idx = tid; idx < 64 * 64; idx += 128) {
    const int k = idx / 64, m = idx % 64;
    *reinterpret_cast<uint16_t*>(sW + swizzled_chunk_offset<128>(k, m >> 3) + (m & 7) * 2) = W[m * 64 + k];
  }
  fence_proxy_async_smem();
  __syncthreads();
  if (tid == 0) {
    mbar_arrive_expect_tx(bar, 3 * TILE);
    tma_load_3d(sA, &tA, bar, 0, 0, 0);
    tma_load_3d(sB, &tB, bar, 0, 0, 0);
    tma_load_3d(sV, &tV, bar, 0, 0, 0);
  }
  mbar_wait(bar, 0);

  float s[32];
  wgmma_fence();
#pragma unroll
  for (int ks = 0; ks < D / 16; ++ks)
    wgmma_ss<64, true, 0, 0>(s, desc_kmajor<SW>(smem_u32(sA), ks * 32), desc_kmajor<SW>(smem_u32(sB), ks * 32), ks > 0);
  wgmma_commit();
  wgmma_wait<0>();
  fence_regs(s);

  uint32_t a_hi[4][4], a_lo[4][4];
#pragma unroll
  for (int kk = 0; kk < 4; ++kk)
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const Operand<true> x(s[8 * kk + 2 * r], s[8 * kk + 2 * r + 1]);
      a_hi[kk][r] = x.hi;
      a_lo[kk][r] = x.lo;
    }
  float o[D / 2], e[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) o[i] = e[i] = 0.f;
  wgmma_fence();
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    const uint64_t vd = desc_mnmajor<SW>(smem_u32(sV), kk * 16, TILE);
    wgmma_rs<D, true, 1>(o, a_hi[kk], vd, 1);
    wgmma_rs<D, true, 1>(o, a_lo[kk], vd, 1);
    wgmma_ss<D, true, 1, 1>(e, desc_mnmajor<128>(smem_u32(sW), kk * 16, WBYTES), vd, 1);
  }
  wgmma_commit();
  wgmma_wait<0>();
  fence_regs(o);
  fence_regs(e);
  fence_regs(a_hi);
  fence_regs(a_lo);

#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = w * 16 + g + 8 * h;
#pragma unroll
    for (int nb = 0; nb < 8; ++nb)
#pragma unroll
      for (int c = 0; c < 2; ++c) S[row * 64 + nb * 8 + 2 * t4 + c] = s[nb * 4 + h * 2 + c];
#pragma unroll
    for (int nb = 0; nb < D / 8; ++nb)
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        O[row * D + nb * 8 + 2 * t4 + c] = o[nb * 4 + h * 2 + c];
        E[row * D + nb * 8 + 2 * t4 + c] = e[nb * 4 + h * 2 + c];
      }
  }
}

// one warpgroup; A, B: [64 rows][D] e4m3 loaded by TMA as bytes (swizzle D bytes, D <= 128)
template <int D>
__global__ void __launch_bounds__(128) selftest_e4m3_kernel(const __grid_constant__ CUtensorMap tA, const __grid_constant__ CUtensorMap tB,
                                                            float* S) {
  constexpr int SW = D, TILE = 64 * D;
  extern __shared__ uint8_t raw[];
  uint8_t* sm = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(raw) + 1023) & ~uintptr_t(1023));
  uint8_t *sA = sm, *sB = sm + TILE;
  uint64_t* bar = reinterpret_cast<uint64_t*>(sm + 2 * TILE);
  const int tid = threadIdx.x, w = tid >> 5, g = (tid & 31) >> 2, t4 = tid & 3;
  if (tid == 0) {
    mbar_init(bar, 1);
    fence_barrier_init();
  }
  __syncthreads();
  if (tid == 0) {
    mbar_arrive_expect_tx(bar, 2 * TILE);
    tma_load_3d(sA, &tA, bar, 0, 0, 0);
    tma_load_3d(sB, &tB, bar, 0, 0, 0);
  }
  mbar_wait(bar, 0);
  float s[32];
  wgmma_fence();
#pragma unroll
  for (int ks = 0; ks < D / 32; ++ks)
    wgmma_ss_64_e4m3(s, desc_kmajor<SW>(smem_u32(sA), ks * 32), desc_kmajor<SW>(smem_u32(sB), ks * 32), ks > 0);
  wgmma_commit();
  wgmma_wait<0>();
  fence_regs(s);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = w * 16 + g + 8 * h;
#pragma unroll
    for (int nb = 0; nb < 8; ++nb)
#pragma unroll
      for (int c = 0; c < 2; ++c) S[row * 64 + nb * 8 + 2 * t4 + c] = s[nb * 4 + h * 2 + c];
  }
}

static void appendf(std::string& s, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  s += buf;
}

#define ST_CUDA(expr)                                                                       \
  do {                                                                                      \
    cudaError_t _e = (expr);                                                                \
    if (_e != cudaSuccess) {                                                                \
      appendf(rep, "CUDA error: %s: %s\n", #expr, cudaGetErrorString(_e));                  \
      return -1;                                                                            \
    }                                                                                       \
  } while (0)

template <int D>
static int run_case(std::string& rep) {
  constexpr int SMEM = 3 * 64 * D * 2 + 64 * 128 + 64 + 1024;
  uint32_t rng = 12345u + D;
  auto next = [&]() {
    rng = rng * 1664525u + 1013904223u;
    return (float)((int)((rng >> 16) % 17) - 8) / 8.0f;  // multiple of 1/8 in [-1, 1]: exact in bf16
  };
  auto bits = [](float x) { uint32_t u; memcpy(&u, &x, 4); return (uint16_t)(u >> 16); };
  std::vector<float> A(64 * D), B(64 * D), V(64 * D), W(64 * 64);
  for (auto* m : {&A, &B, &V, &W})
    for (float& x : *m) x = next();
  std::vector<uint16_t> hA(64 * D), hB(64 * D), hV(64 * D), hW(64 * 64);
  for (int i = 0; i < 64 * D; ++i) hA[i] = bits(A[i]), hB[i] = bits(B[i]), hV[i] = bits(V[i]);
  for (int i = 0; i < 64 * 64; ++i) hW[i] = bits(W[i]);
  std::vector<double> rS(64 * 64, 0.0), rO(64 * D, 0.0), rE(64 * D, 0.0);
  for (int m = 0; m < 64; ++m)
    for (int n = 0; n < 64; ++n)
      for (int k = 0; k < D; ++k) rS[m * 64 + n] += (double)A[m * D + k] * B[n * D + k];
  for (int m = 0; m < 64; ++m)
    for (int n = 0; n < D; ++n)
      for (int k = 0; k < 64; ++k) {
        rO[m * D + n] += rS[m * 64 + k] * V[k * D + n];
        rE[m * D + n] += (double)W[m * 64 + k] * V[k * D + n];
      }

  uint16_t *dA, *dB, *dV, *dW;
  float *dS, *dO, *dE;
  ST_CUDA(cudaMalloc(&dA, 64 * D * 2));
  ST_CUDA(cudaMalloc(&dB, 64 * D * 2));
  ST_CUDA(cudaMalloc(&dV, 64 * D * 2));
  ST_CUDA(cudaMalloc(&dW, 64 * 64 * 2));
  ST_CUDA(cudaMalloc(&dS, 64 * 64 * 4));
  ST_CUDA(cudaMalloc(&dO, 64 * D * 4));
  ST_CUDA(cudaMalloc(&dE, 64 * D * 4));
  ST_CUDA(cudaMemcpy(dA, hA.data(), 64 * D * 2, cudaMemcpyHostToDevice));
  ST_CUDA(cudaMemcpy(dB, hB.data(), 64 * D * 2, cudaMemcpyHostToDevice));
  ST_CUDA(cudaMemcpy(dV, hV.data(), 64 * D * 2, cudaMemcpyHostToDevice));
  ST_CUDA(cudaMemcpy(dW, hW.data(), 64 * 64 * 2, cudaMemcpyHostToDevice));
  CUtensorMap tA, tB, tV;
  if (make_tmap_rows_heads(&tA, dA, 64, 1, D, D, D, D, 64) || make_tmap_rows_heads(&tB, dB, 64, 1, D, D, D, D, 64) ||
      make_tmap_rows_heads(&tV, dV, 64, 1, D, D, D, D, 64)) {
    appendf(rep, "tensor map: %s\n", g_selftest_err);
    return -1;
  }
  ST_CUDA(cudaFuncSetAttribute(selftest_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
  selftest_kernel<D><<<1, 128, SMEM>>>(tA, tB, tV, dW, dS, dO, dE);
  ST_CUDA(cudaGetLastError());
  ST_CUDA(cudaDeviceSynchronize());
  std::vector<float> S(64 * 64), O(64 * D), E(64 * D);
  ST_CUDA(cudaMemcpy(S.data(), dS, S.size() * 4, cudaMemcpyDeviceToHost));
  ST_CUDA(cudaMemcpy(O.data(), dO, O.size() * 4, cudaMemcpyDeviceToHost));
  ST_CUDA(cudaMemcpy(E.data(), dE, E.size() * 4, cudaMemcpyDeviceToHost));
  for (void* p : {(void*)dA, (void*)dB, (void*)dV, (void*)dW, (void*)dS, (void*)dO, (void*)dE}) cudaFree(p);

  int fails = 0;
  auto check = [&](const char* what, const std::vector<float>& got, const std::vector<double>& ref) {
    double worst = 0.0;
    for (size_t i = 0; i < ref.size(); ++i) worst = fmax(worst, fabs((double)got[i] - ref[i]));
    const bool ok = worst == 0.0;
    fails += ok ? 0 : 1;
    appendf(rep, "%s d=%d (swizzle %dB): max |device - host| = %g %s\n", what, D, 2 * D, worst, ok ? "ok" : "FAIL");
  };
  check("S = A B^T  (SS, K-major x K-major)", S, rS);
  check("O = S V    (RS, A hi + lo from the accumulator, B MN-major)", O, rO);
  check("E = W V    (SS, A MN-major via swizzled stores, B MN-major)", E, rE);
  return fails;
}

template <int D>
static int run_case_e4m3(std::string& rep) {
  constexpr int SMEM = 2 * 64 * D + 64 + 1024;
  uint32_t rng = 777u + D;
  // e4m3 bytes of j / 4, j in [-4, 4]: 0.25 = 2^-2 (exponent field 5), 0.5 (6), 0.75 = 1.5 * 2^-1 (6, mantissa 4), 1 (7)
  static const uint8_t kMag[5] = {0x00, 0x28, 0x30, 0x34, 0x38};
  std::vector<float> A(64 * D), B(64 * D);
  std::vector<uint8_t> hA(64 * D), hB(64 * D);
  for (int m = 0; m < 2; ++m)
    for (int i = 0; i < 64 * D; ++i) {
      rng = rng * 1664525u + 1013904223u;
      const int j = (int)((rng >> 16) % 9) - 4;
      (m ? B : A)[i] = j / 4.0f;
      (m ? hB : hA)[i] = (uint8_t)(kMag[j < 0 ? -j : j] | (j < 0 ? 0x80 : 0));
    }
  std::vector<double> rS(64 * 64, 0.0);
  for (int m = 0; m < 64; ++m)
    for (int n = 0; n < 64; ++n)
      for (int k = 0; k < D; ++k) rS[m * 64 + n] += (double)A[m * D + k] * B[n * D + k];
  uint8_t *dA, *dB;
  float* dS;
  ST_CUDA(cudaMalloc(&dA, 64 * D));
  ST_CUDA(cudaMalloc(&dB, 64 * D));
  ST_CUDA(cudaMalloc(&dS, 64 * 64 * 4));
  ST_CUDA(cudaMemcpy(dA, hA.data(), 64 * D, cudaMemcpyHostToDevice));
  ST_CUDA(cudaMemcpy(dB, hB.data(), 64 * D, cudaMemcpyHostToDevice));
  CUtensorMap tA, tB;
  if (make_tmap_rows_heads(&tA, dA, 64, 1, D, D, D, D, 64, 1) || make_tmap_rows_heads(&tB, dB, 64, 1, D, D, D, D, 64, 1)) {
    appendf(rep, "tensor map: %s\n", g_selftest_err);
    return -1;
  }
  ST_CUDA(cudaFuncSetAttribute(selftest_e4m3_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
  selftest_e4m3_kernel<D><<<1, 128, SMEM>>>(tA, tB, dS);
  ST_CUDA(cudaGetLastError());
  ST_CUDA(cudaDeviceSynchronize());
  std::vector<float> S(64 * 64);
  ST_CUDA(cudaMemcpy(S.data(), dS, S.size() * 4, cudaMemcpyDeviceToHost));
  for (void* p : {(void*)dA, (void*)dB, (void*)dS}) cudaFree(p);
  double worst = 0.0;
  for (size_t i = 0; i < rS.size(); ++i) worst = fmax(worst, fabs((double)S[i] - rS[i]));
  const bool ok = worst == 0.0;
  appendf(rep, "S = A B^T  (SS, e4m3 m64n64k32, K-major x K-major) d=%d (swizzle %dB): max |device - host| = %g %s\n", D, D, worst,
          ok ? "ok" : "FAIL");
  return ok ? 0 : 1;
}

}  // namespace hstu

extern "C" {

const char* hstu_selftest_last_error(void) { return hstu::g_selftest_err; }

int hstu_umma_selftest(char* report, size_t report_bytes) {
  std::string rep = "wgmma / TMA self test (sm_90a)\n";
  int dev = 0;
  cudaDeviceProp prop;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaGetDeviceProperties(&prop, dev) != cudaSuccess || prop.major != 9) {
    rep += "needs an sm_90 device\n";
    snprintf(report, report_bytes, "%s", rep.c_str());
    return -1;
  }
  hstu::appendf(rep, "device: %s\n", prop.name);
  int fails = 0;
  for (int r : {hstu::run_case<32>(rep), hstu::run_case<64>(rep), hstu::run_case_e4m3<32>(rep), hstu::run_case_e4m3<64>(rep),
                hstu::run_case_e4m3<128>(rep)})
    fails = (r < 0 || fails < 0) ? -1 : fails + r;
  if (report && report_bytes) snprintf(report, report_bytes, "%s", rep.c_str());
  return fails;
}

}  // extern "C"
