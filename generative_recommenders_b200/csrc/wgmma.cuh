// sm_90a primitives used by the wgmma/TMA attention kernels: mbarrier, TMA (cp.async.bulk.tensor), warpgroup MMA
// (wgmma.mma_async, shared-memory matrix descriptors, fence / commit / wait) and register-level helpers.  Everything is inline
// PTX; the encodings follow the PTX ISA "Asynchronous Warpgroup Level Matrix Multiply-Accumulate" chapter.
#pragma once
#include <cuda.h>  // CUtensorMap (types only; the driver entry point is resolved at run time)
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "wgmma_ops.cuh"

namespace hstu {
namespace wg {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

#ifndef HSTU_WAIT_LIMIT_CLK
#define HSTU_WAIT_LIMIT_CLK 4000000000ll  // bounded wait (~2 s): a protocol bug traps instead of hanging the GPU
#endif

// ---------------------------------------------------------------------------------------------
// mbarrier
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
#ifdef HSTU_DEBUG_SPIN
// debug build: report the wait site that timed out (line number) instead of trapping, then fall through
__device__ __forceinline__ void mbar_wait_line(uint64_t* bar, uint32_t parity, int line) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 20)) {
      printf("MBAR TIMEOUT line %d block (%d,%d,%d) thread %d parity %u\n", line, (int)blockIdx.x, (int)blockIdx.y,
             (int)blockIdx.z, (int)threadIdx.x, parity);
      return;
    }
  }
}
#define mbar_wait(bar, parity) mbar_wait_line(bar, parity, __LINE__)
#else
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  // bounded in TIME (try_wait may suspend the thread for a while, so a spin COUNT bounds nothing)
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > HSTU_WAIT_LIMIT_CLK) __trap();
  }
}
#endif

__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// ---------------------------------------------------------------------------------------------
// TMA loads (tile mode) into shared memory, completion on an mbarrier
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void prefetch_tensormap(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

// ---------------------------------------------------------------------------------------------
// wgmma: descriptors, ordering
// ---------------------------------------------------------------------------------------------
// 64-bit shared-memory matrix descriptor (sm_90): start address, leading / stride byte offsets (16-byte units), swizzle mode
// in bits 62-63 (1 = 128B, 2 = 64B, 3 = 32B).  Tiles are aligned to their swizzle atom, so the base-offset field stays 0.
__host__ __device__ constexpr int swizzle_mode(int swizzle_bytes) {
  return swizzle_bytes == 128 ? 1 : swizzle_bytes == 64 ? 2 : swizzle_bytes == 32 ? 3 : 0;
}
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes, int mode) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFFu) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32;
  d |= (uint64_t)(mode & 3) << 62;
  return d;
}
// K-major operand: rows x K, K contiguous, stored as boxes of [rows][SW bytes]; 8-row swizzle atoms of 8*SW bytes.  The
// 16-element K slice starting `k_byte_off` bytes into the row of the box at `box_addr` (LBO unused for swizzled K-major).
template <int SW>
__device__ __forceinline__ uint64_t desc_kmajor(uint32_t box_addr, uint32_t k_byte_off) {
  return make_desc(box_addr + k_byte_off, 16, 8 * SW, swizzle_mode(SW));
}
// MN-major operand: K rows x MN, MN contiguous, stored as boxes of [K rows][SW bytes] (SW/2 elements of MN per box, boxes
// `box_stride` bytes apart).  The 16 K rows starting at row k0: SBO = 8*SW (next 8 K rows), LBO = box_stride (next MN block).
template <int SW>
__device__ __forceinline__ uint64_t desc_mnmajor(uint32_t tile_addr, uint32_t k0_rows, uint32_t box_stride) {
  return make_desc(tile_addr + k0_rows * SW, box_stride, 8 * SW, swizzle_mode(SW));
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving reads / writes of accumulator registers across the asynchronous MMAs that own them
template <int N>
__device__ __forceinline__ void fence_regs(float (&r)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(r[i])::"memory");
}
// the same for A fragments in registers: they must stay intact until the MMA that reads them has completed
template <int M>
__device__ __forceinline__ void fence_regs(uint32_t (&r)[M][4]) {
#pragma unroll
  for (int i = 0; i < M; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) asm volatile("" : "+r"(r[i][j])::"memory");
}

// ---------------------------------------------------------------------------------------------
// register-level helpers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}
__device__ __forceinline__ uint32_t pack_f16x2(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}
// saturating form (clamps to +-65504 instead of producing inf): used for the fp16 tensor-core operands P / dS
__device__ __forceinline__ uint32_t pack_f16x2_sat(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}
__device__ __forceinline__ float tanh_approx(float x) {
  float y;
  asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// A 16-bit MMA operand computed in fp32 (P or dS).  wgmma takes ONE format for A and B, so with bf16 inputs the operand is
// bf16, and its 8-bit significand alone costs ~1.7e-3 of relative error.  It is therefore split into hi = bf16(x) and
// lo = bf16(x - hi) (16 significant bits together) and multiplied twice; fp16 inputs use one fp16 operand (11 bits).
template <bool BF16>
struct Operand {
  uint32_t hi, lo;
  __device__ __forceinline__ Operand(float a, float b) {
    if constexpr (BF16) {
      hi = pack_bf16x2(a, b);
      const float ha = __uint_as_float(hi << 16), hb = __uint_as_float(hi & 0xffff0000u);
      lo = pack_bf16x2(a - ha, b - hb);
    } else {
      hi = pack_f16x2_sat(a, b);
      lo = 0u;
    }
  }
};

// Byte offset of the 16-byte chunk `chunk` of row `row` inside a [rows][SW bytes] swizzled box whose base is aligned to
// 8*SW bytes (Swizzle<B,4,3>: byte-address bits [4, 4+B) ^= bits [7, 7+B)).
template <int SW>
__device__ __forceinline__ uint32_t swizzled_chunk_offset(uint32_t row, uint32_t chunk) {
  constexpr uint32_t kChunks = SW / 16;
  uint32_t x = (SW == 128) ? (row & 7u) : (SW == 64) ? ((row >> 1) & 3u) : ((row >> 2) & 1u);
  return row * SW + (((chunk ^ x) & (kChunks - 1)) << 4);
}

}  // namespace wg

// ---------------------------------------------------------------------------------------------
// host: tensor maps
// ---------------------------------------------------------------------------------------------
// 3-D map over a [rows, heads, d] bf16/fp16 tensor with arbitrary row / head strides (elements): dims (d, heads, rows),
// box (box_cols, 1, box_rows), swizzle = box_cols * 2 bytes (32/64/128).  Returns 0 on success.
int make_tmap_rows_heads(CUtensorMap* out, const void* base, long long rows, int heads, int d, long long row_stride,
                         long long head_stride, int box_cols, int box_rows);

}  // namespace hstu
