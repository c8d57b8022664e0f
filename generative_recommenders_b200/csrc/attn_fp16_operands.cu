// Pre-pass of the bf16 d = 32 wgmma attention: per (sequence, head) amax of the operands and their exactly scaled fp16
// copies (attn_fp16_operands.cuh, DESIGN.md 3.0).  Two kernels on the caller's stream, before the attention kernels:
//   fp16_operands_amax_kernel     atomicMax of the bits of |x| (order-independent, so the result is bitwise reproducible)
//   fp16_operands_convert_kernel  x * 2^e as fp16 into the workspace, [L, H, 32] per operand
// Both run one CTA per (256-row block, head, sequence) over the rows < max_seq_len of each sequence.  Rows of the copies
// past max_seq_len are not written: the attention kernels treat them as rows past the sequence end, which never reach an
// MMA (zero_tile_rows, DESIGN.md 2).
// The forward's workspace, [B, H, 4] amax bits then the q, k, v copies, is also the layout of the operands buffer that
// hstu_attn_fwd_keep_fp16_operands leaves to the caller.  hstu_attn_bwd_on_fp16_operands reads q, k, v and their amax from
// that buffer and runs both kernels over dO alone, into its own workspace: the amax block copied from the buffer (its dO
// slots are zero there), then the dO copy.  Its q, k, v exponents are then the forward's, and so are the bits of the copies.
// The fp8 forward (attn_wgmma_fwd_e4m3.cu) reuses the convert kernel to widen its e4m3 v to fp16, [L, H, dv]: every finite
// e4m3 value is a normal fp16 value, so that copy is exact and needs no scale (and no amax pass).
#include <cuda_fp16.h>
#include <cuda_fp8.h>
#include <string.h>

#include "attn_fp16_operands.cuh"
#include "common.cuh"
#include "internal.h"

namespace hstu {

constexpr int kPreRows = 256, kPreThreads = 256, kPreD = 32;

struct PreOperand {
  const void* src;      // bf16 [L, H, 32] view (e4m3 [L, H, d] for the fp8 forward's v)
  long long row_stride, head_stride;
  __half* dst;          // fp16 [L, H, 32], contiguous
};

struct PreParams {
  PreOperand op[kAmaxSlots];
  int nops;   // 3 (q, k, v), 4 (+ dO), or 1 (dO alone, or the fp8 forward's v)
  int slot0;  // amax slot of op[0]: kAmaxQ, or kAmaxDO for dO alone
  const void* seq_offsets;
  int offsets_i64, max_seq_len, heads;
  int d;  // columns of the e4m3 operand (the bf16 operands have kPreD)
  float alpha;
  uint32_t* amax;  // [B, H, kAmaxSlots], zeroed before the amax kernel
};

__device__ __forceinline__ float bf16_bits_to_float(uint32_t b) { return __uint_as_float(b << 16); }

__global__ void __launch_bounds__(kPreThreads) fp16_operands_amax_kernel(const __grid_constant__ PreParams p) {
  const int b = blockIdx.z, h = blockIdx.y;
  const long long row0 = load_index(p.seq_offsets, p.offsets_i64, b);
  const int len = min((int)(load_index(p.seq_offsets, p.offsets_i64, b + 1) - row0), p.max_seq_len);
  const int r0 = blockIdx.x * kPreRows;
  if (r0 >= len) return;
  const int rows = min(kPreRows, len - r0);
  __shared__ uint32_t red[kAmaxSlots][kPreThreads / 32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int o = 0; o < p.nops; ++o) {
    const PreOperand& op = p.op[o];
    uint32_t m = 0u;
    // 4 threads per row, 8 elements (16 bytes) each
    for (int c = threadIdx.x; c < rows * 4; c += kPreThreads) {
      const int r = c >> 2, part = c & 3;
      const uint4 x = *reinterpret_cast<const uint4*>(reinterpret_cast<const uint16_t*>(op.src) + (row0 + r0 + r) * op.row_stride +
                                                      (long long)h * op.head_stride + part * 8);
      const uint32_t w[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        // |x| as fp32 bits: the bf16 bits without the sign, shifted up (NaN sorts above Inf, Inf above every finite value)
        m = max(m, (w[i] & 0x7fffu) << 16);
        m = max(m, (w[i] >> 16 & 0x7fffu) << 16);
      }
    }
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, s));
    if (lane == 0) red[o][warp] = m;
  }
  __syncthreads();
  if (threadIdx.x < p.nops) {
    uint32_t m = 0u;
#pragma unroll
    for (int w = 0; w < kPreThreads / 32; ++w) m = max(m, red[threadIdx.x][w]);
    if (m) atomicMax(p.amax + ((long long)b * p.heads + h) * kAmaxSlots + p.slot0 + threadIdx.x, m);
  }
}

// E4M3 = false: the scaled fp16 copies of the bf16 d = 32 operands.  E4M3 = true: the exact fp16 copy of an e4m3 operand of
// p.d columns (no scale), [L, H, p.d]
template <bool E4M3>
__global__ void __launch_bounds__(kPreThreads) fp16_operands_convert_kernel(const __grid_constant__ PreParams p) {
  const int b = blockIdx.z, h = blockIdx.y;
  const long long row0 = load_index(p.seq_offsets, p.offsets_i64, b);
  const int len = min((int)(load_index(p.seq_offsets, p.offsets_i64, b + 1) - row0), p.max_seq_len);
  const int r0 = blockIdx.x * kPreRows;
  if (r0 >= len) return;
  const int rows = min(kPreRows, len - r0);
  const int d = E4M3 ? p.d : kPreD, cpr = d / 8;  // columns; chunks of 8 elements per row
  int exps[kAmaxSlots] = {0, 0, 0, 0};
  if constexpr (!E4M3) {
    const OperandExps ex = operand_exps(p.amax + ((long long)b * p.heads + h) * kAmaxSlots, p.alpha, kPreD);
    exps[0] = ex.q, exps[1] = ex.k, exps[2] = ex.v, exps[3] = ex.o;
  }
  for (int o = 0; o < p.nops; ++o) {
    const PreOperand& op = p.op[o];
    const int e = exps[p.slot0 + o];
    for (int c = threadIdx.x; c < rows * cpr; c += kPreThreads) {
      const int r = c / cpr, part = c % cpr;
      const long long row = row0 + r0 + r;
      uint32_t y[4];
      if constexpr (E4M3) {
        const uint2 x = *reinterpret_cast<const uint2*>(reinterpret_cast<const uint8_t*>(op.src) + row * op.row_stride +
                                                        (long long)h * op.head_stride + part * 8);
        const uint32_t w[2] = {x.x, x.y};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          // exact: e4m3 -> fp16 (NaN stays NaN)
          const __half2_raw v = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)(w[i >> 1] >> (16 * (i & 1))), __NV_E4M3);
          y[i] = (uint32_t)v.x | ((uint32_t)v.y << 16);
        }
      } else {
        const uint4 x = *reinterpret_cast<const uint4*>(reinterpret_cast<const uint16_t*>(op.src) + row * op.row_stride +
                                                        (long long)h * op.head_stride + part * 8);
        const uint32_t w[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          // exact: a power-of-two scale of an 8-bit significand into fp16's range (scalbnf is exact wherever the result is)
          const __half2 v = __floats2half2_rn(scalbnf(bf16_bits_to_float(w[i] & 0xffffu), e), scalbnf(bf16_bits_to_float(w[i] >> 16), e));
          y[i] = *reinterpret_cast<const uint32_t*>(&v);
        }
      }
      *reinterpret_cast<uint4*>(op.dst + (row * p.heads + h) * d + part * 8) = make_uint4(y[0], y[1], y[2], y[3]);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// host
// ------------------------------------------------------------------------------------------------
static size_t align256(size_t n) { return (n + 255) / 256 * 256; }
static size_t amax_bytes(const hstu_attn_params& p) { return (size_t)p.batch * p.heads * kAmaxSlots * sizeof(uint32_t); }
static size_t copy_bytes(const hstu_attn_params& p) { return align256((size_t)p.total_rows * p.heads * kPreD * sizeof(__half)); }

size_t fp16_operands_workspace_bytes(const hstu_attn_params& p, bool bwd) {
  return align256(amax_bytes(p)) + (bwd ? 4 : 3) * copy_bytes(p);
}

size_t fp16_operands_dout_workspace_bytes(const hstu_attn_params& p) { return align256(amax_bytes(p)) + copy_bytes(p); }

Fp16Operands fp16_operands_at(const hstu_attn_params& p, void* buf) {
  uint8_t* base = reinterpret_cast<uint8_t*>(buf);
  Fp16Operands f;
  f.amax = reinterpret_cast<uint32_t*>(base);
  for (int o = 0; o < kAmaxSlots; ++o) f.copy[o] = base + align256(amax_bytes(p)) + o * copy_bytes(p);
  return f;
}

// Both kernels over pp.op[0 .. pp.nops), into pp.amax (zeroed, or holding the amax of the other operands) and pp.op[].dst
static int launch_prepass(const hstu_attn_params& p, PreParams& pp, cudaStream_t st) {
  pp.seq_offsets = p.seq_offsets;
  pp.offsets_i64 = p.offsets_are_i64;
  pp.max_seq_len = p.max_seq_len;
  pp.heads = p.heads;
  pp.alpha = p.alpha;
  if (p.batch == 0 || p.max_seq_len <= 0) return 0;
  const dim3 grid((p.max_seq_len + kPreRows - 1) / kPreRows, p.heads, p.batch);
  fp16_operands_amax_kernel<<<grid, kPreThreads, 0, st>>>(pp);
  HSTU_CUDA_OK(cudaGetLastError());
  fp16_operands_convert_kernel<false><<<grid, kPreThreads, 0, st>>>(pp);
  HSTU_CUDA_OK(cudaGetLastError());
  return 0;
}

int fp16_operands_prepass(const hstu_attn_params& p, bool bwd, Fp16Operands* out, cudaStream_t st) {
  const size_t need = fp16_operands_workspace_bytes(p, bwd);
  if (p.workspace == nullptr || p.workspace_bytes < need) {
    set_error("hstu_attn_%s: workspace of %zu bytes required (got %zu)", bwd ? "bwd" : "fwd", need, p.workspace_bytes);
    return HSTU_ERR_WORKSPACE;
  }
  *out = fp16_operands_at(p, p.workspace);
  PreParams pp;
  memset(&pp, 0, sizeof(pp));
  pp.amax = const_cast<uint32_t*>(out->amax);
  const void* src[kAmaxSlots] = {p.q, p.k, p.v, p.dout};
  const long long rs[kAmaxSlots] = {p.q_row_stride, p.k_row_stride, p.v_row_stride, p.do_row_stride};
  const long long hs[kAmaxSlots] = {p.q_head_stride, p.k_head_stride, p.v_head_stride, p.do_head_stride};
  pp.nops = bwd ? 4 : 3;
  for (int o = 0; o < pp.nops; ++o) {
    pp.op[o].src = src[o];
    pp.op[o].row_stride = rs[o];
    pp.op[o].head_stride = hs[o];
    pp.op[o].dst = reinterpret_cast<__half*>(const_cast<void*>(out->copy[o]));
  }
  HSTU_CUDA_OK(cudaMemsetAsync(pp.amax, 0, amax_bytes(p), st));
  return launch_prepass(p, pp, st);
}

int fp16_operands_dout_prepass(const hstu_attn_params& p, const void* kept, Fp16Operands* out, cudaStream_t st) {
  const size_t need = fp16_operands_dout_workspace_bytes(p);
  if (p.workspace == nullptr || p.workspace_bytes < need) {
    set_error("hstu_attn_bwd_on_fp16_operands: workspace of %zu bytes required (got %zu)", need, p.workspace_bytes);
    return HSTU_ERR_WORKSPACE;
  }
  const Fp16Operands k = fp16_operands_at(p, const_cast<void*>(kept)), w = fp16_operands_at(p, p.workspace);
  out->amax = w.amax;
  for (int o = 0; o < 3; ++o) out->copy[o] = k.copy[o];
  out->copy[kAmaxDO] = w.copy[0];  // the only copy of the workspace
  PreParams pp;
  memset(&pp, 0, sizeof(pp));
  pp.amax = const_cast<uint32_t*>(w.amax);
  pp.nops = 1;
  pp.slot0 = kAmaxDO;
  pp.op[0].src = p.dout;
  pp.op[0].row_stride = p.do_row_stride;
  pp.op[0].head_stride = p.do_head_stride;
  pp.op[0].dst = reinterpret_cast<__half*>(const_cast<void*>(w.copy[0]));
  HSTU_CUDA_OK(cudaMemcpyAsync(pp.amax, k.amax, amax_bytes(p), cudaMemcpyDeviceToDevice, st));
  return launch_prepass(p, pp, st);
}

size_t e4m3_v_copy_bytes(const hstu_attn_params& p) { return align256((size_t)p.total_rows * p.heads * p.dv * sizeof(__half)); }

int e4m3_v_prepass(const hstu_attn_params& p, const void** v16, cudaStream_t st) {
  const size_t need = e4m3_v_copy_bytes(p);
  if (p.workspace == nullptr || p.workspace_bytes < need) {
    set_error("hstu_attn_fwd_fp8: workspace of %zu bytes required (got %zu)", need, p.workspace_bytes);
    return HSTU_ERR_WORKSPACE;
  }
  PreParams pp;
  memset(&pp, 0, sizeof(pp));
  pp.nops = 1;
  pp.op[0].src = p.v;
  pp.op[0].row_stride = p.v_row_stride;
  pp.op[0].head_stride = p.v_head_stride;
  pp.op[0].dst = reinterpret_cast<__half*>(p.workspace);
  *v16 = p.workspace;
  pp.seq_offsets = p.seq_offsets;
  pp.offsets_i64 = p.offsets_are_i64;
  pp.max_seq_len = p.max_seq_len;
  pp.heads = p.heads;
  pp.d = p.dv;
  if (p.batch == 0 || p.max_seq_len <= 0) return 0;
  const dim3 grid((p.max_seq_len + kPreRows - 1) / kPreRows, p.heads, p.batch);
  fp16_operands_convert_kernel<true><<<grid, kPreThreads, 0, st>>>(pp);
  HSTU_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace hstu
