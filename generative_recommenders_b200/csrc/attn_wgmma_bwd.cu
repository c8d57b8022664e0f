// Jagged HSTU attention backward on the wgmma kernels at dqk == dv in {32, 64, 128, 256} (bf16 / fp16): the fused key-tile
// kernel with its dQ convert, the split dK / dV and dQ kernels, and the routing of every wgmma backward.  The kernel bodies,
// their design and the split launcher are in attn_wgmma_bwd.cuh; the dqk < dv instantiations are in attn_wgmma_mixed_bwd.cu.
#include "attn_wgmma_bwd.cuh"

namespace hstu {

template <int D, bool BF16>
__global__ void __launch_bounds__(kAttnThreads, 1) attn_bwd_wgmma_kernel(const __grid_constant__ BwdParams p) {
  bwd_key_tile<D, D, BF16, true>(p);
}

// d = 32: two CTAs per SM (<= 128 registers per thread, 49 KB of shared memory); d = 256: one 128-column half per CTA
template <int D, bool BF16>
__global__ void __launch_bounds__(kAttnThreads, split_min_blocks(D)) attn_bwd_dkdv_wgmma_kernel(const __grid_constant__ BwdParams p) {
  bwd_key_tile<D, D, BF16, false>(p);
}

template <int D, bool BF16>
__global__ void __launch_bounds__(kAttnThreads, split_min_blocks(D)) attn_bwd_dq_wgmma_kernel(const __grid_constant__ BwdParams p) {
  bwd_dq_body<D, D, BF16>(p);
}

// dq[r, h, :] = convert(dq_acc[r, h, :] * scale)
template <bool BF16>
__global__ void dq_convert_kernel(const float* __restrict__ acc, uint16_t* __restrict__ dq, long long rows, int heads, int D,
                                  long long row_stride, long long head_stride, float scale) {
  const long long nvec = rows * heads * (D / 8);
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < nvec; idx += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(idx % (D / 8));
    const long long rh = idx / (D / 8);
    const int hh = (int)(rh % heads);
    const long long r = rh / heads;
    const float4 a = *reinterpret_cast<const float4*>(acc + rh * D + v * 8);
    const float4 c = *reinterpret_cast<const float4*>(acc + rh * D + v * 8 + 4);
    uint4 o;
    if (BF16) {
      o = make_uint4(pack_bf16x2(a.x * scale, a.y * scale), pack_bf16x2(a.z * scale, a.w * scale),
                     pack_bf16x2(c.x * scale, c.y * scale), pack_bf16x2(c.z * scale, c.w * scale));
    } else {
      o = make_uint4(pack_f16x2(a.x * scale, a.y * scale), pack_f16x2(a.z * scale, a.w * scale),
                     pack_f16x2(c.x * scale, c.y * scale), pack_f16x2(c.z * scale, c.w * scale));
    }
    *reinterpret_cast<uint4*>(dq + r * row_stride + hh * head_stride + v * 8) = o;
  }
}

// ------------------------------------------------------------------------------------------------
// host
// ------------------------------------------------------------------------------------------------
static bool wgmma_bwd_supported(const hstu_attn_params& p) {
  if (!wgmma_fwd_supported(p)) return false;  // dtype / dims / alignment of q, k, v (out is not used by the backward)
  // d = 256 and dqk < dv run the split kernels only; a deterministic backward there stays on the generic kernels
  if ((p.dqk == 256 || p.dqk != p.dv) && p.deterministic) return false;
  return aligned_view(p.dout, p.do_row_stride, p.do_head_stride) && aligned_view(p.dq, p.dq_row_stride, p.dq_head_stride) &&
         aligned_view(p.dk, p.dk_row_stride, p.dk_head_stride) && aligned_view(p.dv_out, p.dv_row_stride, p.dv_head_stride);
}

bool wgmma_supported(const hstu_attn_params& p, bool bwd) {
  if (!bwd) return wgmma_fwd_supported(p);
  hstu_attn_params q = p;
  if (q.out == nullptr) q.out = const_cast<void*>(q.q);  // the forward check also looks at `out`
  q.o_row_stride = 8;
  q.o_head_stride = 8;
  return wgmma_bwd_supported(q);
}

// d = 32 / 256, dqk < dv, or a deterministic backward: dK / dV and dQ in two kernels, without atomics or dQ workspace;
// otherwise the fused kernel (DESIGN.md 3.2).  At d = 256 the fused kernel's fp32 dQ accumulator would be L * H * 1 KB.
static bool split_dq(const hstu_attn_params& p) {
  return p.dqk == 32 || p.dqk == 256 || p.dqk != p.dv || p.deterministic != 0;
}

// bf16 at dqk == dv == 32: the fp16 kernels on exactly scaled copies (attn_fp16_operands.cu)
static bool fp16_copies(const hstu_attn_params& p) { return p.dtype == HSTU_BF16 && p.dqk == 32 && p.dv == 32; }

size_t wgmma_workspace_bytes(const hstu_attn_params& p, bool bwd) {
  if (!bwd && p.delta_q_len > 0) return wgmma_delta_workspace_bytes(p);  // the fp32 partials of split key chunks, or 0
  if (fp16_copies(p)) return fp16_operands_workspace_bytes(p, bwd);
  if (!bwd || split_dq(p)) return 0;
  return (size_t)p.total_rows * p.heads * p.dqk * sizeof(float);  // fp32 dQ accumulator [L, H, D]
}

// kSplit: the dK / dV and dQ kernels, else the fused kernel and the dQ convert.  f16: the scaled fp16 copies of bf16 inputs
// (the kernels are then the fp16 ones), or null
template <int D, bool BF16, bool kSplit>
static int launch_bwd_wgmma(const hstu_attn_params& p, cudaStream_t st, const Fp16Operands* f16 = nullptr) {
  if constexpr (kSplit) {
    return launch_bwd_split<D, D, BF16>(p, st, attn_bwd_dkdv_wgmma_kernel<D, BF16>, attn_bwd_dq_wgmma_kernel<D, BF16>, f16);
  } else {
    using Cfg = BwdCfg<D, D, true>;
    const size_t need = wgmma_workspace_bytes(p, true);
    if (p.workspace == nullptr || p.workspace_bytes < need) {
      set_error("hstu_attn_bwd: workspace of %zu bytes required (got %zu)", need, p.workspace_bytes);
      return HSTU_ERR_WORKSPACE;
    }
    const BwdOperands o = bwd_operands(p, f16);
    BwdParams bp = bwd_params(p, f16);
    if (int e = make_tmap_rows_heads(&bp.tmQ, o.src[0], p.total_rows, p.heads, D, o.rs[0], o.hs[0], Cfg::BOX_COLS, Cfg::BQ)) return e;
    if (int e = make_tmap_rows_heads(&bp.tmK, o.src[1], p.total_rows, p.heads, D, o.rs[1], o.hs[1], Cfg::BOX_COLS, Cfg::BKV)) return e;
    if (int e = make_tmap_rows_heads(&bp.tmV, o.src[2], p.total_rows, p.heads, D, o.rs[2], o.hs[2], Cfg::BOX_COLS, Cfg::BKV)) return e;
    if (int e = make_tmap_rows_heads(&bp.tmDO, o.src[3], p.total_rows, p.heads, D, o.rs[3], o.hs[3], Cfg::BOX_COLS, Cfg::BQ)) return e;
    HSTU_CUDA_OK(cudaMemsetAsync(p.workspace, 0, need, st));
    auto kern = attn_bwd_wgmma_kernel<D, BF16>;
    HSTU_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    dim3 grid((p.max_seq_len + Cfg::BKV - 1) / Cfg::BKV, p.heads, p.batch);
    kern<<<grid, kAttnThreads, Cfg::SMEM_BYTES, st>>>(bp);
    HSTU_CUDA_OK(cudaGetLastError());
    const long long nvec = p.total_rows * p.heads * (D / 8);
    long long blocks = (nvec + 255) / 256;
    if (blocks > 132 * 16) blocks = 132 * 16;
    dq_convert_kernel<BF16><<<(int)blocks, 256, 0, st>>>(bp.dq_acc, reinterpret_cast<uint16_t*>(p.dq), p.total_rows, p.heads, D,
                                                         p.dq_row_stride, p.dq_head_stride, bp.dk_scale);
    HSTU_CUDA_OK(cudaGetLastError());
    return 0;
  }
}

int attn_wgmma_bwd(const hstu_attn_params& p, cudaStream_t st) {
  if (p.dqk != p.dv) return attn_wgmma_bwd_mixed(p, st);  // split kernels only
  const bool bf = p.dtype == HSTU_BF16;
  const bool split = split_dq(p);
  switch (p.dqk) {
    case 32: {  // bf16: the fp16 kernels on exactly scaled copies (DESIGN.md 3.0)
      if (!bf) return launch_bwd_wgmma<32, false, true>(p, st);
      Fp16Operands f16;
      if (int e = fp16_operands_prepass(p, true, &f16, st)) return e;
      return launch_bwd_wgmma<32, false, true>(p, st, &f16);
    }
    case 64:
      if (split) return bf ? launch_bwd_wgmma<64, true, true>(p, st) : launch_bwd_wgmma<64, false, true>(p, st);
      return bf ? launch_bwd_wgmma<64, true, false>(p, st) : launch_bwd_wgmma<64, false, false>(p, st);
    case 128:
      if (split) return bf ? launch_bwd_wgmma<128, true, true>(p, st) : launch_bwd_wgmma<128, false, true>(p, st);
      return bf ? launch_bwd_wgmma<128, true, false>(p, st) : launch_bwd_wgmma<128, false, false>(p, st);
    case 256:  // split only (split_dq)
      return bf ? launch_bwd_wgmma<256, true, true>(p, st) : launch_bwd_wgmma<256, false, true>(p, st);
  }
  set_error("wgmma backward: unsupported head dim %d", p.dqk);
  return HSTU_ERR_UNSUPPORTED;
}

int attn_wgmma_bwd_on_fp16_operands(const hstu_attn_params& p, const void* kept, cudaStream_t st) {
  Fp16Operands f16;
  if (int e = fp16_operands_dout_prepass(p, kept, &f16, st)) return e;
  return launch_bwd_wgmma<32, false, true>(p, st, &f16);
}

}  // namespace hstu
