// Jagged HSTU attention backward on the wgmma kernels at dqk == dv in {32, 64, 128, 256} (bf16 / fp16): the fused key-tile
// kernel with its dQ convert, the split dK / dV and dQ kernels, and the routing of every wgmma backward.  The kernel bodies,
// their design and the launchers are in attn_wgmma_bwd.cuh; the dqk < dv instantiations are in attn_wgmma_mixed_bwd.cu.
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
// bidir: the non-causal kernels take no delta-q, and their backward is always split
size_t wgmma_workspace_bytes(const hstu_attn_params& p, bool bwd, bool bidir) {
  if (!bwd && p.delta_q_len > 0) return wgmma_delta_workspace_bytes(p);  // the fp32 partials of split key chunks, or 0
  if (runs_on_fp16_operands(p)) return fp16_operands_workspace_bytes(p, bwd);
  if (!bwd || bidir || split_dq(p)) return 0;
  return (size_t)p.total_rows * p.heads * p.dqk * sizeof(float);  // fp32 dQ accumulator [L, H, D]
}

int attn_wgmma_bwd(const hstu_attn_params& p, cudaStream_t st) {
  if (p.dqk != p.dv) return attn_wgmma_bwd_mixed(p, st);  // split kernels only
  return dispatch_dims(SquareDims{}, p, "wgmma backward", [&]<int D, int, bool BF16>() {
    return launch_on_operands<D, BF16>(p, true, st, [&]<bool B>(const Fp16Operands* f16) {
      if constexpr (fused_bwd_dims(D, D))
        if (!split_dq(p)) return launch_bwd_fused<D>(p, st, attn_bwd_wgmma_kernel<D, B>, dq_convert_kernel<B>);
      return launch_bwd_split<D, D, B>(p, st, attn_bwd_dkdv_wgmma_kernel<D, B>, attn_bwd_dq_wgmma_kernel<D, B>, f16);
    });
  });
}

int attn_wgmma_bwd_on_fp16_operands(const hstu_attn_params& p, const void* kept, cudaStream_t st) {
  Fp16Operands f16;
  if (int e = fp16_operands_dout_prepass(p, kept, &f16, st)) return e;
  return launch_bwd_split<32, 32, false>(p, st, attn_bwd_dkdv_wgmma_kernel<32, false>, attn_bwd_dq_wgmma_kernel<32, false>, &f16);
}

}  // namespace hstu
