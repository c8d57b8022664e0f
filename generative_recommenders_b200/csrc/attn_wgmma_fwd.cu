// Jagged HSTU attention forward on the wgmma kernels at dqk == dv in {32, 64, 128, 256} (bf16 / fp16), the delta-q reduction,
// which calls the wgmma kernels take (causal and non-causal), and the routing of every causal wgmma forward.  The kernel body, its design and its launcher are in attn_wgmma_fwd.cuh; the
// dqk < dv instantiations are in attn_wgmma_mixed_fwd.cu.
#include "attn_wgmma_fwd.cuh"

namespace hstu {

template <int D, bool BF16>
__global__ void __launch_bounds__(kAttnThreads, kFwdMinBlocks<D>) attn_fwd_wgmma_kernel(const __grid_constant__ FwdParams p) {
  attn_fwd_wgmma_body<D, D, BF16, false>(p);
}
template <int D, bool BF16>
__global__ void __launch_bounds__(kAttnThreads, kFwdMinBlocks<D>) attn_fwd_delta_wgmma_kernel(const __grid_constant__ FwdParams p) {
  attn_fwd_wgmma_body<D, D, BF16, true>(p);
}

// Split delta-q: out = (sum of the chunks' fp32 partials [chunks, rows, H, d], in chunk order) * 1/N, 4 columns per thread.
template <bool BF16>
__global__ void __launch_bounds__(256) delta_reduce_kernel(const float* __restrict__ part, void* out, long long rows, int heads, int d,
                                                            int chunks, long long o_row_stride, long long o_head_stride, float inv_n) {
  const long long plane = rows * heads * d, n4 = plane / 4;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n4; i += (long long)gridDim.x * 256) {
    float4 a = reinterpret_cast<const float4*>(part)[i];
    for (int c = 1; c < chunks; ++c) {
      const float4 x = reinterpret_cast<const float4*>(part + c * plane)[i];
      a.x += x.x, a.y += x.y, a.z += x.z, a.w += x.w;
    }
    const long long e = i * 4, r = e / ((long long)heads * d), hc = e % ((long long)heads * d);
    const long long off = r * o_row_stride + (hc / d) * o_head_stride + hc % d;
    a.x *= inv_n, a.y *= inv_n, a.z *= inv_n, a.w *= inv_n;
    const uint2 v = BF16 ? make_uint2(pack_bf16x2(a.x, a.y), pack_bf16x2(a.z, a.w)) : make_uint2(pack_f16x2(a.x, a.y), pack_f16x2(a.z, a.w));
    *reinterpret_cast<uint2*>(reinterpret_cast<uint16_t*>(out) + off) = v;
  }
}

// ------------------------------------------------------------------------------------------------
// host
// ------------------------------------------------------------------------------------------------
// Key chunks of a delta-q call, from sizes only (no device query, no read of seq_offsets).  The CTAs of one chunk are
// B * H * ceil(delta / 128); the keys are split only while those fill fewer than kDeltaCtaTarget CTAs (two per SM of a 132-SM
// H100), into at most kDeltaCtaTarget / CTAs chunks and at most ceil(N / kDeltaChunkKeys), so that no chunk of a full-length
// sequence is shorter than 8 key tiles.  chunks * CTAs <= kDeltaCtaTarget bounds the workspace of the partials by
// kDeltaCtaTarget * 128 rows * dv * 4 bytes: 34.6 MB at dv = 256, 4.3 MB at dv = 32.
// The sizing constants assume the 132 SMs of an H100 SXM (kH100Sms); on another part they only shift the balance, never the result.
constexpr int kDeltaCtaTarget = 2 * kH100Sms, kDeltaChunkKeys = 512;
constexpr int kDeltaReduceBlocks = 8 * kH100Sms;  // grid cap of delta_reduce_kernel (grid-strided: any grid is correct)
int delta_chunks(const hstu_attn_params& p) {
  const long long ctas = (long long)p.batch * p.heads * ((p.delta_q_len + FwdCfg<32>::BM - 1) / FwdCfg<32>::BM);
  if (ctas >= kDeltaCtaTarget) return 1;
  const long long by_len = ((long long)p.max_seq_len + kDeltaChunkKeys - 1) / kDeltaChunkKeys;
  return (int)std::max(1ll, std::min(by_len, kDeltaCtaTarget / ctas));
}

size_t wgmma_delta_workspace_bytes(const hstu_attn_params& p) {
  const int c = delta_chunks(p);
  return c > 1 ? (size_t)c * p.batch * p.delta_q_len * p.heads * p.dv * sizeof(float) : 0;
}

bool is_sm90() {
  static int cached = -1;
  if (cached < 0) {
    int dev = 0;
    cudaDeviceProp prop;
    cached = (cudaGetDevice(&dev) == cudaSuccess && cudaGetDeviceProperties(&prop, dev) == cudaSuccess && prop.major == 9) ? 1 : 0;
  }
  return cached == 1;
}

bool aligned_view(const void* ptr, long long row_stride, long long head_stride) {
  return (reinterpret_cast<uintptr_t>(ptr) & 15) == 0 && (row_stride % 8) == 0 && (head_stride % 8) == 0;
}

// What the wgmma kernels need of a call in either direction: a 16-bit dtype, the head dims, no relative bias, the row limits,
// aligned q, k, v views, and an sm_90 device
static bool wgmma_qkv_supported(const hstu_attn_params& p) {
  if (p.dtype != HSTU_BF16 && p.dtype != HSTU_F16) return false;
  if (!wgmma_dims(p.dqk, p.dv)) return false;
  if (p.delta_q_len < 0 || p.pos_w != nullptr || p.ts_w != nullptr) return false;
  if (p.total_rows >= (1ll << 31) - 256 || (long long)p.batch * p.delta_q_len >= (1ll << 31) - 256) return false;
  if (!aligned_view(p.q, p.q_row_stride, p.q_head_stride) || !aligned_view(p.k, p.k_row_stride, p.k_head_stride) ||
      !aligned_view(p.v, p.v_row_stride, p.v_head_stride))
    return false;
  return is_sm90();
}

static bool wgmma_fwd_supported(const hstu_attn_params& p) {
  return wgmma_qkv_supported(p) && aligned_view(p.out, p.o_row_stride, p.o_head_stride);
}

// The backward does not read out; a given one still needs a 16-byte aligned base
static bool wgmma_bwd_supported(const hstu_attn_params& p) {
  if (!wgmma_qkv_supported(p) || (p.out != nullptr && !aligned_view(p.out, 0, 0))) return false;
  // d = 256 and dqk < dv run the split kernels only; a deterministic backward there stays on the generic kernels
  if ((p.dqk == 256 || p.dqk != p.dv) && p.deterministic) return false;
  return aligned_view(p.dout, p.do_row_stride, p.do_head_stride) && aligned_view(p.dq, p.dq_row_stride, p.dq_head_stride) &&
         aligned_view(p.dk, p.dk_row_stride, p.dk_head_stride) && aligned_view(p.dv_out, p.dv_row_stride, p.dv_head_stride);
}

bool wgmma_supported(const hstu_attn_params& p, bool bwd, bool bidir) {
  if (bidir && (p.delta_q_len != 0 || !has_dims(BidirDims{}, p.dqk, p.dv))) return false;
  return bwd ? wgmma_bwd_supported(p) : wgmma_fwd_supported(p);
}

int launch_delta_reduce(bool bf16, const float* part, void* out, long long rows, int heads, int d, int chunks,
                        long long o_row_stride, long long o_head_stride, float inv_n, cudaStream_t st) {
  const long long n4 = rows * heads * d / 4;
  const int blocks = (int)std::min<long long>((n4 + 255) / 256, kDeltaReduceBlocks);
  auto kern = bf16 ? delta_reduce_kernel<true> : delta_reduce_kernel<false>;
  kern<<<blocks, 256, 0, st>>>(part, out, rows, heads, d, chunks, o_row_stride, o_head_stride, inv_n);
  HSTU_CUDA_OK(cudaGetLastError());
  return 0;
}

int attn_wgmma_fwd(const hstu_attn_params& p, cudaStream_t st) {
  if (p.dqk != p.dv) return attn_wgmma_fwd_mixed(p, st);
  return dispatch_dims(SquareDims{}, p, "wgmma forward", [&]<int D, int, bool BF16>() {
    // bf16 keeps the hi / lo P at d = 32 too: a pre-pass over the whole cache would cost more than it saves
    if (p.delta_q_len > 0) return launch_fwd_wgmma<D, D, BF16, true>(p, st, attn_fwd_delta_wgmma_kernel<D, BF16>);
    return launch_on_operands<D, BF16>(p, false, st, [&]<bool B>(const Fp16Operands* f16) {
      return launch_fwd_wgmma<D, D, B, false>(p, st, attn_fwd_wgmma_kernel<D, B>, f16);
    });
  });
}

}  // namespace hstu
