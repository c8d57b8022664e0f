// C-ABI entry points of libhstu_b200.so (declared in include/hstu_b200.h): argument validation, error reporting,
// dispatch between the wgmma/TMA kernels and the generic kernels.  No torch / ATen types anywhere.
#include <stdarg.h>
#include <string.h>

#include "common.cuh"
#include "internal.h"

namespace hstu {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

static int validate_attn(const hstu_attn_params* p, bool bwd) {
  HSTU_CHECK_ARG(p != nullptr, "params is NULL");
  HSTU_CHECK_ARG(p->abi_version == HSTU_B200_ABI_VERSION, "ABI version mismatch: caller %d, library %d", p->abi_version,
                 HSTU_B200_ABI_VERSION);
  HSTU_CHECK_ARG(p->dtype == HSTU_F32 || p->dtype == HSTU_BF16 || p->dtype == HSTU_F16 || p->dtype == HSTU_E4M3, "bad dtype %d",
                 p->dtype);
  HSTU_CHECK_ARG(p->max_seq_len > 0, "max_seq_len must be larger than 0");  // ops/hstu_attention.py:64
  HSTU_CHECK_ARG(p->batch >= 0 && p->heads > 0, "bad batch/heads");
  HSTU_CHECK_ARG(p->dqk > 0 && p->dv > 0 && p->dqk <= 256 && p->dv <= 256, "head dims must be in [1, 256] (dqk=%d, dv=%d)",
                 p->dqk, p->dv);
  HSTU_CHECK_ARG(p->total_rows >= 0, "negative total_rows");
  HSTU_CHECK_ARG(p->max_attn_len >= 0 && p->contextual_seq_len >= 0 && p->min_full_attn_seq_len >= 0, "negative mask option");
  if (p->batch == 0 || p->total_rows == 0) return 0;
  HSTU_CHECK_ARG(p->seq_offsets != nullptr, "seq_offsets is NULL");
  HSTU_CHECK_ARG(p->q && p->k && p->v, "q/k/v is NULL");
  if (!bwd) HSTU_CHECK_ARG(p->out != nullptr, "out is NULL");
  if (bwd) {
    HSTU_CHECK_ARG(p->dout && p->dq && p->dk && p->dv_out, "dout/dq/dk/dv is NULL");
    HSTU_CHECK_ARG(p->delta_q_len == 0, "backward of delta-q attention is not defined by the reference");
  }
  if (p->ts_w) HSTU_CHECK_ARG(p->timestamps != nullptr, "ts_w given without timestamps");
  HSTU_CHECK_ARG(p->impl >= HSTU_IMPL_AUTO && p->impl <= HSTU_IMPL_UMMA, "bad impl %d", p->impl);
  HSTU_CHECK_ARG(p->deterministic == 0 || p->deterministic == 1, "deterministic must be 0 or 1 (got %d)", p->deterministic);
  return 0;
}

// Make the device that owns `ptr` current on the calling thread.  The caller may be a thread that has never touched
// CUDA (e.g. the autograd engine thread): kernels must go to the device of the data, and driver-API calls such as
// cuTensorMapEncodeTiled need a current context.
int bind_device(const void* ptr) {
  if (ptr == nullptr) return 0;  // empty tensor: nothing will be launched
  cudaPointerAttributes attr;
  cudaError_t e = cudaPointerGetAttributes(&attr, ptr);
  if (e != cudaSuccess || (attr.type != cudaMemoryTypeDevice && attr.type != cudaMemoryTypeManaged)) {
    cudaGetLastError();
    set_error("expected a CUDA device pointer (got %p: %s)", ptr, e == cudaSuccess ? "host memory" : cudaGetErrorString(e));
    return HSTU_ERR_INVALID_ARGUMENT;
  }
  HSTU_CUDA_OK(cudaSetDevice(attr.device));
  return 0;
}

// Which kernels take a call: HSTU_IMPL_UMMA (the wgmma kernels), HSTU_IMPL_GENERIC, or a refusal.  bidir: the non-causal
// mask, whose kernels take no delta-q, relative bias or e4m3 input (the reference's KV-cached path is causal, and there is no
// fp8 backward).  A deterministic backward takes the same route as any other: the wgmma kernels run their atomic-free split
// path (attn_wgmma_bwd.cu), and the generic kernels have no atomics on q / k / v.
static int select_impl(const hstu_attn_params* p, bool bwd, bool bidir) {
  if (bidir) {
    if (p->delta_q_len > 0) {
      set_error("non-causal attention: delta_q (the KV-cached forward) is causal only");
      return HSTU_ERR_UNSUPPORTED;
    }
    if (p->pos_w != nullptr || p->ts_w != nullptr) {
      set_error("non-causal attention: the relative bias is not supported");
      return HSTU_ERR_UNSUPPORTED;
    }
    if (p->dtype == HSTU_E4M3) {
      set_error("non-causal attention: fp8 (e4m3) inputs are not supported");
      return HSTU_ERR_UNSUPPORTED;
    }
  }
  if (p->dtype == HSTU_E4M3) {  // the fp8 forward: wgmma kernels only, whatever the device (hstu_attn_fwd_fp8 checks it)
    if (bwd) {
      set_error("fp8 (e4m3) attention has no backward: hstu_attn_fwd_fp8 is a forward-only entry");
      return HSTU_ERR_UNSUPPORTED;
    }
    if (p->impl == HSTU_IMPL_GENERIC) {
      set_error("fp8 (e4m3) attention runs on the wgmma kernels only: the generic kernels take no fp8 input");
      return HSTU_ERR_UNSUPPORTED;
    }
    if (int e = e4m3_fwd_check(*p)) return e;
    return HSTU_IMPL_UMMA;
  }
  if (bwd && p->deterministic && (p->pos_w != nullptr || p->ts_w != nullptr)) {
    set_error("deterministic backward with a relative bias is not supported: the dpos_w / dts_w gradients are added "
              "with atomics");
    return HSTU_ERR_UNSUPPORTED;
  }
  const bool can = wgmma_supported(*p, bwd, bidir);
  if (p->impl == HSTU_IMPL_GENERIC) return HSTU_IMPL_GENERIC;
  if (p->impl == HSTU_IMPL_UMMA) {
    if (!can) {
      if (bidir)
        set_error("non-causal wgmma path does not support this problem (dtype=%d dqk=%d dv=%d): it takes bf16 / fp16 at "
                  "dqk == dv in {32, 64, 128}; d = 256, dqk != dv and fp32 run on the generic kernels", p->dtype, p->dqk, p->dv);
      else
        set_error("wgmma path does not support this problem (dtype=%d dqk=%d dv=%d delta=%d bias=%d)", p->dtype, p->dqk,
                  p->dv, p->delta_q_len, p->pos_w != nullptr || p->ts_w != nullptr);
      return HSTU_ERR_UNSUPPORTED;
    }
    return HSTU_IMPL_UMMA;
  }
  return can ? HSTU_IMPL_UMMA : HSTU_IMPL_GENERIC;
}

// The calls that run on scaled fp16 operands (attn_fp16_operands.cu): those of runs_on_fp16_operands on the wgmma kernels
static bool wgmma_on_fp16_operands(const hstu_attn_params* p, bool bwd) {
  return runs_on_fp16_operands(*p) && select_impl(p, bwd, false) == HSTU_IMPL_UMMA;
}

// The bodies of hstu_attn_select_impl, _workspace_bytes, _fwd and _bwd and of their non-causal twins (bidir)
static int checked_select_impl(const hstu_attn_params* p, bool bwd, bool bidir) {
  if (int e = validate_attn(p, bwd)) return e;
  return select_impl(p, bwd, bidir);
}

static size_t workspace_bytes(const hstu_attn_params* p, bool bwd, bool bidir) {
  if (p == nullptr || validate_attn(p, bwd) != 0 || p->batch == 0 || p->total_rows == 0) return 0;
  if (select_impl(p, bwd, bidir) != HSTU_IMPL_UMMA) return 0;
  return p->dtype == HSTU_E4M3 ? e4m3_v_copy_bytes(*p) : wgmma_workspace_bytes(*p, bwd, bidir);  // e4m3: the fp16 copy of v
}

// The causal entries refuse e4m3 themselves, return 0 on an empty problem (triton_hstu_attention.py:1789-1790) and bind the
// device of q before routing; the non-causal ones route first, so their refusals come before all three.
static int run_attn(const hstu_attn_params* p, bool bwd, bool bidir, cudaStream_t st) {
  if (int e = validate_attn(p, bwd)) return e;
  if (!bidir && p->dtype == HSTU_E4M3) {
    if (!bwd) {
      set_error("hstu_attn_fwd: fp8 (e4m3) inputs go through hstu_attn_fwd_fp8 (with their descales)");
      return HSTU_ERR_INVALID_ARGUMENT;
    }
    set_error("hstu_attn_bwd: fp8 (e4m3) attention has no backward (hstu_attn_fwd_fp8 is forward only)");
    return HSTU_ERR_UNSUPPORTED;
  }
  int impl = bidir ? select_impl(p, bwd, true) : 0;
  if (impl < 0) return impl;
  if (p->batch == 0 || p->total_rows == 0) return 0;
  if (int e = bind_device(p->q)) return e;
  if (!bidir) impl = select_impl(p, bwd, false);
  if (impl < 0) return impl;
  if (impl == HSTU_IMPL_GENERIC) return bwd ? attn_generic_bwd(*p, st, bidir) : attn_generic_fwd(*p, st, bidir);
  if (bidir) return bwd ? attn_wgmma_bidir_bwd(*p, st) : attn_wgmma_bidir_fwd(*p, st);
  return bwd ? attn_wgmma_bwd(*p, st) : attn_wgmma_fwd(*p, st);
}

// Nullable descales: no negative strides, fp32-aligned pointers.
static int validate_descales(const hstu_attn_descales* d) {
  if (d == nullptr) return 0;
  const float* ptr[3] = {d->q, d->k, d->v};
  const int64_t bs[3] = {d->q_batch_stride, d->k_batch_stride, d->v_batch_stride};
  const int64_t hs[3] = {d->q_head_stride, d->k_head_stride, d->v_head_stride};
  for (int i = 0; i < 3; ++i) {
    const char name = "qkv"[i];
    HSTU_CHECK_ARG(bs[i] >= 0 && hs[i] >= 0, "%c descale: negative stride (batch %lld, head %lld)", name, (long long)bs[i],
                   (long long)hs[i]);
    HSTU_CHECK_ARG((reinterpret_cast<uintptr_t>(ptr[i]) & 3) == 0, "%c descale: %p is not a float pointer", name, (const void*)ptr[i]);
  }
  return 0;
}

// Every non-null descale is device memory of the device that runs the call (the current one, after bind_device).
static int check_descale_devices(const hstu_attn_descales* d) {
  if (d == nullptr) return 0;
  int dev = 0;
  HSTU_CUDA_OK(cudaGetDevice(&dev));
  const float* ptr[3] = {d->q, d->k, d->v};
  for (int i = 0; i < 3; ++i) {
    if (ptr[i] == nullptr) continue;
    cudaPointerAttributes attr;
    const cudaError_t e = cudaPointerGetAttributes(&attr, ptr[i]);
    if (e != cudaSuccess || (attr.type != cudaMemoryTypeDevice && attr.type != cudaMemoryTypeManaged) || attr.device != dev) {
      cudaGetLastError();
      set_error("%c descale: expected device memory of CUDA device %d (got %p)", "qkv"[i], dev, (const void*)ptr[i]);
      return HSTU_ERR_INVALID_ARGUMENT;
    }
  }
  return 0;
}

// The bodies of the mask exports (hstu_mask_valid, hstu_kv_range_for_q_rows, hstu_q_range_for_kv_rows) and of their
// non-causal twins (bidir)
static int seq_mask_valid(bool bidir, int len, int num_targets, int max_attn_len, int min_full, int ctx, int i, int j) {
  const SeqMask m = make_seq_mask(len, num_targets, max_attn_len, min_full, ctx);
  return (bidir ? mask_valid_bidir(m, i, j) : mask_valid(m, i, j)) ? 1 : 0;
}

static int kv_range(bool bidir, int len, int num_targets, int max_attn_len, int min_full, int ctx, int m0, int m1, int32_t* lo,
                    int32_t* hi) {
  HSTU_CHECK_ARG(lo && hi && m0 >= 0 && m1 > m0 && m1 <= len, "bad row range");
  const SeqMask m = make_seq_mask(len, num_targets, max_attn_len, min_full, ctx);
  int l, h;
  if (bidir) kv_range_for_q_rows_bidir(m, m0, m1, &l, &h);
  else kv_range_for_q_rows(m, m0, m1, &l, &h);
  *lo = l;
  *hi = h;
  return 0;
}

static int q_range(bool bidir, int len, int num_targets, int max_attn_len, int min_full, int ctx, int n0, int n1, int32_t* lo,
                   int32_t* hi, int32_t* ctx_hi) {
  HSTU_CHECK_ARG(lo && hi && ctx_hi && n0 >= 0 && n1 > n0 && n1 <= len, "bad row range");
  const SeqMask m = make_seq_mask(len, num_targets, max_attn_len, min_full, ctx);
  int l, h, c;
  if (bidir) q_range_for_kv_rows_bidir(m, n0, n1, &l, &h, &c);
  else q_range_for_kv_rows(m, n0, n1, &l, &h, &c);
  *lo = l;
  *hi = h;
  *ctx_hi = c;
  return 0;
}

}  // namespace hstu

using namespace hstu;

extern "C" {

const char* hstu_last_error(void) { return g_err; }
int hstu_abi_version(void) { return HSTU_B200_ABI_VERSION; }

int hstu_attn_select_impl(const hstu_attn_params* p, int is_backward) { return checked_select_impl(p, is_backward != 0, false); }
size_t hstu_attn_workspace_bytes(const hstu_attn_params* p, int is_backward) { return workspace_bytes(p, is_backward != 0, false); }
int hstu_attn_fwd(const hstu_attn_params* p, void* stream) { return run_attn(p, false, false, (cudaStream_t)stream); }
int hstu_attn_bwd(const hstu_attn_params* p, void* stream) { return run_attn(p, true, false, (cudaStream_t)stream); }

int hstu_attn_bidir_select_impl(const hstu_attn_params* p, int is_backward) { return checked_select_impl(p, is_backward != 0, true); }
size_t hstu_attn_bidir_workspace_bytes(const hstu_attn_params* p, int is_backward) { return workspace_bytes(p, is_backward != 0, true); }
int hstu_attn_fwd_bidir(const hstu_attn_params* p, void* stream) { return run_attn(p, false, true, (cudaStream_t)stream); }
int hstu_attn_bwd_bidir(const hstu_attn_params* p, void* stream) { return run_attn(p, true, true, (cudaStream_t)stream); }

int hstu_attn_fwd_fp8(const hstu_attn_params* p, const hstu_attn_descales* descales, void* stream) {
  if (int e = validate_attn(p, false)) return e;
  HSTU_CHECK_ARG(p->dtype == HSTU_E4M3, "hstu_attn_fwd_fp8: q, k, v must be HSTU_E4M3 (got dtype %d)", p->dtype);
  if (int e = validate_descales(descales)) return e;
  const int impl = select_impl(p, false, false);
  if (impl < 0) return impl;
  if (p->batch == 0 || p->total_rows == 0) return 0;
  if (int e = bind_device(p->q)) return e;
  if (int e = check_descale_devices(descales)) return e;
  if (!is_sm90()) {
    set_error("hstu_attn_fwd_fp8: the fp8 kernels need an sm_90 device");
    return HSTU_ERR_UNSUPPORTED;
  }
  hstu_attn_descales none;
  memset(&none, 0, sizeof(none));
  return attn_wgmma_fwd_e4m3(*p, descales ? *descales : none, (cudaStream_t)stream);
}

int hstu_attn_fwd_delta_fp8_kv(const hstu_attn_params* p, const hstu_attn_descales* descales, void* stream) {
  if (int e = validate_attn(p, false)) return e;
  HSTU_CHECK_ARG(descales == nullptr || descales->q == nullptr,
                 "hstu_attn_fwd_delta_fp8_kv: q is bf16 / fp16 and takes no descale (descales->q must be NULL)");
  if (int e = validate_descales(descales)) return e;
  if (int e = delta_fp8_kv_check(*p)) return e;
  if (p->batch == 0 || p->total_rows == 0) return 0;
  if (int e = bind_device(p->q)) return e;
  if (int e = check_descale_devices(descales)) return e;
  if (!is_sm90()) {
    set_error("hstu_attn_fwd_delta_fp8_kv: the fp8 K / V kernels need an sm_90 device");
    return HSTU_ERR_UNSUPPORTED;
  }
  hstu_attn_descales none;
  memset(&none, 0, sizeof(none));
  return attn_wgmma_fwd_delta_fp8_kv(*p, descales ? *descales : none, (cudaStream_t)stream);
}

size_t hstu_attn_fp8_kv_workspace_bytes(const hstu_attn_params* p) {
  if (p == nullptr || validate_attn(p, false) != 0 || p->batch == 0 || p->total_rows == 0) return 0;
  if (delta_fp8_kv_check(*p) != 0) return 0;
  return wgmma_delta_workspace_bytes(*p);  // the partials of the key chunks, by the rule of the 16-bit delta-q forward
}

size_t hstu_attn_fp16_operands_bytes(const hstu_attn_params* p) {
  if (p == nullptr || validate_attn(p, false) != 0) return 0;
  if (p->batch == 0 || p->total_rows == 0 || !wgmma_on_fp16_operands(p, false)) return 0;
  return fp16_operands_workspace_bytes(*p, false);
}

int hstu_attn_fwd_keep_fp16_operands(const hstu_attn_params* p, void* operands, size_t operands_bytes, void* stream) {
  if (int e = validate_attn(p, false)) return e;
  if (p->batch == 0 || p->total_rows == 0) return 0;
  HSTU_CHECK_ARG(operands != nullptr && (reinterpret_cast<uintptr_t>(operands) & 255) == 0,
                 "operands must be a 256-byte aligned buffer (got %p)", operands);
  if (int e = bind_device(p->q)) return e;
  if (!wgmma_on_fp16_operands(p, false)) {
    set_error("hstu_attn_fwd_keep_fp16_operands: only bf16 at dqk == dv == 32 on the wgmma kernels runs on fp16 operands");
    return HSTU_ERR_UNSUPPORTED;
  }
  const size_t need = fp16_operands_workspace_bytes(*p, false);
  HSTU_CHECK_ARG(operands_bytes >= need, "operands buffer of %zu bytes required (got %zu)", need, operands_bytes);
  hstu_attn_params c = *p;  // the operands buffer has the layout of the forward's workspace
  c.workspace = operands;
  c.workspace_bytes = need;
  return attn_wgmma_fwd(c, (cudaStream_t)stream);
}

size_t hstu_attn_bwd_fp16_operands_workspace_bytes(const hstu_attn_params* p) {
  if (p == nullptr || p->batch <= 0 || p->heads <= 0 || p->total_rows <= 0) return 0;
  return fp16_operands_dout_workspace_bytes(*p);
}

int hstu_attn_bwd_on_fp16_operands(const hstu_attn_params* p, const void* operands, size_t operands_bytes, void* stream) {
  HSTU_CHECK_ARG(p != nullptr, "params is NULL");
  HSTU_CHECK_ARG(operands != nullptr && (reinterpret_cast<uintptr_t>(operands) & 255) == 0,
                 "operands must be a 256-byte aligned buffer (got %p)", operands);
  // q, k, v: the copies in the buffer, contiguous [L, H, 32] views, so that every check sees the tensors the kernels read
  hstu_attn_params c = *p;
  const Fp16Operands kept = fp16_operands_at(c, const_cast<void*>(operands));
  c.q = kept.copy[0], c.k = kept.copy[1], c.v = kept.copy[2];
  c.q_row_stride = c.k_row_stride = c.v_row_stride = (int64_t)c.heads * c.dqk;
  c.q_head_stride = c.k_head_stride = c.v_head_stride = c.dqk;
  if (int e = validate_attn(&c, true)) return e;
  if (c.batch == 0 || c.total_rows == 0) return 0;
  // a buffer kept for other sizes (batch, heads, rows) would be read out of bounds
  const size_t need = fp16_operands_workspace_bytes(c, false);
  HSTU_CHECK_ARG(operands_bytes >= need, "operands buffer of %zu bytes required (got %zu): not kept by a forward of these sizes",
                 need, operands_bytes);
  if (int e = bind_device(c.dout)) return e;
  if (!wgmma_on_fp16_operands(&c, true)) {
    set_error("hstu_attn_bwd_on_fp16_operands: only bf16 at dqk == dv == 32 on the wgmma kernels runs on fp16 operands");
    return HSTU_ERR_UNSUPPORTED;
  }
  return attn_wgmma_bwd_on_fp16_operands(c, operands, (cudaStream_t)stream);
}

int hstu_mask_valid(int32_t len, int32_t num_targets, int32_t max_attn_len, int32_t min_full_attn_seq_len,
                    int32_t contextual_seq_len, int32_t i, int32_t j) {
  return seq_mask_valid(false, len, num_targets, max_attn_len, min_full_attn_seq_len, contextual_seq_len, i, j);
}

int hstu_kv_range_for_q_rows(int32_t len, int32_t num_targets, int32_t max_attn_len, int32_t min_full_attn_seq_len,
                             int32_t contextual_seq_len, int32_t m0, int32_t m1, int32_t* lo, int32_t* hi) {
  return kv_range(false, len, num_targets, max_attn_len, min_full_attn_seq_len, contextual_seq_len, m0, m1, lo, hi);
}

int hstu_q_range_for_kv_rows(int32_t len, int32_t num_targets, int32_t max_attn_len, int32_t min_full_attn_seq_len,
                             int32_t contextual_seq_len, int32_t n0, int32_t n1, int32_t* lo, int32_t* hi,
                             int32_t* ctx_hi) {
  return q_range(false, len, num_targets, max_attn_len, min_full_attn_seq_len, contextual_seq_len, n0, n1, lo, hi, ctx_hi);
}

int hstu_mask_valid_bidir(int32_t len, int32_t num_targets, int32_t max_attn_len, int32_t min_full_attn_seq_len,
                          int32_t contextual_seq_len, int32_t i, int32_t j) {
  return seq_mask_valid(true, len, num_targets, max_attn_len, min_full_attn_seq_len, contextual_seq_len, i, j);
}

int hstu_kv_range_for_q_rows_bidir(int32_t len, int32_t num_targets, int32_t max_attn_len, int32_t min_full_attn_seq_len,
                                   int32_t contextual_seq_len, int32_t m0, int32_t m1, int32_t* lo, int32_t* hi) {
  return kv_range(true, len, num_targets, max_attn_len, min_full_attn_seq_len, contextual_seq_len, m0, m1, lo, hi);
}

int hstu_q_range_for_kv_rows_bidir(int32_t len, int32_t num_targets, int32_t max_attn_len, int32_t min_full_attn_seq_len,
                                   int32_t contextual_seq_len, int32_t n0, int32_t n1, int32_t* lo, int32_t* hi,
                                   int32_t* ctx_hi) {
  return q_range(true, len, num_targets, max_attn_len, min_full_attn_seq_len, contextual_seq_len, n0, n1, lo, hi, ctx_hi);
}

int hstu_layer_norm_fwd(const void* x, const void* w, const void* b, void* y, float* mean, float* rstd, int64_t n_rows,
                        int32_t D, int64_t x_row_stride, int64_t y_row_stride, float eps, int32_t dtype, int32_t swish,
                        void* stream) {
  if (n_rows > 0) if (int e = bind_device(x)) return e;
  HSTU_CHECK_ARG(n_rows >= 0 && (n_rows == 0 || (x && y)), "layer_norm_fwd: NULL x/y");
  return layer_norm_fwd(x, w, b, y, mean, rstd, n_rows, D, x_row_stride, y_row_stride, eps, dtype, swish, false,
                        (cudaStream_t)stream);
}

int hstu_layer_norm_bwd(const void* dy, const void* x, const void* w, const void* b, const float* mean, const float* rstd,
                        void* dx, float* dw, float* db, float* partial, int64_t n_rows, int32_t D, int64_t x_row_stride,
                        int64_t dy_row_stride, int64_t dx_row_stride, int32_t dtype, int32_t swish, void* stream) {
  if (n_rows > 0) if (int e = bind_device(x)) return e;
  HSTU_CHECK_ARG(n_rows >= 0 && (n_rows == 0 || (dy && x && dx && mean && rstd)), "layer_norm_bwd: NULL argument");
  return layer_norm_bwd(dy, x, w, b, mean, rstd, dx, dw, db, partial, n_rows, D, x_row_stride, dy_row_stride,
                        dx_row_stride, dtype, swish, false, (cudaStream_t)stream);
}

int32_t hstu_norm_bwd_partial_rows(void) { return norm_partial_rows(); }

int hstu_rms_norm_fwd(const void* x, const void* w, void* y, float* rstd, int64_t n_rows, int32_t D, float eps,
                      int32_t dtype, void* stream) {
  if (n_rows > 0) if (int e = bind_device(x)) return e;
  HSTU_CHECK_ARG(n_rows >= 0 && (n_rows == 0 || (x && y && w)), "rms_norm_fwd: NULL argument");
  return layer_norm_fwd(x, w, nullptr, y, nullptr, rstd, n_rows, D, D, D, eps, dtype, 0, true, (cudaStream_t)stream);
}

int hstu_rms_norm_bwd(const void* dy, const void* x, const void* w, const float* rstd, void* dx, float* dw,
                      float* partial, int64_t n_rows, int32_t D, int32_t dtype, void* stream) {
  if (n_rows > 0) if (int e = bind_device(x)) return e;
  HSTU_CHECK_ARG(n_rows >= 0 && (n_rows == 0 || (dy && x && w && dx && rstd)), "rms_norm_bwd: NULL argument");
  return layer_norm_bwd(dy, x, w, nullptr, nullptr, rstd, dx, dw, nullptr, partial, n_rows, D, D, D, D, dtype, 0, true,
                        (cudaStream_t)stream);
}

int hstu_norm_mul_dropout_fwd(const void* attn, const void* u, const void* w, const void* b, void* out, float* mean,
                              float* rstd, int64_t n_rows, int32_t heads, int32_t dv, int64_t attn_row_stride,
                              int64_t u_row_stride, float eps, float dropout_p, uint64_t seed, int32_t dtype,
                              int32_t silu_u, int32_t concat_ux, int32_t group_norm, void* stream) {
  if (n_rows > 0) if (int e = bind_device(attn)) return e;
  HSTU_CHECK_ARG(n_rows >= 0 && (n_rows == 0 || (attn && u && w && b && out)), "norm_mul_dropout_fwd: NULL argument");
  HSTU_CHECK_ARG(dropout_p >= 0.f && dropout_p < 1.f, "dropout_p must be in [0, 1)");
  return norm_mul_dropout_fwd(attn, u, w, b, out, mean, rstd, n_rows, heads, dv, attn_row_stride, u_row_stride, eps,
                              dropout_p, seed, dtype, silu_u, concat_ux, group_norm, (cudaStream_t)stream);
}

int hstu_norm_mul_dropout_bwd(const void* dout, const void* attn, const void* u, const void* w, const void* b,
                              const float* mean, const float* rstd, void* dattn, void* du, float* dw, float* db,
                              float* partial, int64_t n_rows, int32_t heads, int32_t dv, int64_t attn_row_stride,
                              int64_t u_row_stride, int64_t dattn_row_stride, int64_t du_row_stride, float dropout_p,
                              uint64_t seed, int32_t dtype, int32_t silu_u, int32_t concat_ux, int32_t group_norm,
                              void* stream) {
  if (n_rows > 0) if (int e = bind_device(attn)) return e;
  HSTU_CHECK_ARG(n_rows >= 0 && (n_rows == 0 || (dout && attn && u && w && b && mean && rstd && dattn && du)),
                 "norm_mul_dropout_bwd: NULL argument");
  return norm_mul_dropout_bwd(dout, attn, u, w, b, mean, rstd, dattn, du, dw, db, partial, n_rows, heads, dv,
                              attn_row_stride, u_row_stride, dattn_row_stride, du_row_stride, dropout_p, seed, dtype,
                              silu_u, concat_ux, group_norm, (cudaStream_t)stream);
}

int hstu_silu_fwd(const void* x, void* y, int64_t n_rows, int32_t n_cols, int64_t x_row_stride, int64_t y_row_stride,
                  int32_t dtype, void* stream) {
  if (n_rows > 0) if (int e = bind_device(x)) return e;
  HSTU_CHECK_ARG(n_rows >= 0 && (n_rows == 0 || (x && y)), "silu_fwd: NULL argument");
  return silu_fwd_bwd(x, nullptr, y, n_rows, n_cols, x_row_stride, 0, y_row_stride, dtype, false, (cudaStream_t)stream);
}

int hstu_silu_bwd(const void* dy, const void* x, void* dx, int64_t n_rows, int32_t n_cols, int64_t dy_row_stride,
                  int64_t x_row_stride, int64_t dx_row_stride, int32_t dtype, void* stream) {
  if (n_rows > 0) if (int e = bind_device(x)) return e;
  HSTU_CHECK_ARG(n_rows >= 0 && (n_rows == 0 || (dy && x && dx)), "silu_bwd: NULL argument");
  return silu_fwd_bwd(x, dy, dx, n_rows, n_cols, x_row_stride, dy_row_stride, dx_row_stride, dtype, true,
                      (cudaStream_t)stream);
}

int hstu_jagged_concat(const void* left, const void* right, void* out, const void* offsets_left, const void* offsets_right,
                       int32_t offsets_are_i64, int32_t batch, int32_t dense_len_left, int32_t dense_len_right,
                       int32_t n_prefix, int32_t D, int32_t elem_bytes, int32_t max_seq_len, void* stream) {
  if (int e = bind_device(out)) return e;
  HSTU_CHECK_ARG(offsets_left || offsets_right, "offsets_left and offsets_right cannot be None at the same time");
  HSTU_CHECK_ARG(elem_bytes == 1 || elem_bytes == 2 || elem_bytes == 4 || elem_bytes == 8, "bad elem_bytes");
  return jagged_concat_split(false, left, right, out, nullptr, offsets_left, offsets_right, offsets_are_i64, batch,
                             dense_len_left, dense_len_right, n_prefix, D, elem_bytes, max_seq_len, (cudaStream_t)stream);
}

int hstu_jagged_split(const void* in, void* left, void* right, const void* offsets_left, const void* offsets_right,
                      int32_t offsets_are_i64, int32_t batch, int32_t dense_len_left, int32_t dense_len_right,
                      int32_t n_prefix, int32_t D, int32_t elem_bytes, int32_t max_seq_len, void* stream) {
  if (int e = bind_device(in)) return e;
  HSTU_CHECK_ARG(offsets_left || offsets_right, "offsets_left and offsets_right cannot be None at the same time");
  HSTU_CHECK_ARG(elem_bytes == 1 || elem_bytes == 2 || elem_bytes == 4 || elem_bytes == 8, "bad elem_bytes");
  return jagged_concat_split(true, in, nullptr, left, right, offsets_left, offsets_right, offsets_are_i64, batch,
                             dense_len_left, dense_len_right, n_prefix, D, elem_bytes, max_seq_len, (cudaStream_t)stream);
}

int hstu_position_embeddings_fwd(const void* seq_embeddings, void* out, const float* pos_w, const float* ts_w,
                                 const void* seq_offsets, const void* seq_lengths, const void* num_targets,
                                 const int64_t* timestamps, int32_t* pos_inds, int32_t* ts_inds, int64_t total_rows,
                                 int32_t batch, int32_t D, int32_t max_pos_ind, int32_t num_time_buckets,
                                 int32_t max_contextual_seq_len, float alpha, int32_t interleave_targets,
                                 int32_t log_time_bucket, int32_t offsets_are_i64, int32_t lengths_are_i64,
                                 int32_t num_targets_are_i64, int32_t dtype, void* stream) {
  HSTU_CHECK_ARG(total_rows >= 0 && batch >= 0 && D > 0, "position_embeddings_fwd: bad sizes");
  if (total_rows == 0) return 0;
  if (int e = bind_device(seq_embeddings)) return e;
  HSTU_CHECK_ARG(seq_embeddings && out && pos_w && ts_w && seq_offsets && seq_lengths && timestamps,
                 "position_embeddings_fwd: NULL argument");
  HSTU_CHECK_ARG(max_pos_ind > 0 && num_time_buckets >= 0, "position_embeddings_fwd: empty embedding table");
  PosArgs a;
  a.seq = seq_embeddings; a.out = out; a.pos_w = pos_w; a.ts_w = ts_w;
  a.seq_offsets = seq_offsets; a.seq_lengths = seq_lengths; a.num_targets = num_targets;
  a.timestamps = reinterpret_cast<const long long*>(timestamps);
  a.pos_inds = pos_inds; a.ts_inds = ts_inds;
  a.L = total_rows; a.B = batch; a.D = D;
  a.max_pos_ind = max_pos_ind; a.num_time_buckets = num_time_buckets; a.max_contextual = max_contextual_seq_len;
  a.offsets_i64 = offsets_are_i64; a.lengths_i64 = lengths_are_i64; a.targets_i64 = num_targets_are_i64;
  a.interleave = interleave_targets; a.log_bucket = log_time_bucket;
  a.vec_ok = (((uintptr_t)seq_embeddings | (uintptr_t)out | (uintptr_t)pos_w | (uintptr_t)ts_w) & 15) == 0;
  a.alpha = alpha;
  return position_fwd(a, dtype, (cudaStream_t)stream);
}

int hstu_position_embeddings_bwd(const void* dout, void* d_seq_embeddings, float* d_pos_w, float* d_ts_w,
                                 const int32_t* pos_inds, const int32_t* ts_inds, int64_t total_rows, int32_t D, float alpha,
                                 int32_t dtype, void* stream) {
  HSTU_CHECK_ARG(total_rows >= 0 && D > 0, "position_embeddings_bwd: bad sizes");
  if (total_rows == 0) return 0;
  if (int e = bind_device(dout)) return e;
  HSTU_CHECK_ARG(dout && d_seq_embeddings && d_pos_w && d_ts_w && pos_inds && ts_inds, "position_embeddings_bwd: NULL argument");
  return position_bwd(dout, d_seq_embeddings, d_pos_w, d_ts_w, pos_inds, ts_inds, total_rows, D, alpha, dtype, (cudaStream_t)stream);
}

int hstu_jagged_dense_bmm_broadcast_add(const void* jagged, const void* dense, const void* bias, void* out,
                                        const void* seq_offsets, int32_t offsets_are_i64, int32_t batch, int32_t K, int32_t N,
                                        int32_t max_seq_len, int32_t dense_is_transposed, int32_t dtype, void* stream) {
  HSTU_CHECK_ARG(batch >= 0 && K > 0 && N > 0 && max_seq_len > 0, "jagged_dense_bmm_broadcast_add: bad sizes");
  if (batch == 0) return 0;
  if (int e = bind_device(dense)) return e;
  HSTU_CHECK_ARG(dense && seq_offsets, "jagged_dense_bmm_broadcast_add: NULL argument");
  return jagged_bmm(jagged, dense, bias, out, seq_offsets, offsets_are_i64, batch, K, N, max_seq_len, dense_is_transposed != 0, dtype,
                    (cudaStream_t)stream);
}

int hstu_jagged_dense_bmm_wgrad(const void* jagged, const void* dout, void* d_dense, void* d_bias, const void* seq_offsets,
                                int32_t offsets_are_i64, int32_t batch, int32_t K, int32_t N, int32_t max_seq_len, int32_t dtype,
                                void* stream) {
  HSTU_CHECK_ARG(batch >= 0 && K > 0 && N > 0 && max_seq_len > 0, "jagged_dense_bmm_wgrad: bad sizes");
  if (batch == 0) return 0;
  if (int e = bind_device(d_dense)) return e;
  HSTU_CHECK_ARG(d_dense && seq_offsets, "jagged_dense_bmm_wgrad: NULL argument");
  return jagged_bmm_wgrad(jagged, dout, d_dense, d_bias, seq_offsets, offsets_are_i64, batch, K, N, max_seq_len, dtype,
                          (cudaStream_t)stream);
}

static int validate_ssl(const hstu_ssl_params* p, bool bwd) {
  HSTU_CHECK_ARG(p != nullptr, "params is NULL");
  HSTU_CHECK_ARG(p->abi_version == HSTU_B200_ABI_VERSION, "ABI version mismatch: caller %d, library %d", p->abi_version,
                 HSTU_B200_ABI_VERSION);
  HSTU_CHECK_ARG(p->N >= 0 && p->R >= 0 && p->D > 0, "sampled softmax: bad sizes");
  HSTU_CHECK_ARG(p->temperature > 0.f, "sampled softmax: temperature must be positive");
  if (p->N == 0) return 0;
  HSTU_CHECK_ARG(p->q && p->pos_emb && p->table && p->pos_ids && (p->neg_ids || p->R == 0), "sampled softmax: NULL input");
  HSTU_CHECK_ARG(p->logits && p->rnorm && p->lse, "sampled softmax: NULL logits / rnorm / lse");
  if (!bwd) HSTU_CHECK_ARG(p->loss_rows != nullptr, "sampled softmax: NULL loss_rows");
  if (bwd) HSTU_CHECK_ARG(p->row_coef && p->d_q && p->d_pos_emb && p->d_table, "sampled softmax backward: NULL argument");
  return 0;
}

int hstu_sampled_softmax_fwd(const hstu_ssl_params* p, void* stream) {
  if (int e = validate_ssl(p, false)) return e;
  if (p->N == 0) return 0;
  if (int e = bind_device(p->q)) return e;
  return sampled_softmax_fwd(*p, p->dtype, (cudaStream_t)stream);
}

int hstu_sampled_softmax_bwd(const hstu_ssl_params* p, void* stream) {
  if (int e = validate_ssl(p, true)) return e;
  if (p->N == 0) return 0;
  if (int e = bind_device(p->q)) return e;
  return sampled_softmax_bwd(*p, p->dtype, (cudaStream_t)stream);
}


}  // extern "C"
