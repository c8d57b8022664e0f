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
  HSTU_CHECK_ARG(p->dtype == HSTU_F32 || p->dtype == HSTU_BF16 || p->dtype == HSTU_F16, "bad dtype %d", p->dtype);
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

// A deterministic backward takes the same route as any other: the wgmma kernels run their atomic-free split path
// (attn_wgmma_bwd.cu), and the generic kernels have no atomics on q / k / v.
static int select_impl(const hstu_attn_params* p, bool bwd) {
  if (bwd && p->deterministic && (p->pos_w != nullptr || p->ts_w != nullptr)) {
    set_error("deterministic backward with a relative bias is not supported: the dpos_w / dts_w gradients are added "
              "with atomics");
    return HSTU_ERR_UNSUPPORTED;
  }
  const bool can = wgmma_supported(*p, bwd);
  if (p->impl == HSTU_IMPL_GENERIC) return HSTU_IMPL_GENERIC;
  if (p->impl == HSTU_IMPL_UMMA) {
    if (!can) {
      set_error("wgmma path does not support this problem (dtype=%d dqk=%d dv=%d delta=%d bias=%d)", p->dtype, p->dqk,
                p->dv, p->delta_q_len, p->pos_w != nullptr || p->ts_w != nullptr);
      return HSTU_ERR_UNSUPPORTED;
    }
    return HSTU_IMPL_UMMA;
  }
  return can ? HSTU_IMPL_UMMA : HSTU_IMPL_GENERIC;
}

}  // namespace hstu

using namespace hstu;

extern "C" {

const char* hstu_last_error(void) { return g_err; }
int hstu_abi_version(void) { return HSTU_B200_ABI_VERSION; }

int hstu_attn_select_impl(const hstu_attn_params* p, int is_backward) {
  if (int e = validate_attn(p, is_backward != 0)) return e;
  return select_impl(p, is_backward != 0);
}

size_t hstu_attn_workspace_bytes(const hstu_attn_params* p, int is_backward) {
  if (p == nullptr) return 0;
  if (validate_attn(p, is_backward != 0) != 0) return 0;
  if (p->batch == 0 || p->total_rows == 0) return 0;
  int impl = select_impl(p, is_backward != 0);
  if (impl == HSTU_IMPL_UMMA) return wgmma_workspace_bytes(*p, is_backward != 0);
  return 0;
}

int hstu_attn_fwd(const hstu_attn_params* p, void* stream) {
  if (int e = validate_attn(p, false)) return e;
  if (p->batch == 0 || p->total_rows == 0) return 0;  // triton_hstu_attention.py:1789-1790
  if (int e = bind_device(p->q)) return e;
  int impl = select_impl(p, false);
  if (impl < 0) return impl;
  if (impl == HSTU_IMPL_UMMA) return attn_wgmma_fwd(*p, (cudaStream_t)stream);
  return attn_generic_fwd(*p, (cudaStream_t)stream);
}

int hstu_attn_bwd(const hstu_attn_params* p, void* stream) {
  if (int e = validate_attn(p, true)) return e;
  if (p->batch == 0 || p->total_rows == 0) return 0;
  if (int e = bind_device(p->q)) return e;
  int impl = select_impl(p, true);
  if (impl < 0) return impl;
  if (impl == HSTU_IMPL_UMMA) return attn_wgmma_bwd(*p, (cudaStream_t)stream);
  return attn_generic_bwd(*p, (cudaStream_t)stream);
}

int hstu_mask_valid(int32_t len, int32_t num_targets, int32_t max_attn_len, int32_t min_full_attn_seq_len,
                    int32_t contextual_seq_len, int32_t i, int32_t j) {
  SeqMask m = make_seq_mask(len, num_targets, max_attn_len, min_full_attn_seq_len, contextual_seq_len);
  return mask_valid(m, i, j) ? 1 : 0;
}

int hstu_kv_range_for_q_rows(int32_t len, int32_t num_targets, int32_t max_attn_len, int32_t min_full_attn_seq_len,
                             int32_t contextual_seq_len, int32_t m0, int32_t m1, int32_t* lo, int32_t* hi) {
  HSTU_CHECK_ARG(lo && hi && m0 >= 0 && m1 > m0 && m1 <= len, "bad row range");
  SeqMask m = make_seq_mask(len, num_targets, max_attn_len, min_full_attn_seq_len, contextual_seq_len);
  int l, h;
  kv_range_for_q_rows(m, m0, m1, &l, &h);
  *lo = l;
  *hi = h;
  return 0;
}

int hstu_q_range_for_kv_rows(int32_t len, int32_t num_targets, int32_t max_attn_len, int32_t min_full_attn_seq_len,
                             int32_t contextual_seq_len, int32_t n0, int32_t n1, int32_t* lo, int32_t* hi,
                             int32_t* ctx_hi) {
  HSTU_CHECK_ARG(lo && hi && ctx_hi && n0 >= 0 && n1 > n0 && n1 <= len, "bad row range");
  SeqMask m = make_seq_mask(len, num_targets, max_attn_len, min_full_attn_seq_len, contextual_seq_len);
  int l, h, c;
  q_range_for_kv_rows(m, n0, n1, &l, &h, &c);
  *lo = l;
  *hi = h;
  *ctx_hi = c;
  return 0;
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
