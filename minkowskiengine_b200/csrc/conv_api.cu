// C-ABI entry points of the sparse convolution; picks the tensor-core path when the shape
// qualifies (conv_tc.cuh) and the SIMT path otherwise.
#include <stdlib.h>

#include <algorithm>

#include "common.cuh"
#include "conv_simt.cuh"
#include "conv_tc.cuh"

using namespace meb200;

static bool tc_disabled() {
  static int v = -1;
  if (v < 0) {
    const char *e = getenv("MEB200_DISABLE_TC");
    v = (e && e[0] && e[0] != '0') ? 1 : 0;
  }
  return v == 1;
}

extern "C" {

uint64_t meb200_conv_workspace_bytes(uint32_t n_in, uint32_t n_out, uint32_t c_in,
                                     uint32_t c_out, uint32_t K, int dtype) {
  (void)n_in;
  // the row-split partial sums of a SIMT wgrad (any dtype); for bf16/fp16 also the weights
  // re-laid out for the tensor-core kernels (W^T per offset) or the row-split partial sums of
  // the tensor-core wgrad (no call needs two of these at once)
  const uint64_t ws = conv_wgrad_simt_workspace_bytes(c_in, c_out, K, n_out);
  if (dtype == MEB200_F32) return ws;
  const uint64_t wt = (uint64_t)K * c_in * c_out * 2 + 256;
  const uint64_t wg = conv_wgrad_workspace_bytes(c_in, c_out, K, n_out);
  return std::max({ws, wt, wg});
}

uint64_t meb200_conv_wgrad_workspace_bytes(uint32_t c_in, uint32_t c_out, uint32_t K,
                                           uint32_t n_out) {
  return conv_wgrad_workspace_bytes(c_in, c_out, K, n_out);
}

int meb200_conv_forward(const void *in, int in_dtype, uint32_t n_in, uint32_t c_in,
                        const void *weight, uint32_t K, uint32_t c_out, const int32_t *out_nbr,
                        uint32_t n_out, void *out, int out_dtype, void *workspace,
                        uint64_t workspace_bytes, void *stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  if (n_out == 0) return MEB200_OK;
  MEB_CHECK_ARG(in_dtype >= 0 && in_dtype <= 2 && out_dtype >= 0 && out_dtype <= 2, "dtype");
  MEB_CHECK_ARG(out_dtype == MEB200_F32 || out_dtype == in_dtype,
                "output dtype must be fp32 or the input dtype");
  MEB_CHECK_ARG(out && weight && out_nbr && (in || n_in == 0), "null buffer");
  MEB_CHECK_ARG(c_in > 0 && c_out > 0 && K > 0, "empty channel/kernel dims");
  if (!tc_disabled() && conv_tc_supported(in_dtype, c_in, c_out) &&
      workspace_bytes >= (uint64_t)K * c_in * c_out * 2) {
    int rc = conv_forward_tc(in, in_dtype, n_in, c_in, weight, K, c_out, /*dgrad=*/false,
                             out_nbr, n_out, out, out_dtype, workspace, stream);
    if (rc != MEB200_ERR_UNSUPPORTED) return rc;
  }
  if (conv_small_cin_supported(c_in, c_out)) {
    int rc = conv_small_cin_forward(in, in_dtype, c_in, weight, K, c_out, out_nbr, n_out, out,
                                    out_dtype, stream);
    if (rc != MEB200_ERR_UNSUPPORTED) return rc;
  }
  return conv_forward_simt(in, in_dtype, n_in, c_in, weight, K, c_out, /*trans_w=*/false,
                           out_nbr, n_out, out, out_dtype, stream);
}

int meb200_conv_pack_weights(const float *weight, uint32_t K, uint32_t c_in, uint32_t c_out,
                             int dtype, void *w_cast, void *w_t, void *w_cp, void *w_tp,
                             void *stream_) {
  MEB_CHECK_ARG(dtype == MEB200_BF16 || dtype == MEB200_F16, "packed weights are bf16 or fp16");
  MEB_CHECK_ARG(weight && w_cast && w_t, "null buffer");
  MEB_CHECK_ARG(c_in > 0 && c_out > 0 && K > 0 && K <= 65535, "empty channel/kernel dims");
  return conv_pack_weights(weight, K, c_in, c_out, dtype, w_cast, w_t, w_cp, w_tp,
                           (cudaStream_t)stream_);
}

static_assert(sizeof(meb200_pack_job) == sizeof(PackJob), "meb200_pack_job layout");

int meb200_conv_pack_weights_batched(const meb200_pack_job *jobs_dev, uint32_t n_jobs,
                                     uint32_t total_tiles, int dtype, void *stream_) {
  MEB_CHECK_ARG(dtype == MEB200_BF16 || dtype == MEB200_F16, "packed weights are bf16 or fp16");
  MEB_CHECK_ARG(jobs_dev != nullptr || n_jobs == 0, "null job table");
  return conv_pack_weights_batched(reinterpret_cast<const PackJob *>(jobs_dev), n_jobs, total_tiles,
                                   dtype, (cudaStream_t)stream_);
}

uint32_t meb200_conv_stem_virtual_channels(uint32_t K) { return 4u * ((K + 15u) / 16u * 16u); }

int meb200_conv_stem_supported(int dtype, uint32_t K, uint32_t c_out) {
  if (tc_disabled()) return 0;
  return conv_stem_tc_supported(dtype, K, c_out) && conv_stem_wgrad_tc_supported(dtype, K, c_out) ? 1 : 0;
}

int meb200_conv_stem_forward(const void *in4, int dtype, uint32_t K, const void *weight_v,
                             uint32_t c_out, const int32_t *out_nbr, uint32_t n_out, void *out,
                             int out_dtype, void *stream_) {
  if (n_out == 0) return MEB200_OK;
  MEB_CHECK_ARG(out_dtype == MEB200_F32 || out_dtype == dtype, "output dtype must be fp32 or the input dtype");
  MEB_CHECK_ARG(in4 && weight_v && out_nbr && out, "null buffer");
  if (tc_disabled() || !conv_stem_tc_supported(dtype, K, c_out)) {
    set_error("stem forward: shape/dtype outside the tensor-core path (K=%u c_out=%u)", K, c_out);
    return MEB200_ERR_UNSUPPORTED;
  }
  return conv_stem_forward_tc(in4, dtype, K, weight_v, c_out, out_nbr, n_out, out, out_dtype,
                              (cudaStream_t)stream_);
}

int meb200_conv_stem_wgrad(const void *in4, const void *grad_out, int dtype, uint32_t K,
                           uint32_t c_out, const int32_t *out_nbr, uint32_t n_out,
                           float *grad_weight_v, void *workspace, uint64_t workspace_bytes,
                           void *stream_) {
  MEB_CHECK_ARG(grad_weight_v && (n_out == 0 || (in4 && grad_out && out_nbr)), "null buffer");
  if (tc_disabled() || !conv_stem_wgrad_tc_supported(dtype, K, c_out)) {
    set_error("stem wgrad: shape/dtype outside the tensor-core path (K=%u c_out=%u)", K, c_out);
    return MEB200_ERR_UNSUPPORTED;
  }
  return conv_stem_wgrad_tc(in4, grad_out, dtype, K, c_out, out_nbr, n_out, grad_weight_v,
                            workspace, workspace_bytes, (cudaStream_t)stream_);
}

int meb200_conv_forward_packed(const void *in, int in_dtype, uint32_t n_in, uint32_t c_in,
                               const void *weight_t, const void *weight_tp, uint32_t K,
                               uint32_t c_out, const int32_t *out_nbr, uint32_t n_out, void *out,
                               int out_dtype, void *stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  (void)weight_tp;   // the permuted copy: accepted for ABI stability, the kernels read weight_t
  if (n_out == 0) return MEB200_OK;
  MEB_CHECK_ARG(in_dtype >= 0 && in_dtype <= 2 && out_dtype >= 0 && out_dtype <= 2, "dtype");
  MEB_CHECK_ARG(out_dtype == MEB200_F32 || out_dtype == in_dtype,
                "output dtype must be fp32 or the input dtype");
  MEB_CHECK_ARG(out && weight_t && out_nbr && (in || n_in == 0), "null buffer");
  MEB_CHECK_ARG(c_in > 0 && c_out > 0 && K > 0, "empty channel/kernel dims");
  if (tc_disabled() || !conv_tc_supported(in_dtype, c_in, c_out)) {
    set_error("packed forward: shape/dtype outside the tensor-core path");
    return MEB200_ERR_UNSUPPORTED;
  }
  // W^T[k][c_out][c_in] is operand B as the kernels want it: the "no transpose" entry
  return conv_forward_tc(in, in_dtype, n_in, c_in, weight_t, K, c_out, /*dgrad=*/true, out_nbr,
                         n_out, out, out_dtype, nullptr, stream);
}

int meb200_conv_backward_packed(const void *in, const void *grad_out, int dtype, uint32_t n_in,
                                uint32_t c_in, const void *w_cast, const void *w_cp, uint32_t K,
                                uint32_t c_out, const int32_t *out_nbr, const int32_t *in_nbr,
                                uint32_t n_out, void *grad_in, int grad_in_dtype,
                                float *grad_weight, const int32_t *pairs_in,
                                const int32_t *pairs_out, const int32_t *seg_start,
                                uint32_t n_chunks, void *workspace, uint64_t workspace_bytes,
                                void *stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  (void)w_cp;        // the permuted copy: accepted for ABI stability, the kernels read w_cast
  MEB_CHECK_ARG(dtype == MEB200_BF16 || dtype == MEB200_F16, "packed backward is bf16 or fp16");
  MEB_CHECK_ARG(grad_in_dtype == MEB200_F32 || grad_in_dtype == dtype,
                "grad_in dtype must be fp32 or the feature dtype");
  MEB_CHECK_ARG(c_in > 0 && c_out > 0 && K > 0, "empty channel/kernel dims");
  // all-or-nothing: decide before anything is launched, the caller falls back as a whole
  if (tc_disabled() ||
      (grad_in != nullptr && n_in > 0 && !conv_tc_supported(dtype, c_out, c_in)) ||
      (grad_weight != nullptr && !conv_wgrad_tc_supported(dtype, c_in, c_out))) {
    set_error("packed backward: shape outside the tensor-core path");
    return MEB200_ERR_UNSUPPORTED;
  }
  if (grad_in != nullptr && n_in > 0) {
    MEB_CHECK_ARG(in_nbr && w_cast && (grad_out || n_out == 0), "null buffer");
    int rc = conv_forward_tc(grad_out, dtype, n_out, c_out, w_cast, K, c_in, /*dgrad=*/true, in_nbr,
                             n_in, grad_in, grad_in_dtype, nullptr, stream);
    if (rc != MEB200_OK) return rc;
  }
  if (grad_weight != nullptr) {
    MEB_CHECK_ARG(out_nbr && (in || n_in == 0) && (grad_out || n_out == 0), "null buffer");
    static int use_pairs = -1;    // MEB200_TC_WGRAD=dense walks the table instead of the pair lists
    if (use_pairs < 0) {
      const char *e = getenv("MEB200_TC_WGRAD");
      use_pairs = (e && e[0] == 'd') ? 0 : 1;
    }
    if (use_pairs && pairs_in && pairs_out && seg_start && n_chunks > 0 &&
        conv_wgrad_pairs_supported(dtype, c_in, K, c_out)) {
      int rc = conv_wgrad_pairs(in, grad_out, dtype, c_in, K, c_out, pairs_in, pairs_out,
                                seg_start, n_chunks, n_out, grad_weight, workspace,
                                workspace_bytes, stream);
      if (rc != MEB200_ERR_UNSUPPORTED) return rc;
    }
    return conv_wgrad_tc(in, grad_out, dtype, c_in, K, c_out, out_nbr, n_out, grad_weight,
                         workspace, workspace_bytes, stream);
  }
  return MEB200_OK;
}

int meb200_conv_backward(const void *in, const void *grad_out, int dtype, uint32_t n_in,
                         uint32_t c_in, const void *weight, uint32_t K, uint32_t c_out,
                         const int32_t *out_nbr, const int32_t *in_nbr, uint32_t n_out,
                         void *grad_in, int grad_in_dtype, float *grad_weight, void *workspace,
                         uint64_t workspace_bytes, void *stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  MEB_CHECK_ARG(dtype >= 0 && dtype <= 2, "dtype");
  MEB_CHECK_ARG(grad_in_dtype == MEB200_F32 || grad_in_dtype == dtype,
                "grad_in dtype must be fp32 or the feature dtype");
  MEB_CHECK_ARG(c_in > 0 && c_out > 0 && K > 0, "empty channel/kernel dims");
  bool tc = !tc_disabled() && workspace_bytes >= (uint64_t)K * c_in * c_out * 2;
  if (grad_in != nullptr && n_in > 0) {
    MEB_CHECK_ARG(in_nbr && weight && (grad_out || n_out == 0), "null buffer");
    // dgrad = the forward kernel on the transposed table with W_k^T:
    // rows = input rows, reduction over c_out, produces c_in columns.
    int rc = MEB200_ERR_UNSUPPORTED;
    if (tc && conv_tc_supported(dtype, c_out, c_in))
      rc = conv_forward_tc(grad_out, dtype, n_out, c_out, weight, K, c_in, /*dgrad=*/true,
                           in_nbr, n_in, grad_in, grad_in_dtype, workspace, stream);
    if (rc == MEB200_ERR_UNSUPPORTED)
      rc = conv_forward_simt(grad_out, dtype, n_out, c_out, weight, K, c_in, /*trans_w=*/true,
                             in_nbr, n_in, grad_in, grad_in_dtype, stream);
    if (rc != MEB200_OK) return rc;
  }
  if (grad_weight != nullptr) {
    MEB_CHECK_ARG(out_nbr && (in || n_in == 0) && (grad_out || n_out == 0), "null buffer");
    if (tc && conv_wgrad_tc_supported(dtype, c_in, c_out)) {
      int rc = conv_wgrad_tc(in, grad_out, dtype, c_in, K, c_out, out_nbr, n_out, grad_weight,
                             workspace, workspace_bytes, stream);
      if (rc != MEB200_ERR_UNSUPPORTED) return rc;
    }
    if (conv_small_cin_supported(c_in, c_out))
      return conv_small_cin_wgrad(in, grad_out, dtype, c_in, K, c_out, out_nbr, n_out,
                                  grad_weight, workspace, workspace_bytes, stream);
    return conv_wgrad_simt(in, grad_out, dtype, c_in, K, c_out, out_nbr, n_out, grad_weight,
                           workspace, workspace_bytes, stream);
  }
  return MEB200_OK;
}

}
