// C-ABI entry points of the sparse convolution; picks the tensor-core path when the shape
// qualifies (conv_tc.cuh) and the small-cin / SIMT paths otherwise.
#include <algorithm>

#include "common.cuh"
#include "conv_simt.cuh"
#include "conv_tc.cuh"

using namespace meb200;

// dtype of the feature storage: TF32 convolutions keep fp32 features
static int storage_dtype(int dtype) { return dtype == MEB200_TF32 ? MEB200_F32 : dtype; }

// NULL, or scale and shift given; the tensor-core kernels read pairs of columns (8 bytes)
static bool epilogue_ok(const meb200_conv_epilogue *epi) {
  return epi == nullptr || (epi->scale && epi->shift && aligned(8, epi->scale, epi->shift) &&
                            (epi->residual == nullptr || aligned(8, epi->residual)));
}

extern "C" {

uint64_t meb200_conv_workspace_bytes(uint32_t n_out, uint32_t c_in, uint32_t c_out, uint32_t K,
                                     int dtype) {
  // the row-split partial sums of a SIMT wgrad (any dtype); for bf16/fp16/TF32 also those of the
  // tensor-core wgrad (no call needs both at once)
  const uint64_t ws = conv_wgrad_simt_workspace_bytes(c_in, c_out, K, n_out);
  if (dtype == MEB200_F32) return ws;
  return std::max(ws, conv_wgrad_workspace_bytes(c_in, c_out, K, n_out));
}

int meb200_conv_wgrad_uses_pairs(int dtype, uint32_t c_in, uint32_t c_out, uint32_t K) {
  return conv_wgrad_uses_pairs(dtype, c_in, c_out, K) ? 1 : 0;
}

int meb200_conv_forward(const void *in, int in_dtype, uint32_t n_in, uint32_t c_in,
                        const void *w_cast, const void *w_t, uint32_t K, uint32_t c_out,
                        const int32_t *out_nbr, uint32_t n_out, void *out, int out_dtype,
                        const int32_t *out_order, const meb200_conv_epilogue *epi,
                        void *stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  if (n_out == 0) return MEB200_OK;
  MEB_CHECK_ARG(in_dtype >= 0 && in_dtype <= 3 && out_dtype >= 0 && out_dtype <= 2, "dtype");
  MEB_CHECK_ARG(out_dtype == MEB200_F32 || out_dtype == in_dtype,
                "output dtype must be fp32 or the input dtype");
  MEB_CHECK_ARG(out && w_cast && (w_t || in_dtype == MEB200_F32) && out_nbr && (in || n_in == 0),
                "null buffer");
  MEB_CHECK_ARG(c_in > 0 && c_out > 0 && K > 0, "empty channel/kernel dims");
  MEB_CHECK_ARG(epilogue_ok(epi), "epilogue: scale and shift required, 8-byte aligned pointers");
  if (conv_tc_supported(in_dtype, c_in, c_out)) {
    int rc = conv_forward_tc(in, in_dtype, n_in, c_in, w_t, K, c_out, out_nbr, out_order, n_out,
                             out, out_dtype, epi, stream);
    if (rc != MEB200_ERR_UNSUPPORTED) return rc;
  }
  const int fdt = storage_dtype(in_dtype);      // the CUDA-core kernels: exact fp32 for TF32
  if (conv_small_cin_supported(c_in, c_out)) {
    int rc = conv_small_cin_forward(in, fdt, c_in, w_cast, K, c_out, out_nbr, n_out, out,
                                    out_dtype, epi, stream);
    if (rc != MEB200_ERR_UNSUPPORTED) return rc;
  }
  return conv_forward_simt(in, fdt, n_in, c_in, w_cast, K, c_out, /*trans_w=*/false,
                           out_nbr, n_out, out, out_dtype, epi, stream);
}

// The forward with a shadow: the 16-bit tensor-core route only (see include/meb200.h); anything
// else returns MEB200_ERR_UNSUPPORTED before it launches.
int meb200_conv_forward_q(const void *in, int in_dtype, uint32_t n_in, uint32_t c_in,
                          const void *w_cast, const void *w_t, uint32_t K, uint32_t c_out,
                          const int32_t *out_nbr, uint32_t n_out, void *out, int out_dtype,
                          const int32_t *out_order, const meb200_conv_epilogue *epi, void *q,
                          const float *q_scale, void *stream_) {
  if (n_out == 0) return MEB200_OK;
  MEB_CHECK_ARG(in_dtype == MEB200_BF16 || in_dtype == MEB200_F16, "shadow: bf16 / fp16 operands");
  MEB_CHECK_ARG(out_dtype == MEB200_F32 || out_dtype == in_dtype,
                "output dtype must be fp32 or the input dtype");
  MEB_CHECK_ARG(out && w_t && out_nbr && q && q_scale && (in || n_in == 0), "null buffer");
  MEB_CHECK_ARG(c_in > 0 && c_out > 0 && K > 0, "empty channel/kernel dims");
  MEB_CHECK_ARG(epi != nullptr && epilogue_ok(epi),
                "epilogue required: scale and shift, 8-byte aligned pointers");
  (void)w_cast;
  if (!conv_tc_supported(in_dtype, c_in, c_out)) {
    set_error("shadow: c_in=%u c_out=%u outside the tensor-core route", c_in, c_out);
    return MEB200_ERR_UNSUPPORTED;
  }
  const Shadow sh{reinterpret_cast<uint8_t *>(q), q_scale};
  return conv_forward_tc(in, in_dtype, n_in, c_in, w_t, K, c_out, out_nbr, out_order, n_out, out,
                         out_dtype, epi, (cudaStream_t)stream_, nullptr, &sh);
}

int meb200_conv_fp8_supported(uint32_t c_in, uint32_t c_out) {
  return conv_fp8_supported(c_in, c_out) ? 1 : 0;
}

int meb200_conv_forward_fp8(const void *in_e4m3, const float *a_scale, uint32_t n_in, uint32_t c_in,
                            const void *w_t_e4m3, uint32_t K, uint32_t c_out,
                            const int32_t *out_nbr, uint32_t n_out, void *out, int out_dtype,
                            const int32_t *out_order, const meb200_conv_epilogue *epi,
                            void *stream_) {
  if (n_out == 0) return MEB200_OK;
  MEB_CHECK_ARG(out_dtype >= 0 && out_dtype <= 2, "output dtype");
  MEB_CHECK_ARG(out && w_t_e4m3 && a_scale && out_nbr && (in_e4m3 || n_in == 0), "null buffer");
  MEB_CHECK_ARG(K > 0, "empty kernel");
  MEB_CHECK_ARG(epi != nullptr && epilogue_ok(epi),
                "epilogue required: scale and shift, 8-byte aligned pointers");
  if (!conv_fp8_supported(c_in, c_out)) {
    set_error("fp8 forward: c_in=%u c_out=%u outside the e4m3 grid", c_in, c_out);
    return MEB200_ERR_UNSUPPORTED;
  }
  return conv_forward_tc(in_e4m3, kOperandE4M3, n_in, c_in, w_t_e4m3, K, c_out, out_nbr, out_order,
                         n_out, out, out_dtype, epi, (cudaStream_t)stream_, a_scale);
}

int meb200_conv_forward_fp8_q(const void *in_e4m3, const float *a_scale, uint32_t n_in,
                              uint32_t c_in, const void *w_t_e4m3, uint32_t K, uint32_t c_out,
                              const int32_t *out_nbr, uint32_t n_out, void *out, int out_dtype,
                              const int32_t *out_order, const meb200_conv_epilogue *epi, void *q,
                              const float *q_scale, void *stream_) {
  if (n_out == 0) return MEB200_OK;
  MEB_CHECK_ARG(out_dtype >= 0 && out_dtype <= 2, "output dtype");
  MEB_CHECK_ARG(out && w_t_e4m3 && a_scale && out_nbr && q && q_scale && (in_e4m3 || n_in == 0),
                "null buffer");
  MEB_CHECK_ARG(K > 0, "empty kernel");
  MEB_CHECK_ARG(epi != nullptr && epilogue_ok(epi),
                "epilogue required: scale and shift, 8-byte aligned pointers");
  if (!conv_fp8_supported(c_in, c_out)) {
    set_error("fp8 forward: c_in=%u c_out=%u outside the e4m3 grid", c_in, c_out);
    return MEB200_ERR_UNSUPPORTED;
  }
  const Shadow sh{reinterpret_cast<uint8_t *>(q), q_scale};
  return conv_forward_tc(in_e4m3, kOperandE4M3, n_in, c_in, w_t_e4m3, K, c_out, out_nbr, out_order,
                         n_out, out, out_dtype, epi, (cudaStream_t)stream_, a_scale, &sh);
}

int meb200_conv_pack_weights_e4m3(const float *weight, uint32_t K, uint32_t c_in, uint32_t c_out,
                                  void *w_t_e4m3, float *w_scale, void *stream_) {
  MEB_CHECK_ARG(weight && w_t_e4m3 && w_scale, "null buffer");
  MEB_CHECK_ARG(c_in > 0 && c_out > 0 && K > 0, "empty channel/kernel dims");
  return conv_pack_weights_e4m3(weight, K, c_in, c_out, w_t_e4m3, w_scale, (cudaStream_t)stream_);
}

uint64_t meb200_quantize_e4m3_workspace_bytes(void) { return quantize_e4m3_workspace_bytes(); }

int meb200_quantize_e5m2(const void *in, int dtype, uint32_t n, uint32_t c, void *out_e5m2,
                         float *scale_dev, void *workspace, void *stream_) {
  MEB_CHECK_ARG(dtype >= 0 && dtype <= 2, "dtype");
  MEB_CHECK_ARG(out_e5m2 && scale_dev && workspace && (in || (uint64_t)n * c == 0), "null buffer");
  return quantize_e5m2(in, dtype, (uint64_t)n * c, out_e5m2, scale_dev, workspace,
                       (cudaStream_t)stream_);
}

int meb200_conv_pack_weights_e4m3_dgrad(const float *weight, uint32_t K, uint32_t c_in,
                                        uint32_t c_out, void *w_e4m3, float *w_scale,
                                        void *stream_) {
  MEB_CHECK_ARG(weight && w_e4m3 && w_scale, "null buffer");
  MEB_CHECK_ARG(c_in > 0 && c_out > 0 && K > 0, "empty channel/kernel dims");
  return conv_pack_weights_e4m3_dgrad(weight, K, c_in, c_out, w_e4m3, w_scale,
                                      (cudaStream_t)stream_);
}

// The forward kernel on the transposed table, as meb200_conv_backward's dgrad, with e5m2 gradients
// against e4m3 weights [K, c_in, c_out]; the epilogue is the weight scale of each column alone.
int meb200_conv_dgrad_fp8(const void *grad_e5m2, const float *g_scale, uint32_t n_out,
                          uint32_t c_out, const void *w_e4m3, const float *w_scale, uint32_t K,
                          uint32_t c_in, const int32_t *in_nbr, uint32_t n_in, void *grad_in,
                          int grad_in_dtype, const int32_t *in_order, void *stream_) {
  if (n_in == 0) return MEB200_OK;
  MEB_CHECK_ARG(grad_in_dtype >= 0 && grad_in_dtype <= 2, "grad_in dtype");
  MEB_CHECK_ARG(grad_in && w_e4m3 && w_scale && g_scale && in_nbr && (grad_e5m2 || n_out == 0),
                "null buffer");
  MEB_CHECK_ARG(K > 0, "empty kernel");
  MEB_CHECK_ARG(aligned(8, w_scale), "w_scale must be 8-byte aligned");
  if (!conv_fp8_supported(c_out, c_in)) {
    set_error("fp8 dgrad: c_out=%u c_in=%u outside the e4m3 grid", c_out, c_in);
    return MEB200_ERR_UNSUPPORTED;
  }
  const meb200_conv_epilogue epi{w_scale, nullptr, nullptr, 0};
  return conv_forward_tc(grad_e5m2, kOperandE5M2E4M3, n_out, c_out, w_e4m3, K, c_in, in_nbr,
                         in_order, n_in, grad_in, grad_in_dtype, &epi, (cudaStream_t)stream_,
                         g_scale);
}

int meb200_conv_wgrad_fp8_supported(uint32_t c_in, uint32_t c_out, uint32_t K) {
  return conv_wgrad_fp8_supported(c_in, c_out, K) ? 1 : 0;
}

uint64_t meb200_conv_wgrad_fp8_workspace_bytes(uint32_t n_out, uint32_t c_in, uint32_t c_out,
                                               uint32_t K) {
  return conv_wgrad_workspace_bytes(c_in, c_out, K, n_out);
}

int meb200_conv_wgrad_fp8(const void *in_e4m3, const float *a_scale, const void *grad_e5m2,
                          const float *g_scale, uint32_t c_in, uint32_t K, uint32_t c_out,
                          const int32_t *pairs_in, const int32_t *pairs_out,
                          const int32_t *seg_start, uint32_t n_chunks, uint32_t n_out,
                          float *grad_weight, void *workspace, uint64_t workspace_bytes,
                          void *stream_) {
  MEB_CHECK_ARG(grad_weight && a_scale && g_scale, "null buffer");
  MEB_CHECK_ARG(n_out == 0 || (in_e4m3 && grad_e5m2 && pairs_in && pairs_out && seg_start &&
                               n_chunks > 0),
                "null buffer");
  return conv_wgrad_fp8(in_e4m3, a_scale, grad_e5m2, g_scale, c_in, K, c_out, pairs_in, pairs_out,
                        seg_start, n_chunks, n_out, grad_weight, workspace, workspace_bytes,
                        (cudaStream_t)stream_);
}

int meb200_quantize_e4m3(const void *in, int dtype, uint32_t n, uint32_t c, void *out_e4m3,
                         float *scale_dev, void *workspace, void *stream_) {
  MEB_CHECK_ARG(dtype >= 0 && dtype <= 2, "dtype");
  MEB_CHECK_ARG(out_e4m3 && scale_dev && workspace && (in || (uint64_t)n * c == 0), "null buffer");
  return quantize_e4m3(in, dtype, (uint64_t)n * c, out_e4m3, scale_dev, workspace,
                       (cudaStream_t)stream_);
}

int meb200_amax_accumulate(const void *in, int dtype, uint32_t n, uint32_t c, float *amax_dev,
                           void *stream_) {
  MEB_CHECK_ARG(dtype >= 0 && dtype <= 2, "dtype");
  MEB_CHECK_ARG(amax_dev && (in || (uint64_t)n * c == 0), "null buffer");
  return amax_accumulate(in, dtype, (uint64_t)n * c, amax_dev, (cudaStream_t)stream_);
}

int meb200_e4m3_scales(const float *amax_dev, float *scale_dev, void *stream_) {
  MEB_CHECK_ARG(amax_dev && scale_dev, "null buffer");
  return e4m3_scales_from_amax(amax_dev, scale_dev, (cudaStream_t)stream_);
}

int meb200_quantize_e4m3_static(const void *in, int dtype, uint32_t n, uint32_t c, void *out_e4m3,
                                const float *scale_dev, void *stream_) {
  MEB_CHECK_ARG(dtype >= 0 && dtype <= 2, "dtype");
  MEB_CHECK_ARG(out_e4m3 && scale_dev && (in || (uint64_t)n * c == 0), "null buffer");
  return quantize_e4m3_static(in, dtype, (uint64_t)n * c, out_e4m3, scale_dev,
                              (cudaStream_t)stream_);
}

static bool packed_dtype(int dtype) {
  return dtype == MEB200_BF16 || dtype == MEB200_F16 || dtype == MEB200_TF32;
}

int meb200_conv_pack_weights(const float *weight, uint32_t K, uint32_t c_in, uint32_t c_out,
                             int dtype, void *w_cast, void *w_t, void *stream_) {
  MEB_CHECK_ARG(packed_dtype(dtype), "packed weights are bf16, fp16 or tf32");
  MEB_CHECK_ARG(weight && w_cast && w_t, "null buffer");
  MEB_CHECK_ARG(c_in > 0 && c_out > 0 && K > 0 && K <= 65535, "empty channel/kernel dims");
  return conv_pack_weights(weight, K, c_in, c_out, dtype, w_cast, w_t, (cudaStream_t)stream_);
}

static_assert(sizeof(meb200_pack_job) == sizeof(PackJob), "meb200_pack_job layout");

int meb200_conv_pack_weights_batched(const meb200_pack_job *jobs_dev, uint32_t n_jobs,
                                     uint32_t total_tiles, int dtype, void *stream_) {
  MEB_CHECK_ARG(packed_dtype(dtype), "packed weights are bf16, fp16 or tf32");
  MEB_CHECK_ARG(jobs_dev != nullptr || n_jobs == 0, "null job table");
  return conv_pack_weights_batched(reinterpret_cast<const PackJob *>(jobs_dev), n_jobs, total_tiles,
                                   dtype, (cudaStream_t)stream_);
}

uint32_t meb200_conv_stem_virtual_channels(uint32_t K) { return 4u * ((K + 15u) / 16u * 16u); }

int meb200_conv_stem_supported(int dtype, uint32_t K, uint32_t c_out) {
  return conv_stem_tc_supported(dtype, K, c_out) && conv_stem_wgrad_tc_supported(dtype, K, c_out) ? 1 : 0;
}

int meb200_conv_stem_forward(const void *in4, int dtype, uint32_t K, const void *weight_v,
                             uint32_t c_out, const int32_t *out_nbr, uint32_t n_out, void *out,
                             int out_dtype, const meb200_conv_epilogue *epi, void *stream_) {
  if (n_out == 0) return MEB200_OK;
  MEB_CHECK_ARG(out_dtype == MEB200_F32 || out_dtype == dtype, "output dtype must be fp32 or the input dtype");
  MEB_CHECK_ARG(in4 && weight_v && out_nbr && out, "null buffer");
  MEB_CHECK_ARG(epilogue_ok(epi), "epilogue: scale and shift required, 8-byte aligned pointers");
  if (!conv_stem_tc_supported(dtype, K, c_out)) {
    set_error("stem forward: shape/dtype outside the tensor-core path (K=%u c_out=%u)", K, c_out);
    return MEB200_ERR_UNSUPPORTED;
  }
  return conv_stem_forward_tc(in4, dtype, K, weight_v, c_out, out_nbr, n_out, out, out_dtype, epi,
                              (cudaStream_t)stream_);
}

int meb200_conv_stem_forward_q(const void *in4, int dtype, uint32_t K, const void *weight_v,
                               uint32_t c_out, const int32_t *out_nbr, uint32_t n_out, void *out,
                               int out_dtype, const meb200_conv_epilogue *epi, void *q,
                               const float *q_scale, void *stream_) {
  if (n_out == 0) return MEB200_OK;
  MEB_CHECK_ARG(out_dtype == MEB200_F32 || out_dtype == dtype, "output dtype must be fp32 or the input dtype");
  MEB_CHECK_ARG(in4 && weight_v && out_nbr && out && q && q_scale, "null buffer");
  MEB_CHECK_ARG(epi != nullptr && epilogue_ok(epi),
                "epilogue required: scale and shift, 8-byte aligned pointers");
  if (!conv_stem_tc_supported(dtype, K, c_out)) {
    set_error("stem forward: shape/dtype outside the tensor-core path (K=%u c_out=%u)", K, c_out);
    return MEB200_ERR_UNSUPPORTED;
  }
  const Shadow sh{reinterpret_cast<uint8_t *>(q), q_scale};
  return conv_stem_forward_tc(in4, dtype, K, weight_v, c_out, out_nbr, n_out, out, out_dtype, epi,
                              (cudaStream_t)stream_, &sh);
}

int meb200_conv_stem_wgrad(const void *in4, const void *grad_out, int dtype, uint32_t K,
                           uint32_t c_out, const int32_t *out_nbr, uint32_t n_out,
                           float *grad_weight_v, void *workspace, uint64_t workspace_bytes,
                           void *stream_) {
  MEB_CHECK_ARG(grad_weight_v && (n_out == 0 || (in4 && grad_out && out_nbr)), "null buffer");
  if (!conv_stem_wgrad_tc_supported(dtype, K, c_out)) {
    set_error("stem wgrad: shape/dtype outside the tensor-core path (K=%u c_out=%u)", K, c_out);
    return MEB200_ERR_UNSUPPORTED;
  }
  return conv_stem_wgrad_tc(in4, grad_out, dtype, K, c_out, out_nbr, n_out, grad_weight_v,
                            workspace, workspace_bytes, (cudaStream_t)stream_);
}

int meb200_conv_backward(const void *in, const void *grad_out, int dtype, uint32_t n_in,
                         uint32_t c_in, const void *w_cast, uint32_t K, uint32_t c_out,
                         const int32_t *out_nbr, const int32_t *in_nbr, uint32_t n_out,
                         void *grad_in, int grad_in_dtype, float *grad_weight,
                         const int32_t *pairs_in, const int32_t *pairs_out,
                         const int32_t *seg_start, uint32_t n_chunks, void *workspace,
                         uint64_t workspace_bytes, const int32_t *in_order, void *stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  MEB_CHECK_ARG(dtype >= 0 && dtype <= 3, "dtype");
  MEB_CHECK_ARG(grad_in_dtype == MEB200_F32 || grad_in_dtype == dtype,
                "grad_in dtype must be fp32 or the feature dtype");
  MEB_CHECK_ARG(grad_in_dtype != MEB200_TF32, "grad_in of a TF32 convolution is fp32");
  const int fdt = storage_dtype(dtype);         // the CUDA-core kernels: exact fp32 for TF32
  MEB_CHECK_ARG(c_in > 0 && c_out > 0 && K > 0, "empty channel/kernel dims");
  if (grad_in != nullptr && n_in > 0) {
    MEB_CHECK_ARG(in_nbr && w_cast && (grad_out || n_out == 0), "null buffer");
    // dgrad = the forward kernel on the transposed table with W_k^T:
    // rows = input rows, reduction over c_out, produces c_in columns.
    int rc = MEB200_ERR_UNSUPPORTED;
    if (conv_tc_supported(dtype, c_out, c_in))
      rc = conv_forward_tc(grad_out, dtype, n_out, c_out, w_cast, K, c_in, in_nbr, in_order, n_in,
                           grad_in, grad_in_dtype, nullptr, stream);
    if (rc == MEB200_ERR_UNSUPPORTED)
      rc = conv_forward_simt(grad_out, fdt, n_out, c_out, w_cast, K, c_in, /*trans_w=*/true,
                             in_nbr, n_in, grad_in, grad_in_dtype, nullptr, stream);
    if (rc != MEB200_OK) return rc;
  }
  if (grad_weight != nullptr) {
    // an empty output map's table [K, 0] may be a null pointer: its weight gradient is zero
    MEB_CHECK_ARG((out_nbr || n_out == 0) && (in || n_in == 0) && (grad_out || n_out == 0),
                  "null buffer");
    if (pairs_in && pairs_out && seg_start && n_chunks > 0 &&
        conv_wgrad_uses_pairs(dtype, c_in, c_out, K)) {
      int rc = conv_wgrad_pairs(in, grad_out, dtype, c_in, K, c_out, pairs_in, pairs_out,
                                seg_start, n_chunks, n_out, grad_weight, workspace,
                                workspace_bytes, stream);
      if (rc != MEB200_ERR_UNSUPPORTED) return rc;
    }
    if (conv_wgrad_tc_supported(dtype, c_in, c_out)) {
      int rc = conv_wgrad_tc(in, grad_out, dtype, c_in, K, c_out, out_nbr, n_out, grad_weight,
                             workspace, workspace_bytes, stream);
      if (rc != MEB200_ERR_UNSUPPORTED) return rc;
    }
    if (conv_small_cin_supported(c_in, c_out))
      return conv_small_cin_wgrad(in, grad_out, fdt, c_in, K, c_out, out_nbr, n_out,
                                  grad_weight, workspace, workspace_bytes, stream);
    return conv_wgrad_simt(in, grad_out, fdt, c_in, K, c_out, out_nbr, n_out, grad_weight,
                           workspace, workspace_bytes, stream);
  }
  return MEB200_OK;
}

}
