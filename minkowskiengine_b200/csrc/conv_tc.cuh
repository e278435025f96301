// Tensor-core sparse convolution kernels: bf16/fp16 operands, or fp32 ones multiplied in TF32
// (MEB200_TF32), fp32 accumulation.
#pragma once
#include "common.cuh"

namespace meb200 {

// bf16/fp16/TF32 operands with channel counts the tiles cover.
bool conv_tc_supported(int dtype, uint32_t c_reduce, uint32_t c_cols);

// Operand code of the e4m3 forward (internal: not a feature dtype of the ABI).  Grid: whole 32-byte
// k-steps of the reduction, output columns in multiples of 16.
constexpr int kOperandE4M3 = 100;
// Operand pair of the fp8 dgrad: A e5m2 (the gradient), B e4m3 (the weights); the same grid.  The
// kernel multiplies column c by epi->scale[c] after *a_scale and runs no other epilogue.
constexpr int kOperandE5M2E4M3 = 101;
bool conv_fp8_supported(uint32_t c_in, uint32_t c_out);
bool conv_wgrad_tc_supported(int dtype, uint32_t c_in, uint32_t c_out);

// The shadow of a forward (the _q entries of include/meb200.h): q [n_rows, c_cols] e4m3 bytes of the
// stored output at the scale q_scale (device fp32 [2]: scale, inv) of the layer it feeds.
struct Shadow {
  uint8_t *q;
  const float *q_scale;
};

// out[r,:] = sum_k A[nbr[k][r],:] @ B[k]^T with B [K, c_cols, c_reduce] (reduction contiguous):
// the forward passes w_t [K, c_out, c_in], the dgrad the layer's w_cast [K, c_in, c_out].
// order (may be NULL; read when K <= 32): the tile order of nbr from meb200_kernel_map, so that
// each 128-row tile runs only the offsets its rows reach.  epi (may be NULL): the forward's
// epilogue (meb200_conv_epilogue); the dgrad passes NULL.
// dtype kOperandE4M3: A and B are e4m3 bytes, out_dtype bf16 / fp16 / fp32, and the epilogue
// (required) runs on the accumulator times *a_scale (a device pointer).
// shadow (may be NULL; bf16 / fp16 / e4m3 operands with an epilogue): also write the shadow.
int conv_forward_tc(const void *A, int dtype, uint32_t n_a, uint32_t c_reduce, const void *B,
                    uint32_t K, uint32_t c_cols, const int32_t *nbr, const int32_t *order,
                    uint32_t n_rows, void *out, int out_dtype, const meb200_conv_epilogue *epi,
                    cudaStream_t stream, const float *a_scale = nullptr,
                    const Shadow *shadow = nullptr);

// fp32 W [K, c_in, c_out] -> w_t [K, c_out, c_in] in e4m3 with a scale per output channel:
// w_scale[c] = amax_c / 448 (1 when amax_c = 0), w_t = satfinite_rn(W * (448 / amax_c)).
int conv_pack_weights_e4m3(const float *W, uint32_t K, uint32_t c_in, uint32_t c_out, void *w_t,
                           float *w_scale, cudaStream_t stream);

// fp32 W [K, c_in, c_out] -> w_c [K, c_in, c_out] in e4m3 with a scale per input channel (the
// dgrad's output column), amax over (k, co), by the formula of conv_pack_weights_e4m3.
int conv_pack_weights_e4m3_dgrad(const float *W, uint32_t K, uint32_t c_in, uint32_t c_out,
                                 void *w_c, float *w_scale, cudaStream_t stream);

// Per-tensor e4m3 / e5m2 quantisation of [n, c] features (meb200_quantize_e4m3 / _e5m2); both
// use the same zero-filled workspace.
uint64_t quantize_e4m3_workspace_bytes();
int quantize_e4m3(const void *in, int dtype, uint64_t count, void *out, float *scale, void *workspace,
                  cudaStream_t stream);
int quantize_e5m2(const void *in, int dtype, uint64_t count, void *out, float *scale, void *workspace,
                  cudaStream_t stream);
// Static scales (meb200_amax_accumulate, meb200_e4m3_scales, meb200_quantize_e4m3_static).
int amax_accumulate(const void *in, int dtype, uint64_t count, float *amax, cudaStream_t stream);
int e4m3_scales_from_amax(const float *amax, float *scale, cudaStream_t stream);
int quantize_e4m3_static(const void *in, int dtype, uint64_t count, void *out, const float *scale,
                         cudaStream_t stream);

// fp32 W[K,c_in,c_out] -> w_cast [K,c_in,c_out] and w_t [K,c_out,c_in] in bf16/fp16, or in fp32
// words rounded to tf32 (MEB200_TF32).
int conv_pack_weights(const float *W, uint32_t K, uint32_t c_in, uint32_t c_out, int dtype,
                      void *w_cast, void *w_t, cudaStream_t stream);

// One job of conv_pack_weights_batched == one meb200_pack_job of include/meb200.h.
struct PackJob {
  const void *w;                      // fp32 [K, c_in, c_out]
  void *w_cast, *w_t;                 // as conv_pack_weights
  uint32_t K, c_in, c_out;
  uint32_t tile_begin;                // first 32x32 tile of this job in the launch
};
int conv_pack_weights_batched(const PackJob *jobs_dev, uint32_t n_jobs, uint32_t total_tiles,
                              int dtype, cudaStream_t stream);

int conv_wgrad_tc(const void *in, const void *grad_out, int dtype, uint32_t c_in, uint32_t K,
                  uint32_t c_out, const int32_t *out_nbr, uint32_t n_out, float *grad_weight,
                  void *workspace, uint64_t workspace_bytes, cudaStream_t stream);

// Bytes of workspace that let wgrad over n_out rows use all its planned row splits (0: one split).
// With less (or none) it uses fewer splits.  For a given workspace size the result never depends
// on the order in which CTAs finish (the splits' partial sums are added in a fixed order).
uint64_t conv_wgrad_workspace_bytes(uint32_t c_in, uint32_t c_out, uint32_t K, uint32_t n_out);

// wgrad over the compacted pair lists of meb200_kernel_map_pairs (meb200_conv_wgrad_uses_pairs).
bool conv_wgrad_uses_pairs(int dtype, uint32_t c_in, uint32_t c_out, uint32_t K);
int conv_wgrad_pairs(const void *in, const void *grad_out, int dtype, uint32_t c_in, uint32_t K,
                     uint32_t c_out, const int32_t *pairs_in, const int32_t *pairs_out,
                     const int32_t *seg_start, uint32_t n_chunks, uint32_t n_out,
                     float *grad_weight, void *workspace, uint64_t workspace_bytes,
                     cudaStream_t stream);

// fp8 wgrad over the pair lists (meb200_conv_wgrad_fp8): e4m3 input and e5m2 output gradient, each
// with its device dequantisation factor; c_in and c_out multiples of 32 up to 1024, K <= 1023.
// Its row splits are those of conv_wgrad_pairs (conv_wgrad_workspace_bytes covers them).
bool conv_wgrad_fp8_supported(uint32_t c_in, uint32_t c_out, uint32_t K);
int conv_wgrad_fp8(const void *in, const float *a_scale, const void *grad_out,
                   const float *g_scale, uint32_t c_in, uint32_t K, uint32_t c_out,
                   const int32_t *pairs_in, const int32_t *pairs_out, const int32_t *seg_start,
                   uint32_t n_chunks, uint32_t n_out, float *grad_weight, void *workspace,
                   uint64_t workspace_bytes, cudaStream_t stream);

// ---- network stem: rows of <= 4 channels, padded to 4 (8 bytes) ------------------------------
// The layer is run as a K = 1 convolution over 4 * 16 ceil(K / 16) VIRTUAL channels (offset k,
// channel c) -> 4 k + c, by the forward and wgrad kernels in their stem mode.
bool conv_stem_tc_supported(int dtype, uint32_t K, uint32_t c_cols);
int conv_stem_forward_tc(const void *A4, int dtype, uint32_t K, const void *Wv, uint32_t c_cols,
                         const int32_t *nbr, uint32_t n_rows, void *out, int out_dtype,
                         const meb200_conv_epilogue *epi, cudaStream_t stream,
                         const Shadow *shadow = nullptr);
bool conv_stem_wgrad_tc_supported(int dtype, uint32_t K, uint32_t c_out);
int conv_stem_wgrad_tc(const void *in4, const void *grad_out, int dtype, uint32_t K,
                       uint32_t c_out, const int32_t *nbr, uint32_t n_rows, float *dWv,
                       void *workspace, uint64_t workspace_bytes, cudaStream_t stream);

}  // namespace meb200
