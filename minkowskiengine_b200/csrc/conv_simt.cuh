// SIMT (CUDA-core, fp32-accumulate) sparse convolution kernels: the exact-fp32 parity
// path and the fallback for channel counts the wgmma path does not take.
#pragma once
#include "common.cuh"

namespace meb200 {

// epi (may be NULL; forward only, trans_w = false): the epilogue of meb200_conv_epilogue.
int conv_forward_simt(const void *in, int in_dtype, uint32_t n_in, uint32_t c_in,
                      const void *weight, uint32_t K, uint32_t c_out, bool trans_w,
                      const int32_t *nbr, uint32_t n_out, void *out, int out_dtype,
                      const meb200_conv_epilogue *epi, cudaStream_t stream);

// Weight gradients reduce over row splits (workspace_splits / launch_split_sum in common.cuh).
// The size below fits every split the plan wants, for the kernel conv_small_cin_supported()
// selects.
uint64_t conv_wgrad_simt_workspace_bytes(uint32_t c_in, uint32_t c_out, uint32_t K,
                                         uint32_t n_out);
int conv_wgrad_simt(const void *in, const void *grad_out, int dtype, uint32_t c_in,
                    uint32_t K, uint32_t c_out, const int32_t *out_nbr, uint32_t n_out,
                    float *grad_weight, void *workspace, uint64_t workspace_bytes,
                    cudaStream_t stream);

// Stem layers (c_in <= 4, c_out <= 64): table-scan bound kernels, any feature dtype.
bool conv_small_cin_supported(uint32_t c_in, uint32_t c_out);
int conv_small_cin_forward(const void *in, int in_dtype, uint32_t c_in, const void *W, uint32_t K,
                           uint32_t c_out, const int32_t *nbr, uint32_t n_out, void *out,
                           int out_dtype, const meb200_conv_epilogue *epi, cudaStream_t stream);
int conv_small_cin_wgrad(const void *in, const void *grad_out, int dtype, uint32_t c_in, uint32_t K,
                         uint32_t c_out, const int32_t *out_nbr, uint32_t n_out, float *grad_weight,
                         void *workspace, uint64_t workspace_bytes, cudaStream_t stream);

}  // namespace meb200
