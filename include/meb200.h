/*
 * meb200.h — C ABI of the H100-native (sm_90a) sparse-convolution hot path.
 *
 * Every entry point is `extern "C"`, takes plain device pointers + sizes + the CUDA
 * stream to launch on (as `void*`, i.e. a cudaStream_t), allocates nothing the caller
 * did not hand in, and returns 0 on success or a negative MEB200_ERR_* code; the text
 * of the last failure on the calling thread is available from meb200_last_error().
 * No torch / C++ types appear in any signature.
 *
 * These are the calls the reference's FFI for this path would bind.  The reference's
 * boundary is the pybind module `MinkowskiEngineBackend._C` (pybind/extern.hpp); each
 * function below names the reference interface it stands in for.  The Python host in
 * `minkowskiengine_b200/` binds them through ctypes (see INTEGRATION.md).
 *
 * Conventions
 *   coords      int32 [n, ncols] row-major, ncols = D+1, column 0 = batch index
 *               (reference: src/coordinate.hpp:36-61, MinkowskiSparseTensor.py:293-345)
 *   table       uint32 [capacity] open-addressing hash table of ROW INDICES into the
 *               coords array it was built over (0xFFFFFFFF = empty); capacity is a
 *               power of two from meb200_hash_capacity()
 *   nbr tables  int32 [K, n] "neighbour tables", k-major: nbr[k*n + r] = the row on
 *               the other side reached from row r through kernel offset k, or -1
 *   features    [n, C] row-major; dtype codes MEB200_F32 / MEB200_BF16 / MEB200_F16
 *   weights     [K, Cin, Cout] row-major (reference: MinkowskiConvolution.py:264-279)
 */
#ifndef MEB200_H_
#define MEB200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MEB200_OK 0
#define MEB200_ERR_INVALID (-1) /* bad argument (shape, dtype, null pointer)        */
#define MEB200_ERR_CUDA (-2)    /* a CUDA runtime call or kernel launch failed      */
#define MEB200_ERR_UNSUPPORTED (-3) /* valid request this build has no kernel for   */

#define MEB200_F32 0
#define MEB200_BF16 1
#define MEB200_F16 2
/* fp32 storage, TF32 tensor-core math: the operand code of an fp32 convolution whose caller allows
 * TF32 (torch.backends.cuda.matmul.fp32_precision == "tf32").  Accepted by meb200_conv_forward,
 * meb200_conv_backward, the weight packing calls, meb200_conv_workspace_bytes and
 * meb200_conv_wgrad_uses_pairs; features, outputs and grad_in are fp32 (outputs and grad_in
 * MEB200_F32).  Rounding: the packed weights are rounded to tf32 (10 explicit mantissa bits) to
 * nearest, ties away from zero; features and gradients are read as stored and the tensor cores
 * truncate them to tf32 (observed on the H100); products are accumulated in fp32.  Grid: forward and dgrad run on the
 * tensor cores when the reduction width (c_in forward, c_out dgrad) is a multiple of 8 and the
 * output width a multiple of 16 and <= 1024; the weight gradient when c_in is a multiple of 8
 * (>= 16) and c_out a multiple of 16 in [16, 256].  Any other shape runs the fp32 CUDA-core
 * kernels (on the packed, tf32-rounded weights in forward and dgrad). */
#define MEB200_TF32 3

#define MEB200_MAX_NCOLS 8 /* D+1 <= 8, i.e. up to 7 spatial/temporal axes */

#define MEB200_POOL_SUM 0 /* reference PoolingMode::LOCAL_SUM_POOLING (src/types.hpp:141) */
#define MEB200_POOL_AVG 1 /* LOCAL_AVG_POOLING */
#define MEB200_POOL_MAX 2 /* LOCAL_MAX_POOLING */

/* ---- library ---------------------------------------------------------------------- */
const char *meb200_last_error(void);
/* Compile-time facts: "sm_90a", CUDA runtime version the library was built with.      */
const char *meb200_build_arch(void);
int meb200_cudart_version(void); /* reference: cudart_version(), pybind/extern.hpp:808-838 */
/* Number of kernels this library has launched since load (bench.py's gpu_launches).   */
uint64_t meb200_launch_count(void);
/* ... of which launches of the wgmma (tensor-core) convolution kernels. */
uint64_t meb200_tc_launch_count(void);

/* ---- coordinate hashing (reference a1/a2: src/coordinate.hpp:223-349,
 *      CoordinateMapCPU::insert_and_map coordinate_map_cpu.hpp:353-380,
 *      CoordinateMapGPU::insert coordinate_map_gpu.cu:196-278) ------------------------ */

/* Table capacity (power of two) used for n keys. */
uint32_t meb200_hash_capacity(uint32_t n);

/* Bytes of scratch the dedup pipeline needs for n candidate rows. */
uint64_t meb200_insert_scratch_bytes(uint32_t n);

/*
 * Deduplicating insert with the CPU reference's semantics: among equal coordinates the
 * FIRST row (smallest index) wins and unique rows are numbered by the rank of their
 * first occurrence.
 *   coords        [n, ncols] candidates          valid   optional uint8[n] (NULL = all)
 *   table         [capacity] out, built over `unique_coords` (row ids are NEW ids)
 *   unique_coords [n, ncols] out (first *h_num_unique rows are meaningful)
 *   unique_index  int64 [n] out: original row of each unique row (first m meaningful)
 *   inverse_map   int64 [n] out: new row id of every candidate (-1 where !valid)
 *   scratch       meb200_insert_scratch_bytes(n) bytes
 *   h_num_unique  HOST pointer; written after a stream synchronise (the one blocking
 *                 point of map construction: the caller needs m to size tensors).
 */
int meb200_insert_and_map(const int32_t *coords, const uint8_t *valid, uint32_t n,
                          uint32_t ncols, uint32_t *table, uint32_t capacity,
                          int32_t *unique_coords, int64_t *unique_index,
                          int64_t *inverse_map, void *scratch, uint32_t *h_num_unique,
                          void *stream);
/* The same insert WITHOUT the blocking count read, for maps that can be enqueued before they
 * are needed (the stride pyramid of a network: every level is a function of the input
 * coordinates alone, reference call sites coordinate_map_manager.cpp:406-429).  `n` is an UPPER
 * bound of the candidate count; `d_n` (device, may be NULL = all n) holds the actual count, so
 * a level can be enqueued while its parent's size is still only known on the device.  The unique
 * count is left in `d_num_unique` (DEVICE); `table` is dedup scratch here — build the real table
 * over the first m unique rows with meb200_map_build_table once m is known on the host.
 * Row numbering is identical to meb200_insert_and_map (rows past *d_n never win). */
int meb200_insert_and_map_enqueue(const int32_t *coords, const uint8_t *valid,
                                  const uint32_t *d_n, uint32_t n, uint32_t ncols,
                                  uint32_t *table, uint32_t capacity, int32_t *unique_coords,
                                  int64_t *unique_index, int64_t *inverse_map, void *scratch,
                                  uint32_t *d_num_unique, void *stream);
/* Row-index table over m DISTINCT coordinate rows (what meb200_insert_and_map leaves in `table`). */
int meb200_map_build_table(const int32_t *unique_coords, uint32_t m, uint32_t ncols,
                           uint32_t *table, uint32_t capacity, void *stream);

/* Candidate generation for a strided map: out[i] = floor(c / ts_out) * ts_out per
 * spatial axis, batch kept (reference a3: detail::stride_coordinate
 * src/coordinate_map.hpp:58-76 — integer floor division here, see DESIGN.md).
 * out_tensor_stride: HOST int32[ncols-1]. */
int meb200_stride_coords(const int32_t *coords, uint32_t n, uint32_t ncols,
                         const int32_t *out_tensor_stride, int32_t *out, void *stream);

/* Candidate generation for stride_region (reference: CoordinateMapCPU::stride_region
 * coordinate_map_cpu.hpp:446-487): out[(i*K + k)] = coords[i] + offsets[k]; when
 * `aligned_only` != 0 candidates not aligned to out_tensor_stride get valid = 0.
 * offsets: DEVICE int32 [K, ncols-1]; out_tensor_stride: HOST int32[ncols-1]. */
int meb200_region_coords(const int32_t *coords, uint32_t n, uint32_t ncols,
                         const int32_t *offsets, uint32_t K,
                         const int32_t *out_tensor_stride, int aligned_only,
                         int32_t *out, uint8_t *valid, void *stream);

/* Batch lookup: result[i] = row of query[i] in the map, or -1
 * (reference: CoordinateMapCPU::find coordinate_map_cpu.hpp:388-412). */
int meb200_map_find(const int32_t *map_coords, const uint32_t *table, uint32_t capacity,
                    uint32_t ncols, const int32_t *query, uint32_t nq, int32_t *result,
                    void *stream);

/* ---- kernel map (reference a4/a5: kernel_region::coordinate_at kernel_region.hpp:198-247,
 *      CoordinateMapCPU::kernel_map coordinate_map_cpu.hpp:569-670,
 *      CoordinateMapGPU::kernel_map coordinate_map_gpu.cu:1549-1745) ------------------ */
/*
 * For every row x of the iterated map X and every offset k: probe map Y at
 * X[x] + offsets[k].  x_nbr[k*nx + x] = y (or -1) and, when y_nbr != NULL,
 * y_nbr[k*ny + y] = x (y_nbr must be pre-filled with -1 by the caller).
 * offsets: DEVICE int32 [K, ncols-1] already scaled by dilation * tensor stride.
 * d_num_pairs: optional DEVICE uint32 counter, incremented by the number of hits.
 *
 * x_order / y_order (each may be NULL; K <= 32): the TILE ORDER of x_nbr / y_nbr, which
 * meb200_conv_forward / meb200_conv_backward read to run only the offsets a tile of 128 table rows
 * reaches.  The mask of row r has bit k set when nbr[k][r] >= 0; rows are stably sorted by mask
 * (ties keep row order), slot s holds row slot_row[s].  One int32 buffer of
 * (K + 1) * n + ceil(n / 128) words per table of n rows:
 *   [0, K n)             the table in slot order, k-major: [k][s] = nbr[k][slot_row[s]]
 *   [K n, (K + 1) n)     slot_row
 *   [(K + 1) n, ...)     uint32 mask of tile t = OR of the masks of slots [128 t, 128 t + 128)
 * Both orders asked for are written whenever K > 0, also when nx = 0 (y_nbr is then all -1 and
 * its order the identity with empty tile masks).
 * order_scratch: 4 * (2 m + 256 * ceil(m / 2048) + 256) bytes, m = the larger n of the orders
 * asked for (required when one is).  Deterministic: no atomics decide an order.
 */
int meb200_kernel_map(const int32_t *x_coords, uint32_t nx, const int32_t *y_coords,
                      uint32_t ny, const uint32_t *y_table, uint32_t y_capacity,
                      uint32_t ncols, const int32_t *offsets, uint32_t K, int32_t *x_nbr,
                      int32_t *y_nbr, uint32_t *d_num_pairs, int32_t *x_order, int32_t *y_order,
                      void *order_scratch, void *stream);

/* Compacted pair lists of a neighbour table — the reference's own kernel-map representation
 * (gpu_kernel_map::in_maps / out_maps per offset, src/kernel_map.cuh:48-429; what
 * CoordinateMapManager::kernel_map returns, coordinate_map_manager.cpp:662-823).  The table rows
 * are cut into chunks of `chunk_rows` rows (rounded up to a multiple of 2048; 0 = one chunk);
 * segment s = chunk * K + k holds, in table-row order, pairs_other[i] = nbr[k][r], pairs_row[i] = r
 * for the rows r of the chunk with nbr[k][r] >= 0 and occupies [seg_start[s], seg_start[s+1]),
 * padded with (-1, -1) to a multiple of `stage` entries.  Deterministic, no atomics, no host
 * synchronisation.  Buffers: pairs_* hold meb200_pair_list_capacity(...) int32 each, seg_start
 * meb200_pair_list_chunks(...) * K + 1 int32, scratch meb200_pair_list_scratch_bytes(...) bytes. */
uint32_t meb200_pair_list_chunks(uint32_t n_rows, uint32_t chunk_rows);
uint64_t meb200_pair_list_scratch_bytes(uint32_t K, uint32_t n_rows, uint32_t chunk_rows);
uint64_t meb200_pair_list_capacity(uint32_t K, uint32_t n_rows, uint32_t stage, uint32_t chunk_rows);
int meb200_kernel_map_pairs(const int32_t *nbr, uint32_t K, uint32_t n_rows, uint32_t stage,
                            uint32_t chunk_rows, int32_t *pairs_other, int32_t *pairs_row,
                            int32_t *seg_start, void *scratch, void *stream);

/* ---- sparse convolution (reference a8/a9/a10: ConvolutionForwardKernelCPU /
 *      ConvolutionBackwardKernelCPU src/convolution_kernel.hpp:33-144, GPU
 *      src/convolution_kernel.cu:114-496,553-757) ------------------------------------ */
/*
 * out[o,:] = sum_k in[out_nbr[k,o],:] @ W[k]          (rows with out_nbr = -1 skipped)
 * Output is fully written (no pre-zeroing needed, no atomics, deterministic).
 * in_dtype: dtype of `in`, `w_cast` and `w_t`; out_dtype: dtype of `out` (F32 always allowed).
 * TF32: fp32 `in`, `w_cast` and `w_t` from meb200_conv_pack_weights(..., MEB200_TF32, ...), F32 out.
 *   w_cast  [K, Cin, Cout]  the weights in the feature dtype
 *   w_t     [K, Cout, Cin]  the same, transposed per offset (BF16/F16/TF32: required; F32: not read)
 * Both come from meb200_conv_pack_weights.  The call runs the tensor cores on w_t when the shape
 * qualifies, otherwise the small-cin or SIMT kernels on w_cast.
 * out_order (may be NULL): the tile order of out_nbr from meb200_kernel_map; the tensor-core
 * kernel then runs only the offsets each tile of 128 output rows reaches (read when K <= 32).
 * epi (may be NULL): an epilogue every kernel applies to its fp32 accumulator before the one
 * conversion to out_dtype (see meb200_conv_epilogue); NULL writes the accumulator as it is.
 */
/* Per-channel affine map, residual and ReLU folded into a convolution's output (eval-mode batch
 * norm after a convolution): out[o, c] = relu?(acc[o, c] * scale[c] + shift[c] + residual[o, c]),
 * in fp32 (the product and shift as one fused multiply-add), rounded once to out_dtype.  A row
 * without neighbours has acc = 0.  Host struct; its pointers are device pointers. */
typedef struct meb200_conv_epilogue {
  const float *scale;                 /* [c_out] fp32 */
  const float *shift;                 /* [c_out] fp32 */
  const void *residual;               /* [n_out, c_out] in out_dtype, or NULL */
  int32_t relu;                       /* != 0: clamp at zero after the residual */
} meb200_conv_epilogue;
int meb200_conv_forward(const void *in, int in_dtype, uint32_t n_in, uint32_t c_in,
                        const void *w_cast, const void *w_t, uint32_t K, uint32_t c_out,
                        const int32_t *out_nbr, uint32_t n_out, void *out, int out_dtype,
                        const int32_t *out_order, const meb200_conv_epilogue *epi, void *stream);

/* grad_in[i,:] = sum_k grad_out[in_nbr[k,i],:] @ W[k]^T   (fully written)
 * grad_weight[k] = sum_o in[out_nbr[k,o],:]^T @ grad_out[o,:]   (fully written, fp32)
 * grad_in / grad_weight may be NULL to skip dgrad / wgrad; each picks its kernel on its own.
 * w_cast: [K, Cin, Cout] in the feature dtype.  pairs_in / pairs_out / seg_start (all three or
 * NULL) + n_chunks: the compacted pair lists of out_nbr from meb200_kernel_map_pairs with
 * stage = 64 and their chunk count; when meb200_conv_wgrad_uses_pairs() holds, the wgrad reduces
 * over them instead of the dense table.
 * workspace: meb200_conv_workspace_bytes(n_out, c_in, c_out, K, dtype) bytes, 16-byte aligned.
 * Every wgrad kernel stores its row splits' partial sums there and adds them in split order (no
 * atomics: bit-identical run to run).  It runs as many of its planned splits as the workspace
 * holds; less, NULL or unaligned is legal and means fewer splits, down to one.
 * in_order (may be NULL): the tile order of in_nbr from meb200_kernel_map, read by the tensor-core
 * dgrad as out_order by meb200_conv_forward. */
int meb200_conv_backward(const void *in, const void *grad_out, int dtype, uint32_t n_in,
                         uint32_t c_in, const void *w_cast, uint32_t K, uint32_t c_out,
                         const int32_t *out_nbr, const int32_t *in_nbr, uint32_t n_out,
                         void *grad_in, int grad_in_dtype, float *grad_weight,
                         const int32_t *pairs_in, const int32_t *pairs_out,
                         const int32_t *seg_start, uint32_t n_chunks, void *workspace,
                         uint64_t workspace_bytes, const int32_t *in_order, void *stream);

/* 1 when meb200_conv_backward's wgrad reads pair lists for this layer (so a caller builds them
 * only then), else 0. */
int meb200_conv_wgrad_uses_pairs(int dtype, uint32_t c_in, uint32_t c_out, uint32_t K);

/* Workspace of meb200_conv_backward and meb200_conv_stem_wgrad in any dtype: room for the row
 * splits of every wgrad kernel the call can pick (0: one split). */
uint64_t meb200_conv_workspace_bytes(uint32_t n_out, uint32_t c_in, uint32_t c_out, uint32_t K,
                                     int dtype);

/* ---- fp8 (e4m3) inference forward ----------------------------------------------------------
 * The eval forward of a convolution on the Hopper fp8 tensor cores: the features are quantised to
 * e4m3 with one scale per tensor, the weights with one scale per output channel, the products are
 * summed by the tensor cores and dequantised in the epilogue:
 *   out[o, c] = relu?(fma(acc[o, c] * a_scale, epi->scale[c], epi->shift[c]) [+ residual[o, c]])
 * with acc the sum of e4m3 products, rounded once to out_dtype (F32, BF16 or F16, the layer's
 * feature dtype).  epi->scale must include the weight scale: w_scale[c] times any per-channel
 * factor (eval batch norm).  Accumulation: the products of e4m3 values are exact, but the e4m3
 * tensor cores do not add them in fp32.  Modelled as keeping 13 fraction bits at each of the
 * n = K * c_in / 32 k-steps of 32 channels, an output errs by at most n * 2^-13 * A (A the same sum
 * over |products|); the worst measured on an H100 is about 2^-11.7 * A at K = 27, c_in = 384,
 * where the bf16 / fp16 kernels stay within 4 * 2^-20 * A.  Quantisation, for amax = max |x| over the
 * finite values of the tensor (of the column of W):
 *   scale = amax / 448,  inv = 448 / amax                (IEEE divisions rounded to nearest;
 *                                                         both 1 when amax = 0; inv = FLT_MAX and
 *                                                         scale = 1 / FLT_MAX when 448 / amax
 *                                                         overflows)
 *   q     = cvt.rn.satfinite.e4m3(x * inv)               (the product rounded to nearest in fp32;
 *                                                         +-inf -> +-448, NaN -> NaN)
 * Deterministic, no host synchronisation. */
/* 1 when meb200_conv_forward_fp8 takes the shape: c_in a multiple of 32 (whole 32-byte k-steps),
 * c_out a multiple of 16 in [16, 1024]; else 0. */
int meb200_conv_fp8_supported(uint32_t c_in, uint32_t c_out);
/* in_e4m3 [n_in, c_in] and a_scale (DEVICE fp32, the dequantisation factor) from
 * meb200_quantize_e4m3; w_t_e4m3 [K, c_out, c_in] from meb200_conv_pack_weights_e4m3; epi required;
 * out_nbr / out_order as in meb200_conv_forward. */
int meb200_conv_forward_fp8(const void *in_e4m3, const float *a_scale, uint32_t n_in, uint32_t c_in,
                            const void *w_t_e4m3, uint32_t K, uint32_t c_out,
                            const int32_t *out_nbr, uint32_t n_out, void *out, int out_dtype,
                            const int32_t *out_order, const meb200_conv_epilogue *epi, void *stream);
/* fp32 weight [K, c_in, c_out] -> w_t_e4m3 [K, c_out, c_in] and w_scale fp32 [c_out], with amax
 * taken per output channel over (k, c_in). */
int meb200_conv_pack_weights_e4m3(const float *weight, uint32_t K, uint32_t c_in, uint32_t c_out,
                                  void *w_t_e4m3, float *w_scale, void *stream);
/* Features [n, c] in `dtype` (F32 / BF16 / F16) -> out_e4m3 [n, c] and scale_dev (DEVICE fp32 [2]:
 * scale, then inv) in two launches: the amax (its last CTA writes the scales) and the conversion,
 * 16 output bytes per access when both buffers are 16-byte aligned.  workspace:
 * meb200_quantize_e4m3_workspace_bytes() bytes, zero-filled once by the caller and shared by the
 * calls on one stream; every call leaves it zero. */
uint64_t meb200_quantize_e4m3_workspace_bytes(void);
int meb200_quantize_e4m3(const void *in, int dtype, uint32_t n, uint32_t c, void *out_e4m3,
                         float *scale_dev, void *workspace, void *stream);

/* ---- fp8 static scales and shadows -------------------------------------------------------------
 * A calibrated layer quantises its input with a scale fixed in advance instead of its amax:
 * the amax of calibration runs, turned into (scale, inv) by the formula above.  Values above the
 * calibrated amax saturate to +-448 (satfinite).
 * meb200_amax_accumulate: *amax_dev = max(*amax_dev, max |x| over the finite values of the [n, c]
 *   features) in one launch (per-CTA max, then an atomic max on the fp32 bits).  *amax_dev starts
 *   at 0 (or any earlier amax); calls accumulate, in any order, to the same bits.
 * meb200_e4m3_scales: scale_dev[0] = scale, scale_dev[1] = inv of *amax_dev (one thread).
 * meb200_quantize_e4m3_static: out_e4m3 = e4m3(x * scale_dev[1]), the conversion launch of
 *   meb200_quantize_e4m3 alone. */
int meb200_amax_accumulate(const void *in, int dtype, uint32_t n, uint32_t c, float *amax_dev,
                           void *stream);
int meb200_e4m3_scales(const float *amax_dev, float *scale_dev, void *stream);
int meb200_quantize_e4m3_static(const void *in, int dtype, uint32_t n, uint32_t c, void *out_e4m3,
                                const float *scale_dev, void *stream);
/* The forward that also writes the SHADOW of its output: q [n_out, c_out] e4m3 bytes, at the static
 * scale q_scale (DEVICE fp32 [2], as scale_dev above) of the layer the output feeds, stored by the
 * epilogue in the launch that stores out:
 *   q[o, c] = e4m3(round_out_dtype(v[o, c]) * q_scale[1])
 * with v the final epilogue value (after the residual and the ReLU), so that q equals
 * meb200_quantize_e4m3_static(out, q_scale) byte for byte.  The arguments are those of
 * meb200_conv_forward / meb200_conv_forward_fp8 / meb200_conv_stem_forward, plus q and q_scale;
 * epi is required.  Only the tensor-core kernels of bf16 / fp16 and e4m3 operands write a shadow:
 * meb200_conv_forward_q returns MEB200_ERR_UNSUPPORTED, before it launches anything, for a shape
 * or dtype that would run on TF32, the small-cin kernel or the SIMT gather-GEMM (and so does
 * meb200_conv_stem_forward_q off the stem kernels).  The caller then runs meb200_conv_forward, and
 * the next layer quantises its input with meb200_quantize_e4m3_static. */
int meb200_conv_forward_q(const void *in, int in_dtype, uint32_t n_in, uint32_t c_in,
                          const void *w_cast, const void *w_t, uint32_t K, uint32_t c_out,
                          const int32_t *out_nbr, uint32_t n_out, void *out, int out_dtype,
                          const int32_t *out_order, const meb200_conv_epilogue *epi, void *q,
                          const float *q_scale, void *stream);
int meb200_conv_forward_fp8_q(const void *in_e4m3, const float *a_scale, uint32_t n_in,
                              uint32_t c_in, const void *w_t_e4m3, uint32_t K, uint32_t c_out,
                              const int32_t *out_nbr, uint32_t n_out, void *out, int out_dtype,
                              const int32_t *out_order, const meb200_conv_epilogue *epi, void *q,
                              const float *q_scale, void *stream);
int meb200_conv_stem_forward_q(const void *in4, int dtype, uint32_t K, const void *weight_v,
                               uint32_t c_out, const int32_t *out_nbr, uint32_t n_out, void *out,
                               int out_dtype, const meb200_conv_epilogue *epi, void *q,
                               const float *q_scale, void *stream);

/* ---- fp8 training: the input gradient on e5m2 x e4m3 -------------------------------------------
 * The dgrad of a convolution (meb200_conv_backward's grad_in) on the Hopper fp8 tensor cores: the
 * output gradient quantised to e5m2 with one scale per tensor, the weights to e4m3 with one scale
 * per INPUT channel (the dgrad's output column), the products summed by the tensor cores:
 *   grad_in[i, ci] = acc[i, ci] * g_scale * w_scale[ci]
 * with acc the sum of e5m2 x e4m3 products over in_nbr, rounded to grad_in_dtype (F32, BF16 or
 * F16, the layer's feature dtype).  The weight gradient keeps meb200_conv_backward.
 * e5m2 quantisation: the e4m3 formula above with 57344 (the largest finite e5m2) for 448:
 *   scale = amax / 57344, inv = 57344 / amax, q = cvt.rn.satfinite.e5m2(x * inv)
 *   (both 1 when amax = 0; inv = FLT_MAX and scale = 1 / FLT_MAX when 57344 / amax overflows;
 *   +-inf -> +-57344, NaN -> NaN).
 * meb200_quantize_e5m2: as meb200_quantize_e4m3 (two launches, the same workspace), in e5m2.
 * meb200_conv_pack_weights_e4m3_dgrad: fp32 weight [K, c_in, c_out] -> w_e4m3 [K, c_in, c_out]
 *   (not transposed) and w_scale fp32 [c_in], amax per input channel over (k, c_out).
 * meb200_conv_dgrad_fp8: grad_e5m2 [n_out, c_out] and g_scale (DEVICE fp32, the dequantisation
 *   factor) from meb200_quantize_e5m2; in_nbr / in_order as in meb200_conv_backward; the shape
 *   must satisfy meb200_conv_fp8_supported(c_out, c_in).  No stem mode, no shadow. */
int meb200_quantize_e5m2(const void *in, int dtype, uint32_t n, uint32_t c, void *out_e5m2,
                         float *scale_dev, void *workspace, void *stream);
int meb200_conv_pack_weights_e4m3_dgrad(const float *weight, uint32_t K, uint32_t c_in,
                                        uint32_t c_out, void *w_e4m3, float *w_scale, void *stream);
int meb200_conv_dgrad_fp8(const void *grad_e5m2, const float *g_scale, uint32_t n_out,
                          uint32_t c_out, const void *w_e4m3, const float *w_scale, uint32_t K,
                          uint32_t c_in, const int32_t *in_nbr, uint32_t n_in, void *grad_in,
                          int grad_in_dtype, const int32_t *in_order, void *stream);

/* ---- fp8 training: the weight gradient on e4m3 x e5m2 ------------------------------------------
 * The wgrad of a convolution (meb200_conv_backward's grad_weight) on the Hopper fp8 tensor cores,
 * from the operands the forward and the dgrad already quantised: the input in e4m3 and the output
 * gradient in e5m2, each with one scale per tensor:
 *   grad_weight[k, ci, co] = (acc[k, ci, co] * a_scale) * g_scale   (fp32, fully written)
 * with acc the sum over the pairs of offset k of in_e4m3[i, ci] * grad_e5m2[o, co].  Every interval
 * of at most 128 pairs is summed by the tensor cores from zero and then added into fp32, so the
 * error does not grow with the number of pairs (DESIGN.md §3, "fp8 training").
 *   in_e4m3 [n_in, c_in], a_scale: meb200_quantize_e4m3 (a_scale the DEVICE dequantisation factor)
 *   grad_e5m2 [n_out, c_out], g_scale: meb200_quantize_e5m2
 *   pairs_in / pairs_out / seg_start / n_chunks: the pair lists of meb200_conv_backward (required)
 *   workspace: meb200_conv_wgrad_fp8_workspace_bytes(n_out, c_in, c_out, K) bytes, 16-byte aligned;
 *              as in meb200_conv_backward, less, NULL or unaligned means fewer row splits, and the
 *              splits are added in a fixed order (bit-identical run to run)
 * Grid (meb200_conv_wgrad_fp8_supported): c_in and c_out multiples of 32 up to 1024, 1 <= K <= 1023;
 * off it the call returns MEB200_ERR_UNSUPPORTED and launches nothing.  n_out = 0: zero, no MMA. */
int meb200_conv_wgrad_fp8_supported(uint32_t c_in, uint32_t c_out, uint32_t K);
uint64_t meb200_conv_wgrad_fp8_workspace_bytes(uint32_t n_out, uint32_t c_in, uint32_t c_out,
                                               uint32_t K);
int meb200_conv_wgrad_fp8(const void *in_e4m3, const float *a_scale, const void *grad_e5m2,
                          const float *g_scale, uint32_t c_in, uint32_t K, uint32_t c_out,
                          const int32_t *pairs_in, const int32_t *pairs_out,
                          const int32_t *seg_start, uint32_t n_chunks, uint32_t n_out,
                          float *grad_weight, void *workspace, uint64_t workspace_bytes,
                          void *stream);

/* ---- fp8 training with delayed scaling ---------------------------------------------------------
 * Each fp8 operand role (a layer's e4m3 input, its e5m2 output gradient) is an ENTRY: a history of
 * the amax of its last H steps and a current slot (DEVICE fp32, zero at the start of a step) that
 * the running step records into.  Step t converts at the (scale, inv) of the history alone, so the
 * conversion waits on no amax pass and can be fused into whoever writes the tensor:
 *   amax  = max of the H past values
 *   (scale, inv) = the e4m3 / e5m2 formula above of min(amax * 2^margin, FLT_MAX)
 *   q     = cvt.rn.satfinite(x * inv): values beyond the scaled amax saturate to +-448 / +-57344
 *   slot  = max(slot, max |x| over the finite values of x), an atomic max on the fp32 bits
 * meb200_fp8_out describes one such write: q the bytes (8-byte aligned where a batch-norm pass
 * writes them), scale the entry's DEVICE fp32 [2] (scale, inv) of the step, amax_slot its slot. */
#define MEB200_FP8_E4M3 0
#define MEB200_FP8_E5M2 1
#define MEB200_FP8_MAX_HISTORY 1024 /* H of meb200_fp8_roll: one thread walks an entry's history */
typedef struct meb200_fp8_out {
  void *q;
  const float *scale;
  float *amax_slot;
} meb200_fp8_out;
/* Features [n, c] in `dtype` (F32 / BF16 / F16) -> out->q [n, c] in `format` (MEB200_FP8_E4M3 /
 * _E5M2) at out->scale, recording the amax into out->amax_slot, in ONE launch (the conversion of
 * meb200_quantize_e4m3_static, 16 output bytes per access when both buffers are 16-byte aligned).
 * n * c = 0: nothing is launched, and in / out->q may be NULL. */
int meb200_quantize_fp8_record(const void *in, int dtype, uint32_t n, uint32_t c, int format,
                               const meb200_fp8_out *out, void *stream);
/* The step boundary of L = n_e4m3 + n_e5m2 entries in one launch (no host read): entry i's slot
 * cur[i] goes in front of its history row hist[i, 0:H] (newest first) and the oldest value drops
 * out; scales[i, 0:2] = (scale, inv) of the new history by the formula above, in e4m3 for
 * i < n_e4m3 and e5m2 from there; next_cur[i] = 0 (the slots of the new step; may be cur).
 * 1 <= H <= MEB200_FP8_MAX_HISTORY, 0 <= margin <= 127. */
int meb200_fp8_roll(const float *cur, float *hist, uint32_t n_e4m3, uint32_t n_e5m2, uint32_t H,
                    int margin, float *next_cur, float *scales, void *stream);

/* Weight packing, once per optimizer step instead of once per call: fp32 master weight
 * [K, Cin, Cout] -> `dtype` (BF16/F16, or TF32: fp32 words rounded to tf32) operand copies
 * w_cast [K, Cin, Cout] and w_t [K, Cout, Cin].  The reference keeps weights in the feature dtype and needs no such step
 * (MinkowskiConvolution.py:264-279); this is the bf16/fp16 operand cache of this backend. */
int meb200_conv_pack_weights(const float *weight, uint32_t K, uint32_t c_in, uint32_t c_out,
                             int dtype, void *w_cast, void *w_t, void *stream);

/* The same packing for MANY layers in one launch (all weights of a network change together, at
 * the optimizer step): `jobs_dev` is a DEVICE array of n_jobs jobs; job j owns the 32x32 tiles
 * [tile_begin_j, tile_begin_j + K_j * ceil(c_in_j / 32) * ceil(c_out_j / 32)) of the launch,
 * tile_begin ascending from 0, total_tiles = their sum.  The table only has to be rebuilt when
 * the set of tensors (or their addresses) changes. */
typedef struct meb200_pack_job {
  const void *w;                      /* fp32 [K, c_in, c_out] */
  void *w_cast, *w_t;                 /* as meb200_conv_pack_weights */
  uint32_t K, c_in, c_out;
  uint32_t tile_begin;
} meb200_pack_job;
int meb200_conv_pack_weights_batched(const meb200_pack_job *jobs_dev, uint32_t n_jobs,
                                     uint32_t total_tiles, int dtype, void *stream);

/* Network stem (the first layer of a network: c_in <= 4 input channels, e.g. RGB; reference
 * call site examples/minkunet.py:113-116 conv0p1s1, kernel 5 -> K = 125).  Rows of 8 bytes defeat
 * the 64-byte-block gather of the general kernels, so the layer is run as a K = 1 convolution over
 * VIRTUAL channels v = 4 k + c (offset k < 16 ceil(K / 16), channel c < 4):
 *   in4            [n_in, 4]   the features zero-padded to 4 channels
 *   weight_v       [c_out, V]  V = meb200_conv_stem_virtual_channels(K); the `w_t` output of
 *                              meb200_conv_pack_weights(Wv, K=1, c_in=V, c_out) where
 *                              Wv[4 k + c][n] = W[k][c][n] (zero for padded k, c)
 *   grad_weight_v  [V, c_out]  fp32, same indexing (fully written by the call)
 *   workspace      meb200_conv_workspace_bytes(n_out, V, c_out, 1, dtype) bytes, 16-byte aligned,
 *                  for the row-split partial sums, as in meb200_conv_backward (less, NULL or
 *                  unaligned is legal and means fewer splits, down to one)
 *   epi            (forward, may be NULL) as in meb200_conv_forward
 * bf16 / fp16 only; c_out a multiple of 16, <= 256. */
uint32_t meb200_conv_stem_virtual_channels(uint32_t K);
int meb200_conv_stem_supported(int dtype, uint32_t K, uint32_t c_out);
int meb200_conv_stem_forward(const void *in4, int dtype, uint32_t K, const void *weight_v,
                             uint32_t c_out, const int32_t *out_nbr, uint32_t n_out, void *out,
                             int out_dtype, const meb200_conv_epilogue *epi, void *stream);
int meb200_conv_stem_wgrad(const void *in4, const void *grad_out, int dtype, uint32_t K,
                           uint32_t c_out, const int32_t *out_nbr, uint32_t n_out,
                           float *grad_weight_v, void *workspace, uint64_t workspace_bytes,
                           void *stream);

/* ---- channel-wise (depthwise) convolution (reference: MinkowskiChannelwiseConvolution.py:142-191,
 *      a per-offset torch loop with an autograd backward).  W: fp32 [K, C], one weight per offset
 *      and channel.  Every output element is written once: no memset, no atomics, bit-identical
 *      results run to run; fp32 accumulation, one rounding to the feature dtype; 16-byte accesses
 *      where C * sizeof(dtype) % 16 == 0 and the pointers allow, any C >= 1 otherwise. --------- */
/* y[r, c] = sum over k ascending with nbr[k, r] >= 0 of W[k, c] * x[nbr[k, r], c] (0 for a row
 * without neighbours), r < n_rows.  x: [n_x, C], y: [n_rows, C] in `dtype`; nbr: [K, n_rows].
 * Forward: nbr = out_nbr, x = the input features.  Input gradient: nbr = in_nbr, x = the output
 * gradient, the same W. */
int meb200_chwise_gather(const void *x, int dtype, uint32_t n_x, uint32_t C, const float *W,
                         const int32_t *nbr, uint32_t K, uint32_t n_rows, void *y, void *stream);
/* dW[k, c] (fp32 [K, C], fully written) = sum over o with out_nbr[k, o] >= 0 of
 * x[out_nbr[k, o], c] * g[o, c].  x: [n_x, C], g: [n_out, C] in `dtype`.  workspace:
 * meb200_chwise_wgrad_workspace_bytes(n_out, C, K, dtype) bytes, 16-byte aligned, for the row
 * splits' partial sums, added in split order, as in meb200_conv_backward (less, NULL or unaligned
 * is legal and means fewer splits, down to one). */
uint64_t meb200_chwise_wgrad_workspace_bytes(uint32_t n_out, uint32_t C, uint32_t K, int dtype);
int meb200_chwise_wgrad(const void *x, const void *g, int dtype, uint32_t n_x, uint32_t C,
                        const int32_t *out_nbr, uint32_t K, uint32_t n_out, float *dW,
                        void *workspace, uint64_t workspace_bytes, void *stream);

/* ---- local pooling (reference a11: src/pooling_avg_kernel.hpp:40-150,
 *      src/pooling_max_kernel.hpp:35-115, src/local_pooling_cpu.cpp:43-185) ---------- */
/* aux: AVG -> num_nonzero [n_out] (feature dtype); MAX -> max_index int32 [n_out, C]
 * (flat index row*C + c into `in`, -1 for rows without input); SUM -> unused (NULL ok).
 * MAX: an empty window holds the lowest finite value of the dtype (not -inf in bf16/fp16). */
int meb200_pool_forward(const void *in, int dtype, uint32_t n_in, uint32_t C,
                        const int32_t *out_nbr, uint32_t K, uint32_t n_out, int mode,
                        void *out, void *aux, void *stream);
/* grad_in fully written in every mode (no pre-zeroing), accumulated in fp32 in ascending k over
 * in_nbr (required in every mode) and rounded once; deterministic, no atomics.  MAX:
 * grad_in[i,c] = sum over windows o = in_nbr[k,i] with max_index[o,c] == i*C + c of grad_out[o,c]. */
int meb200_pool_backward(const void *grad_out, int dtype, uint32_t n_in, uint32_t C,
                         const int32_t *in_nbr, uint32_t K, uint32_t n_out, int mode,
                         const void *aux, void *grad_in, void *stream);

/* ---- per-cloud grouping, segmented reduction, broadcast (reference: the origin map
 *      coordinate_map_cpu.hpp:492-513,724-783; src/global_pooling_cpu.cpp;
 *      src/broadcast_kernel.hpp).  A "segment" is the set of rows of one cloud: the rows whose
 *      (batch, 0, ..., 0) is row s of the origin map.  Deterministic: no float atomics, no
 *      atomics that decide an order, bit-identical results run to run. ----------------------- */
#define MEB200_SEGMENT_TILE_ROWS 512 /* rows per reduction tile */

#define MEB200_SEG_SUM 0
#define MEB200_SEG_AVG 1
#define MEB200_SEG_MAX 2

#define MEB200_BCAST_ADD 0     /* reference BroadcastMode::ELEMENTWISE_ADDITON (src/types.hpp) */
#define MEB200_BCAST_MUL 1     /* ELEMENTWISE_MULTIPLICATION */
#define MEB200_BCAST_COPY 2    /* out = g[seg]  (sum / avg pooling backward, MinkowskiBroadcast) */
#define MEB200_BCAST_MAXGRAD 3 /* out = g[seg] where argmax[seg] == i*C + c, else 0 */

/* Groups the n rows of `coords` by cloud.  origin_coords / origin_table / origin_capacity: the
 * origin map (B rows (b, 0, ..., 0) and its row-index table, as meb200_insert_and_map leaves
 * them).  Outputs (DEVICE, no host synchronisation):
 *   row_seg    int32 [n]    origin row of every row (-1: its batch index is not in the origin map)
 *   order      int32 [n]    rows grouped by segment, ascending row order inside a segment
 *   seg_start  int32 [B+1]  segment s is order[seg_start[s] .. seg_start[s+1])
 *   tile_start int32 [B+1]  reduction tiles of segment s: [tile_start[s], tile_start[s+1]),
 *                           ceil(rows / MEB200_SEGMENT_TILE_ROWS) each
 * scratch: meb200_origin_group_scratch_bytes(n, B) bytes.  1 <= B <= 12288. */
uint64_t meb200_origin_group_scratch_bytes(uint32_t n, uint32_t B);
int meb200_origin_group(const int32_t *coords, uint32_t n, uint32_t ncols,
                        const int32_t *origin_coords, const uint32_t *origin_table,
                        uint32_t origin_capacity, uint32_t B, int32_t *row_seg, int32_t *order,
                        int32_t *seg_start, int32_t *tile_start, void *scratch, void *stream);
/* The same grouping for the n points of a tensor field: field float32 [n, ncols], a point's cloud
 * is the origin row of (lroundf(field[i, 0]), 0, ..., 0); outputs and scratch as
 * meb200_origin_group.  d_bad (DEVICE uint32 status word, cleared by the call; NULL when the
 * batch column is known valid) is set to 1 when a batch value is not finite or its rounding lies
 * outside int32; such a point gets row_seg -1 and is in no segment. */
int meb200_field_origin_group(const float *field, uint32_t n, uint32_t ncols,
                              const int32_t *origin_coords, const uint32_t *origin_table,
                              uint32_t origin_capacity, uint32_t B, int32_t *row_seg,
                              int32_t *order, int32_t *seg_start, int32_t *tile_start,
                              uint32_t *d_bad, void *scratch, void *stream);
/* The origin map of a tensor field: the candidate rows (lroundf(field[i, 0]), 0, ..., 0) written to
 * ocoords (int32 [n, ncols]) and inserted by meb200_insert_and_map (the other arguments as there).
 * The validity of the batch column reaches the host with the unique count, in the same read; a
 * batch value that is not finite or outside int32 returns MEB200_ERR_DOMAIN. */
int meb200_field_origin_insert(const float *field, uint32_t n, uint32_t ncols, int32_t *ocoords,
                               uint32_t *table, uint32_t capacity, int32_t *unique_coords,
                               int64_t *unique_index, int64_t *inverse_map, void *scratch,
                               uint32_t *h_num_unique, void *stream);

/* out[s, c] (fp32 [B, C]) = SUM / AVG / MAX over the rows i of segment s of a[i, c], or of
 * a[i, c] * b[i, c] when b != NULL (SUM / AVG only).  Each tile of a segment stores fp32 partials
 * into `workspace` (meb200_segment_workspace_bytes(n, C, B) bytes, 16-byte aligned) and a second
 * pass adds them in tile order.  aux (may be NULL): SUM / AVG -> fp32 [B] row counts; MAX -> int32
 * [B, C] flat index row*C + c of the maximum (lowest row on ties).  An empty segment gives 0 (and
 * index -1).  a, b: [n, C] in `dtype`. */
uint32_t meb200_segment_max_tiles(uint32_t n, uint32_t B);
uint64_t meb200_segment_workspace_bytes(uint32_t n, uint32_t C, uint32_t B);
int meb200_segment_reduce(const void *a, const void *b, int dtype, uint32_t n, uint32_t C,
                          const int32_t *order, const int32_t *seg_start,
                          const int32_t *tile_start, uint32_t B, int mode, float *out, void *aux,
                          void *workspace, uint64_t workspace_bytes, void *stream);

/* out[i, c] = x[i, c] op g[row_seg[i], c] for every row (fully written, no memset):
 * op ADD / MUL; COPY: g[row_seg[i], c]; MAXGRAD: g[s, c] where argmax[s, c] == i*C + c, else 0
 * (x unused for COPY / MAXGRAD).  x: [n, C] in `dtype`; g: fp32 [B, C]; argmax: int32 [B, C];
 * out: [n, C] in out_dtype (= dtype or F32). */
int meb200_broadcast(const void *x, int dtype, const float *g, const int32_t *argmax,
                     const int32_t *row_seg, uint32_t n, uint32_t C, int op, void *out,
                     int out_dtype, void *stream);

/* out[i, c] = x[i, c] * g[s, c] + z[i, c] * h[s, c] + k[s, c] with s = row_seg[i]: the per-cloud
 * affine pass of instance normalisation (forward: z = h = NULL; backward: z = the normalised
 * features).  x, z, out: [n, C] in `dtype`; g, h, k: fp32 [B, C]; z / h (together) and k may be
 * NULL. */
int meb200_broadcast_fma(const void *x, const void *z, int dtype, const float *g, const float *h,
                         const float *k, const int32_t *row_seg, uint32_t n, uint32_t C, void *out,
                         void *stream);

/* ---- pruning, union and arithmetic between different coordinate maps (reference:
 *      src/pruning_cpu.cpp, MinkowskiUnion.py:50-82, MinkowskiTensor.py:522-540).  The maps come
 *      from meb200_insert_and_map (pruned: valid = the keep mask; union: the inputs' rows
 *      concatenated).  Every output element is written exactly once: no memset, no atomics,
 *      bit-identical results run to run.  fp32 arithmetic, one rounding to the feature dtype;
 *      16-byte accesses where C * sizeof(dtype) % 16 == 0 and the pointers allow. ------------- */
#define MEB200_UNION_ADD 0
#define MEB200_UNION_SUB 1
#define MEB200_UNION_MUL 2
#define MEB200_UNION_DIV 3

/* out[j, :] = idx[j] >= 0 ? src[idx[j], :] : 0 for j < n_out; src: [n_src, C], out: [n_out, C] in
 * `dtype`.  Pruning forward (idx = the insert's unique_index) and backward (idx = its
 * inverse_map, -1 -> zero row). */
int meb200_gather_rows(const void *src, int dtype, uint32_t n_src, uint32_t C, const int64_t *idx,
                       uint32_t n_out, void *out, void *stream);

/* The union fold.  inputs: DEVICE array of N feature pointers ([n_i, C] in `dtype`);
 * inputs_align: a power of two dividing every one of them (16 enables vector loads);
 * src: int32 [N, M], src[i, u] = row of input i with union row u's coordinate, or -1.
 * Forward, for every union row u:  acc = 0;  for i = 0..N-1 with src[i, u] >= 0:
 *   acc = (i == 0) ? x_i : op(acc, x_i);   out[u] = acc          (out: [M, C])
 * Backward, for input i: grad_i[r] = grad_out[u_i[r]] * d out / d x_i at u_i[r] (u_i: int64
 * [n_i], the union row of every row of input i), the derivative of the piecewise fold above:
 *   ADD 1;  SUB i == 0 ? 1 : -1;  MUL the product of the other present inputs (0 when i > 0 and
 *   input 0 is absent);  DIV i == 0: 1 / x_1 / x_2 ...,  i > 0: -(out / x_i). */
int meb200_union_fold_forward(const void *const *inputs, uint32_t N, uint32_t inputs_align,
                              const int32_t *src, uint32_t M, uint32_t C, int dtype, int op,
                              void *out, void *stream);
int meb200_union_fold_backward(const void *const *inputs, uint32_t N, uint32_t inputs_align,
                               const int32_t *src, uint32_t M, uint32_t C, int dtype, int op,
                               const void *grad_out, uint32_t i, const int64_t *u_i, uint32_t n_i,
                               void *grad_i, void *stream);

/* ---- dense tensors: feature rows <-> a dense volume (reference: SparseTensor.dense
 *      MinkowskiSparseTensor.py:460-557, to_sparse MinkowskiOps.py:279-317).  Data movement only:
 *      bit-exact in every dtype.  Every output element is written exactly once: no memset, no
 *      atomics.  16-byte accesses where C * sizeof(dtype) % 16 == 0 and the pointers and strides
 *      allow.
 *   A dense tensor [B, C, X1..XD] in any axis order, or any strided view of one, is described by
 *   its ELEMENT strides; offsets are 64-bit.  Columns follow coordinate rows: column 0 the batch
 *   index, columns 1..D the axes.  Cell (i_0..i_D) holds the coordinate origin[j] + i_j * step[j]
 *   (column 0: origin 0, step 1). ---------------------------------------------------------------- */
typedef struct {
  uint32_t ncols;                    /* D + 1                                          */
  uint32_t channels;                 /* C                                              */
  uint32_t shape[MEB200_MAX_NCOLS];  /* B, X1..XD                                      */
  int64_t stride[MEB200_MAX_NCOLS];  /* element stride of the batch axis and each axis */
  int64_t channel_stride;
  int32_t origin[MEB200_MAX_NCOLS];  /* 0, min_coordinate                              */
  int32_t step[MEB200_MAX_NCOLS];    /* 1, then the tensor stride (contracted) or 1    */
} meb200_dense_desc;

/* dense[cell, :] = feats[r, :] where row r of the map lies on the cell's coordinate, else 0, for
 * every cell: the map's table is probed once per cell as meb200_map_find probes it, so rows
 * outside the volume are never reached (cropped), and with step 1 on a strided map the cells off
 * its lattice are zero.  feats: [n, C] in `dtype`; desc: HOST.  SparseTensor.dense forward and
 * the backward of to_sparse (reference: the index assignment of MinkowskiSparseTensor.py:546-554). */
int meb200_dense_from_rows(const void *feats, int dtype, uint32_t n, const int32_t *map_coords,
                           const uint32_t *table, uint32_t capacity,
                           const meb200_dense_desc *desc, void *dense, void *stream);

/* out[r, :] = dense[cell of coords[r], :] for r < n, 0 where the row lies outside the volume or
 * off the step lattice.  coords: int32 [n, ncols]; out: [n, C] in `dtype`; desc: HOST.  The
 * features of to_sparse (reference: MinkowskiOps.py:311-316) and the backward of dense. */
int meb200_dense_to_rows(const void *dense, int dtype, const meb200_dense_desc *desc,
                         const int32_t *coords, uint32_t n, void *out, void *stream);

/* Non-zero cells of a dense volume (reference: abs(x).sum(channel) != 0, where, stack —
 * MinkowskiOps.py:308-310): a cell counts when any channel is not +0 / -0 (NaN counts).  _count
 * flags the cells in one pass over the volume, scans the flags and writes the number of non-zero
 * cells to *h_count (HOST) after a stream synchronise: the one blocking point, the caller needs it
 * to size `coords`.  _coords then writes their indices (origin and step are not applied), int32
 * [*h_count, ncols], in row-major (batch, X1..XD) order.  scratch:
 * meb200_dense_nonzero_scratch_bytes(cells) bytes, cells = the product of desc->shape, at most
 * 2^32 - 2049; the same scratch, untouched, goes to _coords. */
uint64_t meb200_dense_nonzero_scratch_bytes(uint64_t cells);
int meb200_dense_nonzero_count(const void *dense, int dtype, const meb200_dense_desc *desc,
                               void *scratch, uint32_t *h_count, void *stream);
int meb200_dense_nonzero_coords(const meb200_dense_desc *desc, void *scratch, int32_t *coords,
                                void *stream);

/* ---- tensor fields: points with float coordinates, quantised to voxels (reference:
 *      MinkowskiTensorField.py, CoordinateFieldMapCPU::quantize_coordinates
 *      coordinate_map_cpu.hpp:994-1037, interpolation_map_weight_kernel :139-240,
 *      src/interpolation_cpu.cpp, src/direct_max_pool.cpp).  Every output element is written
 *      exactly once: no memset, no float atomics, bit-identical results run to run.  fp32
 *      accumulation with one rounding to the feature dtype; 16-byte accesses where
 *      C * sizeof(dtype) % 16 == 0 and the pointers allow.
 *   field   float32 [n, ncols]: column 0 the batch index (rounded with lroundf), then the axes;
 *           a point lies in the voxel floorf(x / s) * s of tensor stride s (float division). ---- */
#define MEB200_ERR_DOMAIN (-4) /* a field coordinate is not finite or its voxel is outside int32 */

#define MEB200_FIELD_SUM 0       /* SparseTensorQuantizationMode.UNWEIGHTED_SUM */
#define MEB200_FIELD_AVG 1       /* UNWEIGHTED_AVERAGE */
#define MEB200_FIELD_MAX 2       /* MAX_POOL */
#define MEB200_FIELD_SUBSAMPLE 3 /* RANDOM_SUBSAMPLE (the first point of a voxel) */

/* Quantises the field at `tensor_stride` (HOST int32 [ncols-1]) into out (int32 [n, ncols]) and,
 * when d_bad != NULL, sets *d_bad (DEVICE uint32 status word, cleared by the call) to 1 when a
 * coordinate is not finite or its voxel falls outside int32 (NULL: the field is known valid). */
int meb200_quantize_field(const float *field, uint32_t n, uint32_t ncols,
                          const int32_t *tensor_stride, int32_t *out, uint32_t *d_bad,
                          void *stream);
/* Quantisation followed by meb200_insert_and_map on the quantised rows (qcoords: int32 [n, ncols]
 * buffer; the other arguments as meb200_insert_and_map): the first point of a voxel is its
 * unique_index.  The validity of the coordinates reaches the host with the unique count, in the
 * same read; invalid coordinates return MEB200_ERR_DOMAIN. */
int meb200_field_insert_and_map(const float *field, uint32_t n, uint32_t ncols,
                                const int32_t *tensor_stride, int32_t *qcoords, uint32_t *table,
                                uint32_t capacity, int32_t *unique_coords, int64_t *unique_index,
                                int64_t *inverse_map, void *scratch, uint32_t *h_num_unique,
                                void *stream);

/* Deterministic grouping of P entries by an int32 key in [0, M) (keys outside are left out):
 * entries of key r are perm[start[r] .. start[r+1]), in ascending entry order (a stable radix
 * sort).  start: int32 [M+1], perm: int32 [P] (entries past start[M] are the left-out ones).
 * scratch: meb200_group_by_row_scratch_bytes(P, M) bytes. */
uint64_t meb200_group_by_row_scratch_bytes(uint32_t P, uint32_t M);
int meb200_group_by_row(const int32_t *keys, uint32_t P, uint32_t M, int32_t *start, int32_t *perm,
                        void *scratch, uint64_t scratch_bytes, void *stream);

/* Points -> voxels.  For every output row r < M, over its entries j = perm[start[r] ..
 * start[r+1]) in order, with source row s = src_row[j] (int32 [P]) when src_row != NULL, else
 * s = j / src_div, and x = src[s, :] (times weight[j] when weight != NULL): SUM the fp32 sum, AVG
 * the sum over the exact count, MAX the maximum (the first entry wins ties) with argmax[r, c] = the
 * winning entry j (int32 [M, C]; its source row s when src_row == NULL and src_div == 1).  A row
 * without entries gives 0 (argmax -1).  src: [n_src, C] in `dtype`, out:
 * [M, C] in `dtype`; src_row values must lie in [0, n_src) (meb200_check_pairs).  Also the
 * backward of a slice (SUM), of interpolation (SUM, weight = the interpolation weights, src_div =
 * 2^D), and, with src_row = the column of each COO entry, a sparse matrix times a dense matrix
 * (SUM, weight = the values), its row average (AVG) and max pooling over a pair list (MAX). */
int meb200_field_reduce(const void *src, int dtype, uint32_t n_src, uint32_t C, const int32_t *perm,
                        const int32_t *start, uint32_t M, const float *weight,
                        const int32_t *src_row, uint32_t src_div, int mode, void *out,
                        int32_t *argmax, void *stream);

/* Range check of a pair list (int32 [P] each): every rows[p] in [0, n_rows) and cols[p] in
 * [0, n_cols), else MEB200_ERR_INVALID.  The status word (d_status: DEVICE uint32, cleared by the
 * call) is read back after a stream synchronise: the one blocking point of a call on a pair list
 * the caller hands in. */
int meb200_check_pairs(const int32_t *rows, const int32_t *cols, uint32_t P, uint32_t n_rows,
                       uint32_t n_cols, uint32_t *d_status, void *stream);

/* mask[r, c] = src_row[argmax[r, c]] * C + c, or -1 where argmax is -1 (argmax: int32 [M, C], the
 * winning entries of a MAX meb200_field_reduce over a [n_src, C] source with per-entry source rows
 * src_row; mask: [M, C] int32 or int64 by index_bits): the flat argmax of direct max pooling.  For
 * int32, n_src * C must be at most 2^31 (the largest index n_src * C - 1 fits). */
int meb200_flat_mask(const int32_t *argmax, const int32_t *src_row, uint32_t M, uint32_t C,
                     uint32_t n_src, int index_bits, void *mask, void *stream);

/* Voxels -> points: out[i, :] = g[inv[i], :] scaled per mode (inv: int64 [n]; -1 -> 0):
 * AVG  times 1 / (start[r+1] - start[r]);  MAX  kept where argmax[r, c] == i, else 0;
 * SUBSAMPLE  kept where unique_index[r] == i, else 0.  The backward of meb200_field_reduce (the
 * plain copy is meb200_gather_rows).  g: [M, C], out: [n, C] in `dtype`. */
int meb200_field_expand(const void *g, int dtype, uint32_t M, uint32_t C, const int64_t *inv,
                        uint32_t n, int mode, const int32_t *start, const int32_t *argmax,
                        const int64_t *unique_index, void *out, void *stream);

/* Trilinear (multilinear) interpolation map of n query points (float32 [n, ncols]) into a
 * coordinate map of tensor stride `tensor_stride` (HOST int32 [ncols-1]): the corners
 * floorf(x / s) * s + b * s (b in {0, 1} per axis; bit ncols-1-j of corner k selects the upper
 * end of axis j) are probed in the map; rows int32 [n, 2^D] = the corner's row or -1, weights
 * fp32 [n, 2^D] = prod_j (1 - |x_j - corner_j| / s_j) (0 where absent; not normalised).
 * A query with a non-finite coordinate has no corners. */
int meb200_interp_map(const float *query, uint32_t n, uint32_t ncols, const int32_t *tensor_stride,
                      const int32_t *map_coords, const uint32_t *table, uint32_t capacity,
                      int32_t *rows, float *weights, void *stream);
/* Splat corners of n field points (float32 [n, ncols]) in one launch: out (int32 [n * 2^D, ncols],
 * point-major) row q * 2^D + k = floorf of every column of point q (the batch column included)
 * plus 1 on axis j when bit ncols-1-j of k is set (the corner order of meb200_interp_map).
 * *d_bad (DEVICE uint32 status word, cleared by the call) gets bit 0 when a coordinate is not
 * finite or a corner falls outside int32, and bit 1 when a batch value is not an integer. */
int meb200_splat_coords(const float *field, uint32_t n, uint32_t ncols, int32_t *out,
                        uint32_t *d_bad, void *stream);
/* out[q, :] = sum_k weights[q, k] * F[rows[q, k], :] over the present corners in ascending k
 * (fp32, one rounding).  F: [M, C], out: [n, C] in `dtype`; K = 2^D. */
int meb200_interp_forward(const void *F, int dtype, uint32_t M, uint32_t C, const int32_t *rows,
                          const float *weights, uint32_t n, uint32_t K, void *out, void *stream);

/* ---- batch normalisation over [n, C] feature rows (SURVEY.md 8(f) "next" row 1; the
 *      reference applies torch.nn.BatchNorm1d to `.F`: MinkowskiEngine/MinkowskiNormalization.py:51-99).
 *      C must be a multiple of 8.  sums: DEVICE double [2C]; statistics tensors fp32 [C]. ------ */
/* mean / invstd (biased variance + eps) from the (possibly all-reduced) sums
 * [sum x | sum x^2] over `count` rows; running statistics (may be NULL) updated with momentum
 * and the unbiased variance.  The row count is `count`, or — for synchronised BN over NCCL,
 * where it is the all-reduced total that only exists on the device — read from *d_count when
 * d_count != NULL. */
int meb200_bn_finalize(const double *sums, double count, const double *d_count, uint32_t C,
                       float eps, float momentum, float *running_mean, float *running_var,
                       float *mean, float *invstd, void *stream);
/* The streaming passes, with the BasicBlock tail of modules/resnet_block.py:52-68 folded in:
 *   apply_fused           y = relu?( bn(x) + residual? ),  bn(x) = (x - mean) * invstd * weight + bias
 *   backward_apply_fused  with dy' = relu ? dy * (y_mask > 0) : dy  (y_mask = the fused output y):
 *                         dx = (dy' - sums[c]/count - xhat * sums[C+c]/count) * invstd * weight,
 *                         d_residual (may be NULL) = dy'
 * weight / bias / residual / y_mask / d_residual may be NULL. */
int meb200_bn_apply_fused(const void *x, int dtype, uint32_t n, uint32_t C, const float *mean,
                          const float *invstd, const float *weight, const float *bias,
                          const void *residual, int relu, void *y, void *stream);
int meb200_bn_backward_apply_fused(const void *dy, const void *x, const void *y_mask, int dtype,
                                   uint32_t n, uint32_t C, const float *mean, const float *invstd,
                                   const float *weight, const double *sums, double count,
                                   const double *d_count, void *dx, void *d_residual,
                                   void *stream);

/* The reductions (two launches per pass, no memset): they take a WORKSPACE of
 * meb200_bn_workspace_bytes() bytes, zero-filled once by the caller and shared by every layer
 * that runs on the same stream; the last CTA of a reduction consumes the totals (finalize /
 * parameter gradients / copy-out) and leaves the workspace zero again.
 *   meb200_bn_forward_train      = stats + finalize (one launch) + apply_fused; n > 0;
 *                                  *num_batches_tracked (int64, may be NULL) is incremented
 *   meb200_bn_stats_to           = stats, totals [sum x | sum x^2] copied to sums_out[2C]
 *                                  (the exchange slot of a synchronised layer)
 *   meb200_bn_backward_reduce_to = backward reduce, totals [sum dy | sum dy*xhat] copied to
 *                                  sums_out[2C] and, when non-NULL, to fp32 grad_bias / grad_weight */
uint64_t meb200_bn_workspace_bytes(void);
int meb200_bn_forward_train(const void *x, int dtype, uint32_t n, uint32_t C, const float *weight,
                            const float *bias, const void *residual, int relu, float eps,
                            float momentum, float *running_mean, float *running_var,
                            long long *num_batches_tracked, void *workspace, float *mean,
                            float *invstd, void *y, void *stream);
int meb200_bn_stats_to(const void *x, int dtype, uint32_t n, uint32_t C, void *workspace,
                       double *sums_out, void *stream);
int meb200_bn_backward_reduce_to(const void *dy, const void *x, const void *y_mask, int dtype,
                                 uint32_t n, uint32_t C, const float *mean, const float *invstd,
                                 void *workspace, double *sums_out, float *grad_weight,
                                 float *grad_bias, void *stream);

/* ---- synchronised batch norm: statistics exchange over NVLink peer memory ----------------
 * Replaces the per-layer NCCL all-reduce of torch.nn.SyncBatchNorm (reference:
 * MinkowskiEngine/MinkowskiNormalization.py:101-192, examples/multigpu_ddp.py:91-95).  Every rank
 * owns a buffer in symmetric memory with the same layout: bytes [0, 1024) hold uint32 flags
 * (flag[r] = last call whose slot of rank r is complete), slots follow.  `peer_bases_dev` is a
 * DEVICE array of `world` device pointers, entry r = base of rank r's buffer as mapped into this
 * process.  An exchange publishes `seq` to every peer, waits for every peer's `seq`, then sums
 * the ranks' slots in rank order (bitwise identical on all ranks).  `seq` must increase by one
 * per call on every rank; consecutive calls must use different slots (a rank can be at most one
 * call ahead of its slowest peer).  Flags must be zero before the first call.
 * The exchange is run by the LAST CTA of the batch-norm reductions themselves (no separate
 * launch): meb200_bn_forward_train / meb200_bn_backward_reduce_to of a synchronised layer.  The
 * slot ([sum | sum2 | rows] forward, [sum dy | sum dy*xhat] backward) is filled by the kernel;
 * mean / 1/std / running statistics come from the global totals and the global row count
 * (returned in *total_rows, device); the parameter gradients stay LOCAL sums (DDP averages them),
 * sums_out receives the global ones for meb200_bn_backward_apply_fused.  A rank with n = 0 rows
 * still takes part. */
int meb200_bn_forward_train_peer(const void *x, int dtype, uint32_t n, uint32_t C,
                                 const float *weight, const float *bias, const void *residual,
                                 int relu, float eps, float momentum, float *running_mean,
                                 float *running_var, long long *num_batches_tracked,
                                 void *workspace, const void *peer_bases_dev,
                                 uint64_t slot_offset_bytes, uint32_t seq, uint32_t rank,
                                 uint32_t world, float *mean, float *invstd, double *total_rows,
                                 void *y, void *stream);
int meb200_bn_backward_reduce_peer(const void *dy, const void *x, const void *y_mask, int dtype,
                                   uint32_t n, uint32_t C, const float *mean, const float *invstd,
                                   void *workspace, const void *peer_bases_dev,
                                   uint64_t slot_offset_bytes, uint32_t seq, uint32_t rank,
                                   uint32_t world, double *sums_out, float *grad_weight,
                                   float *grad_bias, void *stream);

/* ---- batch norm writing an fp8 copy of its output (delayed scaling, above) -----------------------
 * The _q twins take the arguments of their entry plus `fq` (required) and also write, in the apply
 * pass, fq->q [n, C] = the fp8 bytes of the value the pass stores, rounded to `dtype` first:
 *   forward (apply_fused, forward_train, forward_train_peer): q = e4m3(round_dtype(y) * fq->scale[1])
 *   backward_apply_fused:                                      q = e5m2(round_dtype(dx) * fq->scale[1])
 * so that q equals meb200_quantize_fp8_record of the stored y / dx byte for byte, and maxes
 * max |round_dtype(v)| over the finite values into *fq->amax_slot.  Each thread's eight channels
 * are one 8-byte store; fq->q must be 8-byte aligned (it may be NULL when n = 0: a rank without
 * rows still takes part in the exchange of forward_train_peer_q).  Every other output (y, dx,
 * d_residual, statistics, running statistics) is that of the entry without the copy, bit for
 * bit. */
int meb200_bn_apply_fused_q(const void *x, int dtype, uint32_t n, uint32_t C, const float *mean,
                            const float *invstd, const float *weight, const float *bias,
                            const void *residual, int relu, void *y, const meb200_fp8_out *fq,
                            void *stream);
int meb200_bn_forward_train_q(const void *x, int dtype, uint32_t n, uint32_t C,
                              const float *weight, const float *bias, const void *residual,
                              int relu, float eps, float momentum, float *running_mean,
                              float *running_var, long long *num_batches_tracked, void *workspace,
                              float *mean, float *invstd, void *y, const meb200_fp8_out *fq,
                              void *stream);
int meb200_bn_forward_train_peer_q(const void *x, int dtype, uint32_t n, uint32_t C,
                                   const float *weight, const float *bias, const void *residual,
                                   int relu, float eps, float momentum, float *running_mean,
                                   float *running_var, long long *num_batches_tracked,
                                   void *workspace, const void *peer_bases_dev,
                                   uint64_t slot_offset_bytes, uint32_t seq, uint32_t rank,
                                   uint32_t world, float *mean, float *invstd, double *total_rows,
                                   void *y, const meb200_fp8_out *fq, void *stream);
int meb200_bn_backward_apply_fused_q(const void *dy, const void *x, const void *y_mask, int dtype,
                                     uint32_t n, uint32_t C, const float *mean,
                                     const float *invstd, const float *weight, const double *sums,
                                     double count, const double *d_count, void *dx,
                                     void *d_residual, const meb200_fp8_out *fq, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* MEB200_H_ */
