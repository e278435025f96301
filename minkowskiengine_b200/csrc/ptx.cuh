// Thin inline-PTX wrappers for the Hopper (sm_90a) primitives the tensor-core kernels use:
// cp.async, the async-proxy fence, warpgroup MMA (wgmma) with shared-memory descriptors, and the
// warp-level tf32 MMA of the TF32 weight gradient.
#pragma once
#include <stdint.h>

namespace meb200 {
namespace ptx {

__device__ __forceinline__ uint32_t smem_u32(const void *p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---- cp.async (LDGSTS) ------------------------------------------------------------
// 16-byte global->shared copy; src_bytes = 0 zero-fills the destination (missing row).
__device__ __forceinline__ void cp_async16(uint32_t dst, const void *src, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src),
               "r"(src_bytes)
               : "memory");
}
// 8-byte variant (4-channel rows of a network stem); src_bytes = 0 zero-fills
__device__ __forceinline__ void cp_async8(uint32_t dst, const void *src, uint32_t src_bytes) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;" ::"r"(dst), "l"(src), "r"(src_bytes)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() {
  asm volatile("cp.async.commit_group;" ::: "memory");
}
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
// generic-proxy shared-memory writes -> visible to the async proxy (wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ---- wgmma ------------------------------------------------------------------------
// Shared-memory matrix descriptor, no swizzle: the operand is stored as 8 x 16-byte "core
// matrices" (8 rows of 16 contiguous bytes).  lbo = byte distance between core matrices that
// are adjacent along the reduction (K) axis, sbo = along the M / N axis.
__device__ __forceinline__ uint64_t wgmma_desc(uint32_t saddr, uint32_t lbo, uint32_t sbo) {
  return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)((lbo >> 4) & 0x3FFFu) << 16) |
         ((uint64_t)((sbo >> 4) & 0x3FFFu) << 32);
}
__device__ __forceinline__ void wgmma_fence() {
  asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
}
__device__ __forceinline__ void wgmma_commit() {
  asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
}
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}

// D[64 x N] (fp32, registers) += A[64 x 16] * B[16 x N], both operands in shared memory.
// TA / TB = 1: the operand is stored MN-major (M / N contiguous), 0: K-major.
// Accumulator layout per warp w of the warpgroup (rows 16w..16w+15), lane = 4g + t:
//   d[4j + e] = D[16w + g + 8(e >> 1)][8j + 2t + (e & 1)]
#define MEB_F8(d, o) "+f"(d[o]), "+f"(d[o + 1]), "+f"(d[o + 2]), "+f"(d[o + 3]), \
    "+f"(d[o + 4]), "+f"(d[o + 5]), "+f"(d[o + 6]), "+f"(d[o + 7])
template <int TA, int TB>
__device__ __forceinline__ void wgmma_16_bf16(float (&d)[8], uint64_t da, uint64_t db) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7}, "
               "%8, %9, p, 1, 1, %11, %12;\n\t}"
               : MEB_F8(d, 0) : "l"(da), "l"(db), "r"(1), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_16_f16(float (&d)[8], uint64_t da, uint64_t db) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7}, "
               "%8, %9, p, 1, 1, %11, %12;\n\t}"
               : MEB_F8(d, 0) : "l"(da), "l"(db), "r"(1), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_32_bf16(float (&d)[16], uint64_t da, uint64_t db) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
               "%16, %17, p, 1, 1, %19, %20;\n\t}"
               : MEB_F8(d, 0), MEB_F8(d, 8) : "l"(da), "l"(db), "r"(1), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_32_f16(float (&d)[16], uint64_t da, uint64_t db) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
               "%16, %17, p, 1, 1, %19, %20;\n\t}"
               : MEB_F8(d, 0), MEB_F8(d, 8) : "l"(da), "l"(db), "r"(1), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_64_bf16(float (&d)[32], uint64_t da, uint64_t db) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
               "%32, %33, p, 1, 1, %35, %36;\n\t}"
               : MEB_F8(d, 0), MEB_F8(d, 8), MEB_F8(d, 16), MEB_F8(d, 24) : "l"(da), "l"(db), "r"(1), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_64_f16(float (&d)[32], uint64_t da, uint64_t db) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
               "%32, %33, p, 1, 1, %35, %36;\n\t}"
               : MEB_F8(d, 0), MEB_F8(d, 8), MEB_F8(d, 16), MEB_F8(d, 24) : "l"(da), "l"(db), "r"(1), "n"(TA), "n"(TB));
}
// tf32: D[64 x N] += A[64 x 8] * B[8 x N] over fp32 words (the same 32 bytes of a row per k-step
// as the 16-bit forms).  The instruction has no transpose immediates: both operands K-major.
__device__ __forceinline__ void wgmma_16_tf32(float (&d)[8], uint64_t da, uint64_t db) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7}, "
               "%8, %9, p, 1, 1;\n\t}"
               : MEB_F8(d, 0) : "l"(da), "l"(db), "r"(1));
}
__device__ __forceinline__ void wgmma_32_tf32(float (&d)[16], uint64_t da, uint64_t db) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
               "%16, %17, p, 1, 1;\n\t}"
               : MEB_F8(d, 0), MEB_F8(d, 8) : "l"(da), "l"(db), "r"(1));
}
__device__ __forceinline__ void wgmma_64_tf32(float (&d)[32], uint64_t da, uint64_t db) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
               "%32, %33, p, 1, 1;\n\t}"
               : MEB_F8(d, 0), MEB_F8(d, 8), MEB_F8(d, 16), MEB_F8(d, 24) : "l"(da), "l"(db), "r"(1));
}
// e4m3: D[64 x N] += A[64 x 32] * B[32 x N] over fp8 e4m3 bytes (again 32 bytes of a row per
// k-step).  8-bit operands exist K-major only: no transpose immediates.  The tensor cores do not
// add these products into D in fp32 (DESIGN.md §3, "fp8 inference").
__device__ __forceinline__ void wgmma_16_e4m3(float (&d)[8], uint64_t da, uint64_t db) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n16k32.f32.e4m3.e4m3 {%0, %1, %2, %3, %4, %5, %6, %7}, "
               "%8, %9, p, 1, 1;\n\t}"
               : MEB_F8(d, 0) : "l"(da), "l"(db), "r"(1));
}
__device__ __forceinline__ void wgmma_32_e4m3(float (&d)[16], uint64_t da, uint64_t db) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n32k32.f32.e4m3.e4m3 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
               "%16, %17, p, 1, 1;\n\t}"
               : MEB_F8(d, 0), MEB_F8(d, 8) : "l"(da), "l"(db), "r"(1));
}
__device__ __forceinline__ void wgmma_64_e4m3(float (&d)[32], uint64_t da, uint64_t db) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n64k32.f32.e4m3.e4m3 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
               "%32, %33, p, 1, 1;\n\t}"
               : MEB_F8(d, 0), MEB_F8(d, 8), MEB_F8(d, 16), MEB_F8(d, 24) : "l"(da), "l"(db), "r"(1));
}
// e5m2 A times e4m3 B (the fp8 dgrad: gradients against weights), the same shapes and layouts.
__device__ __forceinline__ void wgmma_16_e5m2e4m3(float (&d)[8], uint64_t da, uint64_t db) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n16k32.f32.e5m2.e4m3 {%0, %1, %2, %3, %4, %5, %6, %7}, "
               "%8, %9, p, 1, 1;\n\t}"
               : MEB_F8(d, 0) : "l"(da), "l"(db), "r"(1));
}
__device__ __forceinline__ void wgmma_32_e5m2e4m3(float (&d)[16], uint64_t da, uint64_t db) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n32k32.f32.e5m2.e4m3 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
               "%16, %17, p, 1, 1;\n\t}"
               : MEB_F8(d, 0), MEB_F8(d, 8) : "l"(da), "l"(db), "r"(1));
}
__device__ __forceinline__ void wgmma_64_e5m2e4m3(float (&d)[32], uint64_t da, uint64_t db) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n64k32.f32.e5m2.e4m3 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
               "%32, %33, p, 1, 1;\n\t}"
               : MEB_F8(d, 0), MEB_F8(d, 8), MEB_F8(d, 16), MEB_F8(d, 24) : "l"(da), "l"(db), "r"(1));
}
// e4m3 A times e5m2 B (the fp8 wgrad: features against gradients), the same shapes and layouts.
// scale_d = 0: D = A * B, the accumulator's previous contents ignored (a promotion interval's start).
__device__ __forceinline__ void wgmma_32_e4m3e5m2(float (&d)[16], uint64_t da, uint64_t db,
                                                  uint32_t scale_d) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n32k32.f32.e4m3.e5m2 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
               "%16, %17, p, 1, 1;\n\t}"
               : MEB_F8(d, 0), MEB_F8(d, 8) : "l"(da), "l"(db), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_64_e4m3e5m2(float (&d)[32], uint64_t da, uint64_t db,
                                                  uint32_t scale_d) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n64k32.f32.e4m3.e5m2 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
               "%32, %33, p, 1, 1;\n\t}"
               : MEB_F8(d, 0), MEB_F8(d, 8), MEB_F8(d, 16), MEB_F8(d, 24) : "l"(da), "l"(db), "r"(scale_d));
}
#undef MEB_F8
template <int N>
__device__ __forceinline__ void wgmma_e4m3e5m2(float (&d)[N / 2], uint64_t da, uint64_t db,
                                               uint32_t scale_d) {
  static_assert(N == 32 || N == 64, "fp8 wgrad: N is 32 or 64");
  if constexpr (N == 32) wgmma_32_e4m3e5m2(d, da, db, scale_d);
  else wgmma_64_e4m3e5m2(d, da, db, scale_d);
}
template <int N>
__device__ __forceinline__ void wgmma_e4m3(float (&d)[N / 2], uint64_t da, uint64_t db) {
  static_assert(N == 16 || N == 32 || N == 64, "wgmma: N is 16, 32 or 64");
  if constexpr (N == 16) wgmma_16_e4m3(d, da, db);
  else if constexpr (N == 32) wgmma_32_e4m3(d, da, db);
  else wgmma_64_e4m3(d, da, db);
}
template <int N>
__device__ __forceinline__ void wgmma_e5m2e4m3(float (&d)[N / 2], uint64_t da, uint64_t db) {
  static_assert(N == 16 || N == 32 || N == 64, "wgmma: N is 16, 32 or 64");
  if constexpr (N == 16) wgmma_16_e5m2e4m3(d, da, db);
  else if constexpr (N == 32) wgmma_32_e5m2e4m3(d, da, db);
  else wgmma_64_e5m2e4m3(d, da, db);
}

// fp32 pair -> two e4m3 bytes (lo = a), rounded to nearest even; |x| past 448 (inf included)
// saturates to +-448, NaN stays NaN
__device__ __forceinline__ uint16_t e4m3x2_satfinite(float a, float b) {
  uint16_t r;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(b), "f"(a));
  return r;
}
// fp32 pair -> two e5m2 bytes (lo = a), the same rounding; saturates to +-57344
__device__ __forceinline__ uint16_t e5m2x2_satfinite(float a, float b) {
  uint16_t r;
  asm("cvt.rn.satfinite.e5m2x2.f32 %0, %1, %2;" : "=h"(r) : "f"(b), "f"(a));
  return r;
}

template <int N, int TA, int TB>
__device__ __forceinline__ void wgmma_tf32(float (&d)[N / 2], uint64_t da, uint64_t db) {
  static_assert(N == 16 || N == 32 || N == 64, "wgmma: N is 16, 32 or 64");
  static_assert(TA == 0 && TB == 0, "tf32 wgmma reads K-major operands only");
  if constexpr (N == 16) wgmma_16_tf32(d, da, db);
  else if constexpr (N == 32) wgmma_32_tf32(d, da, db);
  else wgmma_64_tf32(d, da, db);
}

// fp32 -> the nearest tf32 value (ties away from zero), kept in an fp32 word
__device__ __forceinline__ float tf32_rna(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}

// Warp-level D[16 x 8] += A[16 x 8] * B[8 x 8] in tf32 (fp32 words as stored), lane = 4g + t:
//   a = A[g][t], A[g + 8][t], A[g][t + 4], A[g + 8][t + 4];  b = B[t][g], B[t + 4][g]
//   d = D[g][2t], D[g][2t + 1], D[g + 8][2t], D[g + 8][2t + 1]
__device__ __forceinline__ void mma_tf32_16x8x8(float (&d)[4], const uint32_t (&a)[4],
                                                const uint32_t (&b)[2]) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, "
               "{%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

template <int N, bool BF16, int TA, int TB>
__device__ __forceinline__ void wgmma(float (&d)[N / 2], uint64_t da, uint64_t db) {
  static_assert(N == 16 || N == 32 || N == 64, "wgmma: N is 16, 32 or 64");
  if constexpr (N == 16) {
    if constexpr (BF16) wgmma_16_bf16<TA, TB>(d, da, db); else wgmma_16_f16<TA, TB>(d, da, db);
  } else if constexpr (N == 32) {
    if constexpr (BF16) wgmma_32_bf16<TA, TB>(d, da, db); else wgmma_32_f16<TA, TB>(d, da, db);
  } else {
    if constexpr (BF16) wgmma_64_bf16<TA, TB>(d, da, db); else wgmma_64_f16<TA, TB>(d, da, db);
  }
}

}  // namespace ptx
}  // namespace meb200
