// PTX wrappers and layout helpers shared by the Hopper tensor-core assignment kernels (assign_tc.cu, assign_wide.cu):
// mbarrier, TMA, wgmma TF32 descriptors, the 128-byte-swizzle address maps and the packed arg-max key.
#pragma once
#include <cuda.h>
#include "common.cuh"

namespace tpq {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t}"
      :: "r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      :: "r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
// contiguous global -> shared copy by the TMA unit (bytes % 16 == 0, both ends 16-byte aligned)
__device__ __forceinline__ void bulk_load(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               :: "r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

// wgmma shared-memory matrix descriptor, K-major operand with the 128-byte swizzle: 8-row x 128-byte atoms, rows
// 128 bytes apart, atoms SBO = 1024 bytes apart along N; LBO is unused for swizzled K-major layouts (encoded 1).
// Fields: start>>4 [0,14) | LBO>>4 [16,30) | SBO>>4 [32,46) | layout 1 = SWIZZLE_128B [62,64).
__device__ __forceinline__ uint64_t gmma_desc(uint32_t saddr) {
  return (uint64_t)((saddr & 0x3FFFF) >> 4) | (1ull << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}
// byte offset of element (row n, k) in a K-major SWIZZLE_128B region of 32-element (128-byte) rows
__device__ __forceinline__ uint32_t kmaj_off(int n, int k) {
  return (uint32_t)((n >> 3) * 1024 + (n & 7) * 128 + ((((k >> 2) ^ n) & 7) << 4) + (k & 3) * 4);
}
// element (row e, column c) of a [rows x 32-column] fp32 TMA box written with the 128-byte swizzle
__device__ __forceinline__ uint32_t box_off(int e, int c) {
  return (uint32_t)(e * 128 + ((((c >> 2) ^ e) & 7) << 4) + (c & 3) * 4);
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait1() { asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory"); }

// Arg-max key of (score, column j < 256): the score with its 8 low mantissa bits replaced by an index field (a
// perturbation below 2^-15 relative, far below the TF32 rounding of the score itself), so one fmaxf per column replaces
// compare + two selects and the larger key always has the larger truncated score.  Among equal truncated scores the
// LOWEST column has the largest key, for either sign: a positive float grows with its low bits, so the field is
// 255 - j; a negative one shrinks, so the field is (255 - j) ^ 255 = j.  (The 8 masked bits still separate every two
// scores that differ by 2^-3 or more while |score| < 2^13.)
// Two instructions: PRMT = bytes 3..1 of the score and, as byte 0, its sign bit replicated (0x00 or 0xFF); LOP3 = XOR
// with rcol = 255 ^ j (= 255 - j), which the caller splits into a per-thread register and an immediate.
// A score of -0 would lose to +0 here, but the accumulator never holds -0: its last MMA adds the bias K-block, six of
// whose products are 0 * 0 = +0, and the tensor core returns +0 for an exact-zero sum even when every other product
// is -0 (test_max_sim_tensor_core_signed_zero_ties pins that on the GPU), so ties at zero are ties of +0.  (Turning -0
// into +0 here, score + 0, costs one FADD per column, about 10 % of the kernel at C5.)
__device__ __forceinline__ float argmax_key(float score, uint32_t rcol /* 255 ^ j */) {
  uint32_t u;
  asm("prmt.b32 %0, %1, 0, 0x321B;" : "=r"(u) : "r"(__float_as_uint(score)));
  return __uint_as_float(u ^ rcol);
}
// the column j of an arg-max key: undoes the sign-dependent index field
__device__ __forceinline__ int argmax_key_column(float key) {
  const uint32_t u = __float_as_uint(key);
  return 255 - (int)((u ^ (uint32_t)((int32_t)u >> 31)) & 0xFFu);
}
// the score of an arg-max key with its index field cleared (truncated toward zero): equal for equal truncated scores
__device__ __forceinline__ float argmax_key_score(float key) { return __uint_as_float(__float_as_uint(key) & 0xFFFFFF00u); }

// ----------------------------------------------------------------------------- host
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static inline EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

}  // namespace tpq
