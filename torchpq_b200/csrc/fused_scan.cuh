// What the host side of the fused GEMM searches shares (flat_search_kernel and flat_range_kernel in flat.cu,
// ivfflat_scan_kernel and ivfflat_range_kernel in ivfflat.cu): their shared-memory size and their launch.
#pragma once
#include <type_traits>
#include "gemm_tile.cuh"
#include "range.cuh"

namespace tpq {

constexpr int kFusedWarps = 8;

// Shared memory of one CTA: GEMM stages, then the consumer's part.  kp > 0, a top-k kernel: score tile [QT][128] f32 |
// lists [QT][kp] keys | staging [8][kTopkBuf] keys.  kp == 0, a range kernel: the match buffer (range.cuh; QT = 64:
// 24 + 81 = 105 KB, two CTAs per SM).
static inline size_t fused_smem_bytes(int qt, int kp) {
  const size_t stages = 2 * (size_t)GK * (qt + GB) * 4;
  if (kp == 0) return stages + sizeof(RangeBuf);
  return stages + (size_t)qt * GB * 4 + (size_t)qt * kp * 8 + (size_t)kFusedWarps * kTopkBuf * 8;
}

#ifdef __CUDACC__
// Launches the kernel pick(QT, METRIC) names -- both given as std::integral_constant -- for qt in {16, 32, 64} and the
// metric (inner only when INNER), with 256 threads and `smem` bytes of dynamic shared memory.
template <bool INNER, class Pick, class... Args>
static int fused_launch(const char* name, int qt, int metric, dim3 grid, size_t smem, cudaStream_t st, Pick pick,
                        Args... args) {
  auto by_metric = [&](auto q) {
    auto go = [&](auto m) {
      auto kern = pick(q, m);
      TPQ_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      kern<<<grid, 256, smem, st>>>(args...);
      TPQ_LAUNCH_CHECK(name);
      return (int)TPQ_OK;
    };
    if (metric == TPQ_METRIC_EUCLIDEAN) return go(std::integral_constant<int, TPQ_METRIC_EUCLIDEAN>{});
    if constexpr (INNER)
      if (metric == TPQ_METRIC_INNER) return go(std::integral_constant<int, TPQ_METRIC_INNER>{});
    return go(std::integral_constant<int, TPQ_METRIC_COSINE>{});
  };
  if (qt == 16) return by_metric(std::integral_constant<int, 16>{});
  if (qt == 32) return by_metric(std::integral_constant<int, 32>{});
  return by_metric(std::integral_constant<int, 64>{});
}
#endif  // __CUDACC__

}  // namespace tpq
