// The staged ADC look-up table (entry arithmetic: lut.cuh), one kernel for every LUT that goes through global memory:
// tpq_build_lut's reference layout [M, nq, 256] (PQCodec.py:62-75; the reference uses a batched sgemm plus four passes),
// the search's scan-layout LUTs when d/M has no in-CTA build (scan.cu), and the residual cell half (relayout.cu).
#include "lut.cuh"

namespace tpq {

// CTA = 256 codes x mt sub-quantizers x qt rows: every codebook value is loaded once (coalesced over the code) and
// reused for qt rows; the rows' sub-vectors are read from shared memory.  The tile is kLutQT x kLutMT unless a wide
// d/M makes launch_lut shrink it: mt first, then qt to 1, whose register tile then repeats its one row.
// Each thread forms mt (sub-quantizer, code) entries per row.  Thread t takes code t for every sub-quantizer, so a warp
// stores 32 consecutive codes: whole 128-byte lines in the reference layout.  In the scan layout ([code][s] rows) that
// would be 32 scattered words per store, so a full tile there gives a warp 8 consecutive sub-quantizers x 4 codes
// instead: every store is 4 whole 32-byte sectors.
// KIND and LAYOUT are template parameters: the scan-layout instantiations a search launches then fit 32 registers
// (8 CTAs per SM) where one run-time kernel took 40.
constexpr int kLutQT = 8, kLutMT = 16;
template <int KIND, int LAYOUT>
__global__ void __launch_bounds__(256)
lut_kernel(const float* __restrict__ x, int ld, int r0, int n, const float* __restrict__ cb, int dsub, int M, int MR,
           int qt, int mt, float* __restrict__ out) {
  extern __shared__ __align__(16) float xs[];            // [qt][mt * dsub] sub-vectors, then [qt][mt] |x_m|^2
  const int m0 = blockIdx.y * mt;
  const int q0 = blockIdx.x * qt;                        // within the row range
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bool m_fast = LAYOUT == kLutScan && mt == kLutMT;
  float* a2s = xs + qt * mt * dsub;
  const int qs = qt == 1 ? 0 : mt * dsub;                // register-tile row qq reads sub-vectors at qq * qs
  for (int i = threadIdx.x; i < qt * mt * dsub; i += blockDim.x) {
    const int qq = i / (mt * dsub), row = m0 * dsub + i % (mt * dsub);
    xs[i] = (q0 + qq < n && row < M * dsub) ? x[(size_t)row * ld + r0 + q0 + qq] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < qt * mt; i += blockDim.x) {
    const float* v = xs + (size_t)i * dsub;
    float a2 = 0.f;
    for (int e = 0; e < dsub; ++e) a2 = sq_step(a2, v[e]);
    a2s[i] = a2;
  }
  __syncthreads();
  for (int j = 0; j < mt; ++j) {
    const int mm = m_fast ? (lane & 7) + 8 * (warp & 1) : j;
    const int c = m_fast ? (lane >> 3) + 4 * (warp >> 1) + 16 * j : threadIdx.x;
    const int m = m0 + mm;
    if (m >= MR) continue;
    float dot[kLutQT];
    #pragma unroll
    for (int qq = 0; qq < kLutQT; ++qq) dot[qq] = 0.f;
    float b2 = 0.f;
    if (m < M) {
      const float* p = cb + (size_t)m * dsub * 256 + c;
      #pragma unroll 4
      for (int e = 0; e < dsub; ++e) {
        const float pv = __ldg(p + (size_t)e * 256);
        b2 = norm_step(KIND, b2, pv);
        #pragma unroll
        for (int qq = 0; qq < kLutQT; ++qq) dot[qq] = dot_step(dot[qq], xs[qq * qs + mm * dsub + e], pv);
      }
    }
    #pragma unroll
    for (int qq = 0; qq < kLutQT; ++qq) {
      const int q = q0 + qq;
      if (qq >= qt || q >= n) break;
      const float y = m < M ? lut_entry(KIND, dot[qq], a2s[qq * mt + mm], b2) : 0.f;
      out[LAYOUT == kLutScan ? (size_t)q * lut_groups(MR) * kLutGroup + lut_index(m, c) : ((size_t)m * n + q) * 256 + c] = y;
    }
  }
}

// the instantiations that exist: the reference layout holds the metrics, the scan layout every kind
using LutKernel = decltype(&lut_kernel<kLutEuclidean, kLutScan>);
static LutKernel lut_kernel_of(int kind, int layout) {
  if (layout == kLutReference) return kind == kLutEuclidean ? lut_kernel<kLutEuclidean, kLutReference> : lut_kernel<kLutCosine, kLutReference>;
  switch (kind) {
    case kLutEuclidean: return lut_kernel<kLutEuclidean, kLutScan>;
    case kLutCosine:    return lut_kernel<kLutCosine, kLutScan>;
    case kLutPart1:     return lut_kernel<kLutPart1, kLutScan>;
    default:            return lut_kernel<kLutPart2, kLutScan>;
  }
}

int launch_lut(const float* x, int ld, int r0, int n, const float* pq_codebook, int d, int M, int kind, int layout,
               float* out, cudaStream_t st) {
  const int dsub = d / M;
  if (n == 0) return TPQ_OK;
  if (dsub > kLutMaxDsub) {
    set_error("LUT: d/M = %d > %d does not fit one sub-vector in 227 KB of shared memory", dsub, kLutMaxDsub);
    return TPQ_ERR_UNSUPPORTED;
  }
  int qt = kLutQT, mt = kLutMT;
  auto smem = [&] { return (size_t)qt * mt * (dsub + 1) * 4; };
  while (smem() > kSmemLimit) { if (mt > 1) mt /= 2; else qt = 1; }
  const LutKernel kern = lut_kernel_of(kind, layout);
  if (smem() > 48 * 1024) TPQ_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem()));
  const int MR = layout == kLutScan ? scan_m_pad(M) : M;
  const dim3 grid((n + qt - 1) / qt, (MR + mt - 1) / mt);
  kern<<<grid, 256, smem(), st>>>(x, ld, r0, n, pq_codebook, dsub, M, MR, qt, mt, out);
  TPQ_LAUNCH_CHECK("lut_kernel");
  return TPQ_OK;
}

}  // namespace tpq

using namespace tpq;

extern "C" int tpq_build_lut(const float* x_dn, const float* pq_codebook, int d, int M, int nq, int metric,
                             float* lut_mqk, void* stream) {
  TPQ_REQUIRE(x_dn && pq_codebook && lut_mqk, "tpq_build_lut: null pointer");
  TPQ_REQUIRE(d > 0 && M > 0 && d % M == 0, "d_vector=%d must be a multiple of n_subvectors=%d", d, M);
  TPQ_REQUIRE(metric == TPQ_METRIC_EUCLIDEAN || metric == TPQ_METRIC_COSINE, "unsupported metric %d", metric);
  TPQ_REQUIRE(nq >= 0, "bad n_query");
  return launch_lut(x_dn, nq, 0, nq, pq_codebook, d, M, metric, kLutReference, lut_mqk, (cudaStream_t)stream);
}
