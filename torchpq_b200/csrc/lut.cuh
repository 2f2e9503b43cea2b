// The ADC look-up table (LUT): the arithmetic of one entry, the in-CTA builder of the scan kernels (scan.cu), and the
// staged LUT kernel's launcher (lut.cu).  Every LUT the library writes comes from the definitions here.
//
// Entry (m, row, code) of rows x (queries, or the cells of vq_codebook) against p = pq_codebook[m, :, code]
// (PQCodec.py:62-75, MultiKMeans.py:183-223, IVFPQIndex.py:160-170, 377):
//   dot = fmaf chain of x_m[i] * p[i], i ascending from +0
//   euclidean: ((dot * 2) - |x_m|^2) - |p|^2     |v|^2 a sum of separately rounded squares
//   cosine:    dot
//   part 1:    dot * 2                           residual IVFPQ, the query half
//   part 2:    (dot * -2) - nrm * nrm            residual IVFPQ, the cell half: nrm = sqrtf(fmaf chain of p[i]^2), the
//                                                way the reference's `.norm(dim=1).pow(2)` forms |p|^2
#pragma once
#include "scan_layout.cuh"

namespace tpq {

enum LutKind { kLutEuclidean = TPQ_METRIC_EUCLIDEAN, kLutCosine = TPQ_METRIC_COSINE, kLutPart1 = 2, kLutPart2 = 3 };
enum LutLayout {
  kLutReference,    // [M][n][256], the reference's `precomputed` layout
  kLutScan,         // [n][MG][256][64] (scan_layout.cuh), the rows of padding sub-quantizers m in [M, m_pad) +0
};

__device__ __forceinline__ float dot_step(float dot, float x, float p) { return fmaf(x, p, dot); }
// |v|^2 of the euclidean entry
__device__ __forceinline__ float sq_step(float s, float v) { return __fadd_rn(s, __fmul_rn(v, v)); }
// b2 of lut_entry: |p|^2 for every kind but part 2, whose norm is an fmaf chain
__device__ __forceinline__ float norm_step(int kind, float s, float v) { return kind == kLutPart2 ? fmaf(v, v, s) : sq_step(s, v); }

// a2 = |x_m|^2 (read by the euclidean kind only); b2 = the norm_step chain of p
__device__ __forceinline__ float lut_entry(int kind, float dot, float a2, float b2) {
  if (kind == kLutEuclidean) return __fsub_rn(__fsub_rn(__fmul_rn(dot, 2.f), a2), b2);
  if (kind == kLutPart1) return __fmul_rn(dot, 2.f);
  if (kind == kLutPart2) { const float nrm = sqrtf(b2); return __fsub_rn(__fmul_rn(dot, -2.f), __fmul_rn(nrm, nrm)); }
  return dot;
}

// The LUT of query q in scan layout (RES: the query half of the residual LUT), built by the NW warps of a CTA.  Lane l
// owns sub-quantizers m = 32 h + l: reads of the transposed codebook are contiguous across the warp, and so is every
// store (128 B), in shared or global memory.  CU: how many codes of the codebook loop are unrolled.
template <int MP, int NW, int DSUB, bool RES, int CU = (DSUB >= 8 ? 2 : 8)>
__device__ __forceinline__ void build_lut(float* lutf, const float* __restrict__ x, const float* __restrict__ cbt, int M,
                                          int nq, int q, int metric, int lane, int warp) {
  constexpr int NH = MP / 32;
  const int kind = RES ? kLutPart1 : metric == TPQ_METRIC_EUCLIDEAN ? kLutEuclidean : kLutCosine;
  float xr[NH][DSUB], a2[NH];
  #pragma unroll
  for (int h = 0; h < NH; ++h) {
    const int m = 32 * h + lane;
    float s2 = 0.f;
    #pragma unroll
    for (int i = 0; i < DSUB; ++i) {
      const float v = (m < M) ? __ldg(x + (size_t)(m * DSUB + i) * nq + q) : 0.f;
      xr[h][i] = v;
      s2 = sq_step(s2, v);
    }
    a2[h] = s2;
  }
  #pragma unroll CU
  for (int c = warp; c < 256; c += NW) {
    #pragma unroll
    for (int h = 0; h < NH; ++h) {
      const float* p = cbt + ((size_t)c * MP + 32 * h + lane) * DSUB;
      float pv[DSUB];
      if constexpr (DSUB == 2) { const float2 t = __ldg(reinterpret_cast<const float2*>(p)); pv[0] = t.x; pv[1] = t.y; }
      else if constexpr (DSUB % 4 == 0) {
        #pragma unroll
        for (int i = 0; i < DSUB; i += 4) {
          const float4 t = __ldg(reinterpret_cast<const float4*>(p + i));
          pv[i] = t.x; pv[i + 1] = t.y; pv[i + 2] = t.z; pv[i + 3] = t.w;
        }
      }
      else { for (int i = 0; i < DSUB; ++i) pv[i] = __ldg(p + i); }
      float dot = 0.f, b2 = 0.f;
      #pragma unroll
      for (int i = 0; i < DSUB; ++i) { dot = dot_step(dot, xr[h][i], pv[i]); b2 = sq_step(b2, pv[i]); }
      lutf[lut_index(32 * h + lane, c)] = lut_entry(kind, dot, a2[h], b2);
    }
  }
}

// The staged LUT (lut.cu): rows [r0, r0 + n) of x [d, ld] (column-major) against pq_codebook [M, d/M, 256], entries of
// `kind`, written to out in `layout` (row r0 first).  TPQ_ERR_UNSUPPORTED when one sub-vector does not fit in shared
// memory (d/M > kLutMaxDsub).
constexpr int kLutMaxDsub = (int)(kSmemLimit / 4) - 1;
int launch_lut(const float* x, int ld, int r0, int n, const float* pq_codebook, int d, int M, int kind, int layout,
               float* out, cudaStream_t st);

}  // namespace tpq
