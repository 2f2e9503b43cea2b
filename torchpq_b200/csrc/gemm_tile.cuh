// The exact fp32 distance GEMM tile shared by the coarse probe (coarse.cu), the flat search (flat.cu) and the IVF
// scans (ivfflat.cu, with fp32 or SQ-coded stores), and the column reductions they launch (defined in coarse.cu).
#pragma once
#include "common.cuh"
#ifdef __CUDACC__
#include <cuda_fp16.h>
#endif

namespace tpq {

// ----------------------------------------------------------------------------- column reductions (coarse.cu)
// x is [d, n] with row stride ld.  Each launches one kernel on `st`; n == 0 launches nothing.
//   col_sqnorms:       out[j] = sum_i x[i, j]^2, squares separately rounded (torch's (a ** 2).sum(dim=-2))
//   col_norms:         out[j] = sqrtf(fmaf chain of x[i, j]^2) + eps, the divisor of normalize_columns
//   normalize_columns: out[:, j] = x[:, j] / col_norms(x, eps)[j]   (out is [d, n], row stride n)
int col_sqnorms(const float* x, int d, int64_t n, int64_t ld, float* out, cudaStream_t st);
int col_norms(const float* x, int d, int64_t n, int64_t ld, float eps, float* out, cudaStream_t st);
int normalize_columns(const float* x, int d, int n, float eps, float* out, cudaStream_t st);

#ifdef __CUDACC__
// ----------------------------------------------------------------------------- QT x 128 GEMM tile
// 256 threads as a 16 x 16 grid; thread (ty, tx) owns a (QT/16) x 8 micro-tile, its rows and columns each split in
// 4-wide groups 64 apart (fewer and narrower rows for QT < 64), so that every shared-memory read is a conflict-free
// vector.  K step 16, two shared-memory stages: the next K-slab is fetched into registers while the current one is
// multiplied, one barrier per slab.
constexpr int GB = 128, GK = 16;

// ----------------------------------------------------------------------------- B-operand loaders
// A loader owns how GemmTile reads its B operand: fetch() loads the K slab [k0, k0 + 16) x 128 columns of the tile into
// registers (with whatever stash() needs to know of the slab), stash() stores it as fp32 into a shared-memory stage, 0
// for rows k >= d and columns >= cols.  A loader is built from the tile's first column (a T*), the row stride and the
// loader's own extra pointers.  Element e = r * 256 + tid of a slab is (row e >> 7, column e & 127).

// fp32 [d, *] with row stride ld (the coarse codebook, FlatIndex's and IVFFlatIndex's stores): 8 floats per thread
struct BLoadF32 {
  using T = float;
  const float* __restrict__ bt;
  int64_t ld;
  using Regs = float[8];
  __device__ __forceinline__ void fetch(int k0, int d, int cols, int tid, Regs& r) const {
    #pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int e = i * 256 + tid, kk = e >> 7, c = e & 127, gk = k0 + kk;
      r[i] = (gk < d && c < cols) ? __ldg(bt + (size_t)gk * ld + c) : 0.f;
    }
  }
  __device__ __forceinline__ void stash(const Regs& r, int, int, int tid, float (&B)[2][GK][GB], int buf) const {
    #pragma unroll
    for (int i = 0; i < 8; ++i) { const int e = i * 256 + tid; B[buf][e >> 7][e & 127] = r[i]; }
  }
};

// SQCodec 8-bit word planes (IVFSQIndex's store, d % 4 == 0): word w of column c is words[w * ld + c], its byte b the
// code of dimension 4 w + b.  A slab is 4 word rows x 128 columns, 2 words per thread, coalesced along the column.
// stash() decodes as tpq_sq_decode: ((code / 256) * range[k]) + lower[k], each step rounded (no fma); lower and range
// are 16-byte aligned [d] f32, read 4 dimensions at a time through the read-only cache.
struct BLoadSQ8 {
  using T = uint32_t;
  const uint32_t* __restrict__ words;
  int64_t ld;
  const float* __restrict__ lower;
  const float* __restrict__ range;
  struct Regs { uint32_t w[2]; int k0; };
  __device__ __forceinline__ void fetch(int k0, int d, int cols, int tid, Regs& r) const {
    r.k0 = k0;
    #pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int e = i * 256 + tid, wr = e >> 7, c = e & 127, gk = k0 + 4 * wr;
      r.w[i] = (gk < d && c < cols) ? __ldg(words + (size_t)(gk >> 2) * ld + c) : 0u;
    }
  }
  __device__ __forceinline__ void stash(const Regs& r, int d, int cols, int tid, float (&B)[2][GK][GB], int buf) const {
    #pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int e = i * 256 + tid, wr = e >> 7, c = e & 127, gk = r.k0 + 4 * wr;
      const bool ok = gk < d && c < cols;
      const float4 lo = ok ? __ldg(reinterpret_cast<const float4*>(lower + gk)) : make_float4(0.f, 0.f, 0.f, 0.f);
      const float4 rg = ok ? __ldg(reinterpret_cast<const float4*>(range + gk)) : make_float4(0.f, 0.f, 0.f, 0.f);
      const float l[4] = {lo.x, lo.y, lo.z, lo.w}, g[4] = {rg.x, rg.y, rg.z, rg.w};
      #pragma unroll
      for (int b = 0; b < 4; ++b) {
        // code / 256 is exact, so the multiply by 2^-8 is the reference's division
        const float q = __fmul_rn((float)((r.w[i] >> (8 * b)) & 0xFFu), 0.00390625f);
        B[buf][4 * wr + b][c] = ok ? __fadd_rn(__fmul_rn(q, g[b]), l[b]) : 0.f;
      }
    }
  }
};

// SQCodec 16-bit word planes (d % 2 == 0): the low half of word w is the fp16 code of dimension 2 w, the high half of
// 2 w + 1.  A slab is 8 word rows x 128 columns, 4 words per thread; a zero word (outside the tile) decodes to +0.
struct BLoadSQ16 {
  using T = uint32_t;
  const uint32_t* __restrict__ words;
  int64_t ld;
  struct Regs { uint32_t w[4]; };
  __device__ __forceinline__ void fetch(int k0, int d, int cols, int tid, Regs& r) const {
    #pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int e = i * 256 + tid, wr = e >> 7, c = e & 127, gk = k0 + 2 * wr;
      r.w[i] = (gk < d && c < cols) ? __ldg(words + (size_t)(gk >> 1) * ld + c) : 0u;
    }
  }
  __device__ __forceinline__ void stash(const Regs& r, int, int, int tid, float (&B)[2][GK][GB], int buf) const {
    #pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int e = i * 256 + tid, wr = e >> 7, c = e & 127;
      B[buf][2 * wr][c] = __half2float(__ushort_as_half((unsigned short)(r.w[i] & 0xFFFFu)));
      B[buf][2 * wr + 1][c] = __half2float(__ushort_as_half((unsigned short)(r.w[i] >> 16)));
    }
  }
};

template <int QT, class BLoad = BLoadF32>
struct GemmTile {
  static_assert(QT == 16 || QT == 32 || QT == 64 || QT == 128, "QT is 16, 32, 64 or 128");
  static constexpr int MI = QT / 16;                  // rows per thread
  static constexpr int H = MI < 4 ? MI : 4;           // rows per shared-memory vector read
  struct Stages { float A[2][GK][QT]; float B[2][GK][GB]; };

  // tile row of register row i of thread row ty; tile column of register column j of thread column tx
  __device__ static __forceinline__ int row(int i, int ty) { return (i / H) * (16 * H) + ty * H + (i % H); }
  __device__ static __forceinline__ int col(int j, int tx) { return (j / 4) * 64 + tx * 4 + (j % 4); }

  // acc[i][j] = sum over k ascending of x[k, q0 + row(i)] * bt[k, col(j)]: one fmaf chain from +0 per entry
  // (zero-padded K slabs, rows >= nq and columns >= cols add nothing), so a score does not depend on the tiling.
  // x is [d, nq] (row stride nq); bt is the tile's first column of a [d, *] matrix with row stride ld, of which `cols`
  // are valid (a pointer and an int rather than a 64-bit column index keep the coarse instance at 127 registers, two
  // CTAs per SM).  Ends with every thread's reads of `s` issued but without a barrier: the caller separates this
  // tile's last reads from the next tile's first writes.
  __device__ static __forceinline__ void run(const float* __restrict__ x, int nq, int q0,
                                             const float* __restrict__ bt, int64_t ld, int cols, int d,
                                             Stages& s, float (&acc)[MI][8]) {
    run(x, nq, q0, BLoadF32{bt, ld}, cols, d, s, acc);
  }

  // The same with B read through a loader (b: the tile's first column); the product is over B as the loader stashes
  // it, so a decoded store scores exactly as its fp32 image does.  b is taken by value: by reference, ptxas numbered
  // the registers of the fp32 instances differently from the loader-less tile this replaced.
  __device__ static __forceinline__ void run(const float* __restrict__ x, int nq, int q0, const BLoad b, int cols,
                                             int d, Stages& s, float (&acc)[MI][8]) {
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    #pragma unroll
    for (int i = 0; i < MI; ++i)
      #pragma unroll
      for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
    float ra[MI];
    typename BLoad::Regs rb;
    auto fetch = [&](int k0) {                        // 16 x QT and 16 x 128 floats: MI and 8 per thread
      #pragma unroll
      for (int r = 0; r < MI; ++r) {
        const unsigned e = r * 256 + tid;              // unsigned: / and % by QT are shifts and masks
        const int kk = e / QT, c = e % QT, gk = k0 + kk;
        ra[r] = (gk < d && q0 + c < nq) ? __ldg(x + (size_t)gk * nq + q0 + c) : 0.f;
      }
      b.fetch(k0, d, cols, tid, rb);
    };
    auto stash = [&](int buf) {
      #pragma unroll
      for (int r = 0; r < MI; ++r) { const unsigned e = r * 256 + tid; s.A[buf][e / QT][e % QT] = ra[r]; }
      b.stash(rb, d, cols, tid, s.B, buf);
    };
    fetch(0);
    stash(0);
    __syncthreads();
    int cur = 0;
    for (int k0 = 0; k0 < d; k0 += GK) {
      const bool more = k0 + GK < d;
      if (more) fetch(k0 + GK);
      #pragma unroll
      for (int kk = 0; kk < GK; ++kk) {
        float a[MI];
        #pragma unroll
        for (int h = 0; h < MI / H; ++h) {
          const float* p = &s.A[cur][kk][h * 16 * H + ty * H];
          if constexpr (H == 4) {
            const float4 v = *reinterpret_cast<const float4*>(p);
            a[h * 4 + 0] = v.x; a[h * 4 + 1] = v.y; a[h * 4 + 2] = v.z; a[h * 4 + 3] = v.w;
          } else if constexpr (H == 2) {
            const float2 v = *reinterpret_cast<const float2*>(p);
            a[h * 2 + 0] = v.x; a[h * 2 + 1] = v.y;
          } else {
            a[h] = *p;
          }
        }
        const float4 b0 = *reinterpret_cast<const float4*>(&s.B[cur][kk][tx * 4]);
        const float4 b1 = *reinterpret_cast<const float4*>(&s.B[cur][kk][64 + tx * 4]);
        const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
        #pragma unroll
        for (int i = 0; i < MI; ++i)
          #pragma unroll
          for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], bv[j], acc[i][j]);
      }
      if (more) {
        stash(cur ^ 1);                               // the other stage was last read one iteration ago
        __syncthreads();
        cur ^= 1;
      }
    }
  }
};
#endif  // __CUDACC__

}  // namespace tpq
