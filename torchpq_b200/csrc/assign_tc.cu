// MultiKMeans assignment on the Hopper tensor cores (wgmma TF32 + TMA + mbarrier), sm_90a.
//
// Replaces the reference's fused SIMT distance-GEMM + arg-max (torchpq/kernels/cuda/max_sim.cu:182-309,
// 128x128 tiles, 8x8 register micro-tiles, float atomicMax epilogue) for the shape the PQ codec uses
// (MultiKMeans.get_labels, clustering/MultiKMeans.py:314-333): data [l, d, n], centroids [l, d, k<=256].
//
//   label_i = argmax_j ( 2 <x_i, c_j> - |c_j|^2 )         (|x_i|^2 does not change the arg-max)
//
// The inner products run as TF32 wgmma (M=64 points x N=64 centroids x K=8 per instruction, up to four N chunks),
// accumulators in registers.  The points are streamed by TMA exactly as they lie in HBM (points contiguous, 32-point
// boxes with the 128-byte swizzle).  wgmma takes TF32 operands from shared memory only K-major, so A (the points, which
// are MN-major in HBM) is fed from REGISTERS: each thread loads its fragment from the swizzled tile, which is the
// transposition for free.  B (the centroids, <= 64 KB per k-means) is written K-major into shared memory by the
// consumer threads once per k-means, together with one extra K-block that adds -|c_j|^2/2 as (hi, lo) TF32 rows
// against a constant "ones" A fragment -- the accumulator then holds <x,c> - |c|^2/2, whose arg-max is the label.
// The value written to `maxsims` is recomputed EXACTLY (fp32, fmaf(-dif, dif, acc), e ascending, as
// max_sim.cu:78-98) for the chosen centroid from the same shared-memory tiles, so values are bit-identical to the
// exact kernel wherever the label agrees; labels can differ only where two centroids are within TF32 rounding
// (~1e-3 relative) of each other.
//
// Persistent, warp-specialised: warpgroup 0 = TMA producer (one thread), warpgroups 1 and 2 = consumers taking
// alternate 64-point tiles, so one consumer's arg-max epilogue overlaps the other's MMAs.
#include "tc_common.cuh"

namespace tpq {

constexpr int TC_M = 64;           // points per tile = M of one wgmma
constexpr int TC_STAGES = 6;
constexpr int TC_THREADS = 3 * 128;

// the two consumer warpgroups (named barrier 1; barrier 0 is __syncthreads)
__device__ __forceinline__ void consumers_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// D[64 x 64] (+)= A[64 x 8] (registers, TF32) * B[8 x 64] (shared memory, K-major)
__device__ __forceinline__ void wgmma_m64n64k8_tf32(float (&d)[32], const uint32_t (&a)[4], uint64_t desc_b, int accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "{%32, %33, %34, %35}, %36, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(accumulate)
      : "memory");
}

// argmax_key / argmax_key_column: tc_common.cuh

struct TcParams {
  int l, d, n, k;
  int nch;                       // 64-centroid chunks: N of the problem = 64 * nch >= k
  int tiles_per_l;               // ceil(n / 64)
  float* maxsims; int64_t* labels;
  const float* cent;             // [l, d, k]
  int exact_values;              // 1: maxsims recomputed exactly in fp32 for the chosen centroid; 0: 2*score - |x|^2 from the TF32 score
};

// KB = d / 8 K-steps, NCH = P.nch: both compile-time, so every wgmma is issued unconditionally (a wgmma under a
// run-time branch makes ptxas serialise the accumulator chain).
template <int KB, int NCH>
__global__ void __launch_bounds__(TC_THREADS, 1)
assign_tc_kernel(const __grid_constant__ CUtensorMap map_x, TcParams P) {
  extern __shared__ __align__(1024) uint8_t smem[];
  constexpr int d = 8 * KB;
  constexpr int n_kreg = (d + 31) / 32;                                 // K-major B regions of 32 features
  constexpr uint32_t reg_bytes = (uint32_t)NCH * 64 * 128;              // one region: 64*NCH rows x 128 bytes
  const uint32_t box_bytes = (uint32_t)d * 128;                         // one 32-point box
  const uint32_t a_bytes = 2 * box_bytes;
  uint8_t* sB = smem;                                                   // [n_kreg] regions, then the -|c|^2/2 region
  uint8_t* sBias = sB + n_kreg * reg_bytes;
  uint8_t* sA = sBias + reg_bytes;                                      // every region / box is a multiple of 1024 bytes
  uint64_t* full = reinterpret_cast<uint64_t*>(sA + TC_STAGES * a_bytes);
  uint64_t* empty = full + TC_STAGES;

  const int wg = threadIdx.x >> 7, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long total_tiles = (long long)P.l * P.tiles_per_l;
  // contiguous tile range per CTA: one or two centroid-set loads per CTA
  const long long t_begin = total_tiles * blockIdx.x / gridDim.x;
  const long long t_end = total_tiles * (blockIdx.x + 1) / gridDim.x;

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" :: "l"(&map_x) : "memory");
    for (int s = 0; s < TC_STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 4); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (wg == 0) {
    // ===================================================== TMA producer
    if (warp == 0 && lane == 0) {
      long long it = 0;
      for (long long t = t_begin; t < t_end; ++t, ++it) {
        const int li = (int)(t / P.tiles_per_l), ti = (int)(t % P.tiles_per_l);
        const int s = (int)(it % TC_STAGES); const uint32_t ph = (uint32_t)(it / TC_STAGES) & 1;
        mbar_wait(&empty[s], ph ^ 1);
        mbar_expect_tx(&full[s], a_bytes);
        for (int g = 0; g < 2; ++g) tma_load_3d(sA + s * a_bytes + g * box_bytes, &map_x, &full[s], ti * TC_M + g * 32, 0, li);
      }
    }
    return;
  }

  // ===================================================== consumers: warpgroup c takes the tiles with (t - t_begin) % 2 == c
  const int c = wg - 1;
  const int ctid = threadIdx.x - 128;                                   // 0..255 over both consumer warpgroups
  const int w4 = warp & 3;                                              // warp inside the warpgroup: rows [16 w4, +16)
  const int g = lane >> 2, tq = lane & 3;
  const int r0 = 16 * w4 + g, r1 = r0 + 8;                              // the two tile rows (points) of this thread
  for (long long seg = t_begin; seg < t_end;) {                        // one segment per k-means in the CTA's range
    const int li = (int)(seg / P.tiles_per_l);
    const long long seg_end = min(t_end, (long long)(li + 1) * P.tiles_per_l);
    {
      // new centroid set: both consumers are done with the old one, then write it K-major (+ the bias K-block).
      // (The transition lives outside the tile loop: a wgmma after a possibly divergent branch is serialised by ptxas.)
      consumers_sync();
      const float* C = P.cent + (size_t)li * d * P.k;
      for (int j = ctid; j < NCH * 64; j += 256) {
        float v = -1e30f;                                               // padded columns can never win
        if (j < P.k) {
          float s2 = 0.f;
          for (int e = 0; e < d; ++e) {
            const float cv = C[(size_t)e * P.k + j];
            s2 = fmaf(cv, cv, s2);
            *reinterpret_cast<float*>(sB + (e >> 5) * reg_bytes + kmaj_off(j, e & 31)) = cv;
          }
          v = -0.5f * s2;
        } else {
          for (int e = 0; e < d; ++e) *reinterpret_cast<float*>(sB + (e >> 5) * reg_bytes + kmaj_off(j, e & 31)) = 0.f;
        }
        const float hi = __uint_as_float(__float_as_uint(v) & 0xFFFFE000u);   // exactly representable in TF32
        #pragma unroll
        for (int e = 0; e < 8; ++e)
          *reinterpret_cast<float*>(sBias + kmaj_off(j, e)) = e == 0 ? hi : (e == 1 ? v - hi : 0.f);
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> visible to wgmma
      consumers_sync();
    }
    // tile t (local index it = t - t_begin) belongs to consumer it % 2
    for (long long t = seg + ((seg - t_begin + c) & 1); t < seg_end; t += 2) {
      const long long it = t - t_begin;
      const int ti = (int)(t % P.tiles_per_l);
      const int s = (int)(it % TC_STAGES); const uint32_t ph = (uint32_t)(it / TC_STAGES) & 1;
      mbar_wait(&full[s], ph);
      // A fragments (wgmma m64nNk8 TF32 register layout): a0 = (r0, tq), a1 = (r1, tq), a2 = (r0, tq+4), a3 = (r1, tq+4)
      const uint8_t* xa = sA + s * a_bytes + (r0 >> 5) * box_bytes;       // r0 and r1 lie in the same 32-point box
      uint32_t a[KB][4];
      float x2a = 0.f, x2b = 0.f;
      #pragma unroll
      for (int q = 0; q < KB; ++q) {
        const int e = 8 * q + tq;
        const float v0 = *reinterpret_cast<const float*>(xa + box_off(e, r0 & 31));
        const float v1 = *reinterpret_cast<const float*>(xa + box_off(e, r1 & 31));
        const float v2 = *reinterpret_cast<const float*>(xa + box_off(e + 4, r0 & 31));
        const float v3 = *reinterpret_cast<const float*>(xa + box_off(e + 4, r1 & 31));
        a[q][0] = __float_as_uint(v0); a[q][1] = __float_as_uint(v1);
        a[q][2] = __float_as_uint(v2); a[q][3] = __float_as_uint(v3);
        x2a = fmaf(v0, v0, fmaf(v2, v2, x2a));
        x2b = fmaf(v1, v1, fmaf(v3, v3, x2b));
      }
      if (!P.exact_values) {                                              // the tile is in registers: release the stage now
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[s]);
      }
      const float one = tq < 2 ? 1.f : 0.f;                               // A columns 0, 1 of the bias K-block = 1
      const uint32_t ones[4] = {__float_as_uint(one), __float_as_uint(one), 0u, 0u};
      // Packed arg-max (argmax_key): the column index rides in the 8 low mantissa bits of the score, so a running fmaxf
      // over the packed keys of all columns and chunks is the arg-max with lowest-index ties.
      // Accumulator layout: acc[h][4i + {0,1}] = row r0, columns 64 ch + 8 i + 2 tq + {0,1}; acc[h][4i + {2,3}] = row
      // r1, same columns.  Two 64-column chunks per pass keep the accumulators at 64 registers.
      float b0 = -3.0e38f, b1 = -3.0e38f;                                 // below every key (a padded column's is ~-1e30)
      // 255 ^ column: columns 64 ch + 8 i + 2 tq + {0,1} have disjoint bit fields, so 255 ^ j = base ^ (64 ch + 8 i + b)
      const uint32_t base = 255u ^ (2u * (uint32_t)tq);
      #pragma unroll
      for (int c0 = 0; c0 < NCH; c0 += 2) {
        const int nh = NCH - c0 < 2 ? 1 : 2;                              // compile-time after unrolling
        float acc[2][32];
        #pragma unroll
        for (int h = 0; h < 2; ++h)
          #pragma unroll
          for (int i = 0; i < 32; ++i) acc[h][i] = 0.f;
        wgmma_fence();
        #pragma unroll
        for (int q = 0; q < KB; ++q) {
          const uint32_t bq = smem_u32(sB + (q >> 2) * reg_bytes) + (q & 3) * 32;
          #pragma unroll
          for (int h = 0; h < nh; ++h) wgmma_m64n64k8_tf32(acc[h], a[q], gmma_desc(bq + (c0 + h) * 8 * 1024), q > 0);
        }
        #pragma unroll
        for (int h = 0; h < nh; ++h) wgmma_m64n64k8_tf32(acc[h], ones, gmma_desc(smem_u32(sBias) + (c0 + h) * 8 * 1024), 1);
        wgmma_commit();
        wgmma_wait0();
        #pragma unroll
        for (int h = 0; h < nh; ++h) {
          float cb0 = -3.0e38f, cb1 = -3.0e38f;
          #pragma unroll
          for (int i = 0; i < 8; ++i) {
            const uint32_t i0 = base ^ (uint32_t)(64 * (c0 + h) + 8 * i), i1 = i0 ^ 1u;
            cb0 = fmaxf(cb0, fmaxf(argmax_key(acc[h][4 * i + 0], i0), argmax_key(acc[h][4 * i + 1], i1)));
            cb1 = fmaxf(cb1, fmaxf(argmax_key(acc[h][4 * i + 2], i0), argmax_key(acc[h][4 * i + 3], i1)));
          }
          b0 = fmaxf(b0, cb0);
          b1 = fmaxf(b1, cb1);
        }
      }
      #pragma unroll
      for (int o = 1; o <= 2; o <<= 1) {                                  // the 4 threads of a quad share rows r0, r1
        b0 = fmaxf(b0, __shfl_xor_sync(0xffffffffu, b0, o));
        b1 = fmaxf(b1, __shfl_xor_sync(0xffffffffu, b1, o));
        x2a += __shfl_xor_sync(0xffffffffu, x2a, o);
        x2b += __shfl_xor_sync(0xffffffffu, x2b, o);
      }
      const int bi0 = argmax_key_column(b0), bi1 = argmax_key_column(b1);
      // finisher: threads tq = 0, 2 take row r0, tq = 1, 3 row r1 (all compute: no divergent path before the next
      // tile's wgmma), tq = 0, 1 store
      {
        const int row = (tq & 1) ? r1 : r0;
        const float best = (tq & 1) ? b1 : b0;
        const int besti = (tq & 1) ? bi1 : bi0;
        float out;
        if (P.exact_values) {
          // exact fp32 similarity of the chosen centroid (max_sim.cu:78-98 arithmetic)
          const uint8_t* xr = sA + s * a_bytes + (row >> 5) * box_bytes;
          float acc1 = 0.f;
          for (int e = 0; e < d; ++e) {
            const float xv = *reinterpret_cast<const float*>(xr + box_off(e, row & 31));
            const float cv = *reinterpret_cast<const float*>(sB + (e >> 5) * reg_bytes + kmaj_off(besti, e & 31));
            const float dif = xv - cv;
            acc1 = fmaf(-dif, dif, acc1);
          }
          out = acc1;
        } else {
          out = fmaf(2.f, best, -((tq & 1) ? x2b : x2a));                 // -|x - c|^2 = 2 (<x,c> - |c|^2/2) - |x|^2
        }
        const long long p = (long long)ti * TC_M + row;
        if (tq < 2 && p < P.n) {
          P.maxsims[(size_t)li * P.n + p] = out;
          P.labels[(size_t)li * P.n + p] = besti;
        }
      }
      if (P.exact_values) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[s]);                            // this warp is done reading the A stage
      }
    }
    seg = seg_end;
  }
}

// ----------------------------------------------------------------------------- host
// [l][rows][cols] fp32, cols contiguous; box = 32 cols x rows x 1, 128-byte swizzle, zero fill out of bounds
static int make_map(CUtensorMap* map, const float* base, int l, int rows, long long cols) {
  EncodeTiledFn enc = get_encode();
  if (!enc) { set_error("cuTensorMapEncodeTiled is not available from the driver"); return TPQ_ERR_CUDA; }
  cuuint64_t dims[3] = {(cuuint64_t)cols, (cuuint64_t)rows, (cuuint64_t)l};
  cuuint64_t strides[2] = {(cuuint64_t)cols * 4, (cuuint64_t)cols * rows * 4};
  cuuint32_t box[3] = {32, (cuuint32_t)rows, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed (%d)", (int)r); return TPQ_ERR_CUDA; }
  return TPQ_OK;
}

// shapes the tensor-core kernel takes; everything else goes to the exact SIMT kernel
bool assign_tc_supported(int l, int d, long long n, int k, const void* data, const void* cent) {
  return l >= 1 && d >= 8 && d <= 64 && d % 8 == 0 && k >= 8 && k <= 256 && k % 4 == 0 && n % 4 == 0 && n >= 128 &&
         n < (1ll << 31) && (reinterpret_cast<uintptr_t>(data) & 15) == 0 && (reinterpret_cast<uintptr_t>(cent) & 15) == 0;
}

int launch_assign_tc(const float* data, const float* cent, int l, int d, long long n, int k, int exact_values,
                     float* maxsims, int64_t* labels, cudaStream_t st) {
  CUtensorMap mx;
  if (int rc = make_map(&mx, data, l, d, n)) return rc;
  TcParams P;
  P.l = l; P.d = d; P.n = (int)n; P.k = k; P.nch = (k + 63) / 64;
  P.tiles_per_l = (int)((n + TC_M - 1) / TC_M);
  P.maxsims = maxsims; P.labels = labels; P.cent = cent; P.exact_values = exact_values;
  const size_t reg = (size_t)P.nch * 64 * 128;
  const size_t smem = ((size_t)(d + 31) / 32 + 1) * reg + (size_t)TC_STAGES * 2 * d * 128 + 2 * TC_STAGES * 8;
  const int sms = device_sm_count();
  long long total = (long long)l * P.tiles_per_l;
  int grid = (int)(total < sms ? total : sms);
  static void (*const kernels[8][4])(const CUtensorMap, TcParams) = {
#define TPQ_TC_ROW(KB) {assign_tc_kernel<KB, 1>, assign_tc_kernel<KB, 2>, assign_tc_kernel<KB, 3>, assign_tc_kernel<KB, 4>}
      TPQ_TC_ROW(1), TPQ_TC_ROW(2), TPQ_TC_ROW(3), TPQ_TC_ROW(4), TPQ_TC_ROW(5), TPQ_TC_ROW(6), TPQ_TC_ROW(7), TPQ_TC_ROW(8)};
#undef TPQ_TC_ROW
  const auto kern = kernels[d / 8 - 1][P.nch - 1];
  TPQ_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kern<<<grid, TC_THREADS, smem, st>>>(mx, P);
  TPQ_LAUNCH_CHECK("assign_tc_kernel");
  return TPQ_OK;
}

}  // namespace tpq
