// k-means assignment for large k and d on the Hopper tensor cores (wgmma TF32 + TMA + mbarrier), sm_90a.
//
//   label_i = argmax_j score(x_i, c_j)       data [l, d, n], centroids [l, d, k]
//   euclidean: score = <x, c> - |c|^2 / 2    (-|x - c|^2 = 2 score - |x|^2; |x|^2 does not change the arg-max)
//   cosine:    score = <x, c>                (columns normalised by the caller)
//
// assign_tc_kernel keeps every centroid of a k-means in shared memory, which caps it at d <= 64, k <= 256.  This
// kernel streams the centroids instead and covers 8 <= d <= 256 (d % 8 == 0) and any k >= 8:
//
//  * Pre-pass (aw_prepass_kernel): the centroids, MN-major in HBM, are written K-major into a caller-owned workspace,
//    one row of d + 8 floats per (l, j < k_pad): the d features, then a bias K-block (hi, lo, 0 x 6) with
//    hi + lo = -|c_j|^2 / 2 (euclidean; hi is exact in TF32, lo carries the rest) or 0 (cosine).  Rows j >= k are zero
//    with hi = -1e30, so padded columns never win.  Against a constant "ones" A fragment the bias K-block adds the
//    bias inside the MMA, as in assign_tc_kernel; the accumulator then holds the score itself.
//  * Point tiles: 128 points (two consumer warpgroups x 64 rows) stream in by TMA exactly as they lie in HBM (32-point
//    boxes of all d features, 128-byte swizzle) and stay resident while the CTA sweeps every centroid of its k-means.
//    wgmma takes TF32 from shared memory only K-major, so A is fed from registers: each thread loads its fragment
//    from the swizzled tile once per K step (64 x 256 fp32 would be 128 registers per thread at d = 256).
//  * Centroid stream: N tiles of 128 centroids, each cut into 32-feature slices (16 KB stages, TMA from the K-major
//    workspace, 128-byte swizzle) that pass through an mbarrier ring; both consumer warpgroups read every stage.
//    The A fragments of one slice are loaded while the previous slice's wgmmas run (wait_group 1).
//  * Arg-max: within an N tile the packed key of tc_common.cuh (8-bit column field) and fmaxf; across N tiles a
//    running (key, tile) per row, replaced only by a STRICTLY greater truncated score, so the earlier tile keeps ties;
//    finally the quad of threads sharing a row merges by (truncated score desc, global column asc).  The label is
//    therefore the lowest index among the columns whose truncated TF32 score is the maximum -- lowest index on ties for
//    every sign of the score, as the exact kernel.
//  * maxsims: exact_values = 1 recomputes the winner's similarity in fp32 in the exact kernel's order (e ascending,
//    fmaf(-dif, dif, acc) or fmaf(x, c, acc)) from the resident point tile and the workspace row; exact_values = 0
//    writes 2 score - |x|^2 (euclidean) or score (cosine) from the TF32 key.
//
// Persistent, warp-specialised: warpgroup 0 = TMA producer (one thread), warpgroups 1 and 2 = consumers.  Each CTA
// reads all centroids of its k-means once per 128-point tile: (n / 128) * k * (d + 8) * 4 bytes of L2 traffic per
// assignment; DESIGN.md section 4b discusses that bound.
#include "tc_common.cuh"

namespace tpq {

constexpr int AW_M = 128;                         // points per CTA tile
constexpr int AW_N = 128;                         // centroids per N tile
constexpr int AW_THREADS = 3 * 128;
constexpr uint32_t AW_STAGE = AW_N * 128;         // one 32-feature slice of an N tile: 128 rows x 128 bytes
constexpr int AW_MAX_STAGES = 8;
constexpr int AW_K_MAX = 1 << 20;

// D[64 x 128] (+)= A[64 x 8] (registers, TF32) * B[8 x 128] (shared memory, K-major)
__device__ __forceinline__ void wgmma_m64n128k8_tf32(float (&d)[64], const uint32_t (&a)[4], uint64_t desc_b, int accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
      "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, "
      "%46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "{%64, %65, %66, %67}, %68, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(accumulate)
      : "memory");
}

// ----------------------------------------------------------------------------- pre-pass: K-major centroids + bias block
__global__ void __launch_bounds__(256)
aw_prepass_kernel(const float* __restrict__ cent, int d, int k, int kpad, int metric, float* __restrict__ ws) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x, li = blockIdx.y;
  if (j >= kpad) return;
  const float* C = cent + (size_t)li * d * k;
  float* row = ws + ((size_t)li * kpad + j) * (d + 8);
  float v = -1e30f;                                                     // padded columns can never win
  if (j < k) {
    float s2 = 0.f;
    for (int e = 0; e < d; ++e) {
      const float cv = C[(size_t)e * k + j];
      s2 = fmaf(cv, cv, s2);
      row[e] = cv;
    }
    v = metric == TPQ_METRIC_EUCLIDEAN ? -0.5f * s2 : 0.f;
  } else {
    for (int e = 0; e < d; ++e) row[e] = 0.f;
  }
  const float hi = __uint_as_float(__float_as_uint(v) & 0xFFFFE000u);   // exactly representable in TF32
  row[d] = hi;
  row[d + 1] = v - hi;
  for (int e = 2; e < 8; ++e) row[d + e] = 0.f;
}

struct AwParams {
  int l, n, k, kpad;
  int n_ntiles;                  // kpad / AW_N
  int tiles_per_l;               // ceil(n / AW_M)
  int stages;                    // centroid ring depth
  int metric, exact_values;
  const float* ws;               // [l][kpad][d + 8] K-major centroids + bias block
  float* maxsims; int64_t* labels;
};

// KB = d / 8 K steps of features (+ 1 bias step), compile-time so that no wgmma sits under a run-time branch.
template <int KB>
__global__ void __launch_bounds__(AW_THREADS, 1)
assign_wide_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_c, AwParams P) {
  extern __shared__ __align__(1024) uint8_t smem[];
  constexpr int d = 8 * KB;
  constexpr int NSTEP = KB + 1;                                         // feature steps + the bias step
  constexpr int NCHUNK = (NSTEP + 3) / 4;                               // 32-feature slices per N tile
  constexpr uint32_t box_bytes = (uint32_t)d * 128;                     // one 32-point box of all d features
  constexpr uint32_t x_bytes = 4 * box_bytes;                           // the 128-point tile (multiple of 1024)
  uint8_t* sX = smem;
  uint8_t* sB = smem + x_bytes;
  const int S = P.stages;
  uint64_t* full = reinterpret_cast<uint64_t*>(sB + (size_t)S * AW_STAGE);
  uint64_t* empty = full + S;
  uint64_t* xfull = empty + S;
  uint64_t* xempty = xfull + 1;

  const int wg = threadIdx.x >> 7, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long total_tiles = (long long)P.l * P.tiles_per_l;
  const long long t_begin = total_tiles * blockIdx.x / gridDim.x;
  const long long t_end = total_tiles * (blockIdx.x + 1) / gridDim.x;

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" :: "l"(&map_x) : "memory");
    asm volatile("prefetch.tensormap [%0];" :: "l"(&map_c) : "memory");
    for (int s = 0; s < S; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 256); }
    mbar_init(xfull, 1); mbar_init(xempty, 256);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (wg == 0) {
    // ===================================================== TMA producer
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");               // hand registers to the consumers (4 x 40 + 8 x 232 <= 2048 per warp slot)
    if (threadIdx.x == 0) {
      int s = 0; uint32_t ph = 0;
      uint32_t tt = 0;
      for (long long t = t_begin; t < t_end; ++t, ++tt) {
        const int li = (int)(t / P.tiles_per_l), ti = (int)(t % P.tiles_per_l);
        mbar_wait(xempty, (tt & 1) ^ 1);                                // the consumers are done with the last tile
        mbar_expect_tx(xfull, x_bytes);
        for (int g = 0; g < 4; ++g) tma_load_3d(sX + g * box_bytes, &map_x, xfull, ti * AW_M + g * 32, 0, li);
        for (int nt = 0; nt < P.n_ntiles; ++nt)
          for (int kc = 0; kc < NCHUNK; ++kc) {
            mbar_wait(&empty[s], ph ^ 1);
            mbar_expect_tx(&full[s], AW_STAGE);
            tma_load_3d(sB + (size_t)s * AW_STAGE, &map_c, &full[s], 32 * kc, nt * AW_N, li);
            if (++s == S) { s = 0; ph ^= 1; }
          }
      }
    }
    return;
  }

  // ===================================================== consumers: warpgroup c owns rows [64 c, 64 c + 64) of the tile
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  const int c = wg - 1;
  const int w4 = warp & 3;
  const int g = lane >> 2, tq = lane & 3;
  const int r0 = 64 * c + 16 * w4 + g, r1 = r0 + 8;                     // the two tile rows (points) of this thread
  const uint8_t* xa = sX + (r0 >> 5) * box_bytes;                       // r0 and r1 lie in the same 32-point box
  const int c0 = r0 & 31, c1 = r1 & 31;
  const float one = tq < 2 ? 1.f : 0.f;                                 // A columns 0, 1 of the bias K-block = 1
  const uint32_t ones[4] = {__float_as_uint(one), __float_as_uint(one), 0u, 0u};
  const uint32_t base = 255u ^ (2u * (uint32_t)tq);                     // 255 ^ column, see assign_tc_kernel
  int s = 0; uint32_t ph = 0;
  uint32_t tt = 0;
  for (long long t = t_begin; t < t_end; ++t, ++tt) {
    const int li = (int)(t / P.tiles_per_l), ti = (int)(t % P.tiles_per_l);
    mbar_wait(xfull, tt & 1);
    float best0 = -3.0e38f, best1 = -3.0e38f;                           // best key per row (below every real key)
    float bs0 = -3.0e38f, bs1 = -3.0e38f;                               // its truncated score
    int bt0 = 0, bt1 = 0;                                               // its N tile
    for (int nt = 0; nt < P.n_ntiles; ++nt) {
      float acc[64];
      #pragma unroll
      for (int i = 0; i < 64; ++i) acc[i] = 0.f;
      int ps = 0;                                                       // stage of the previous slice
      #pragma unroll
      for (int kc = 0; kc < NCHUNK; ++kc) {
        uint32_t a[4][4];
        #pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int st = 4 * kc + q;                                    // compile-time after unrolling
          if (st < KB) {
            // wgmma m64nNk8 TF32 A layout: a0 = (r0, tq), a1 = (r1, tq), a2 = (r0, tq+4), a3 = (r1, tq+4)
            const int e = 8 * st + tq;
            a[q][0] = *reinterpret_cast<const uint32_t*>(xa + box_off(e, c0));
            a[q][1] = *reinterpret_cast<const uint32_t*>(xa + box_off(e, c1));
            a[q][2] = *reinterpret_cast<const uint32_t*>(xa + box_off(e + 4, c0));
            a[q][3] = *reinterpret_cast<const uint32_t*>(xa + box_off(e + 4, c1));
          } else {
            #pragma unroll
            for (int u = 0; u < 4; ++u) a[q][u] = ones[u];
          }
        }
        mbar_wait(&full[s], ph);
        wgmma_fence();
        const uint32_t bq = smem_u32(sB + (size_t)s * AW_STAGE);
        #pragma unroll
        for (int q = 0; q < 4; ++q)
          if (4 * kc + q < NSTEP) wgmma_m64n128k8_tf32(acc, a[q], gmma_desc(bq + q * 32), kc + q > 0);
        wgmma_commit();
        if (kc > 0) {                                                   // the previous slice's MMAs are done: release it
          wgmma_wait1();
          mbar_arrive(&empty[ps]);
        }
        ps = s;
        if (++s == S) { s = 0; ph ^= 1; }
      }
      wgmma_wait0();
      mbar_arrive(&empty[ps]);
      // Arg-max of this N tile.  Accumulator layout: acc[4i + {0,1}] = row r0, columns 8 i + 2 tq + {0,1};
      // acc[4i + {2,3}] = row r1, same columns.
      float cb0 = -3.0e38f, cb1 = -3.0e38f;
      #pragma unroll
      for (int i = 0; i < 16; ++i) {
        const uint32_t i0 = base ^ (uint32_t)(8 * i), i1 = i0 ^ 1u;
        cb0 = fmaxf(cb0, fmaxf(argmax_key(acc[4 * i + 0], i0), argmax_key(acc[4 * i + 1], i1)));
        cb1 = fmaxf(cb1, fmaxf(argmax_key(acc[4 * i + 2], i0), argmax_key(acc[4 * i + 3], i1)));
      }
      const float ts0 = argmax_key_score(cb0), ts1 = argmax_key_score(cb1);
      if (ts0 > bs0) { bs0 = ts0; best0 = cb0; bt0 = nt; }             // strictly greater: the earlier tile keeps ties
      if (ts1 > bs1) { bs1 = ts1; best1 = cb1; bt1 = nt; }
    }
    // quad merge: the 4 threads of a quad share rows r0, r1; (truncated score desc, global column asc)
    int gi0 = bt0 * AW_N + argmax_key_column(best0), gi1 = bt1 * AW_N + argmax_key_column(best1);
    #pragma unroll
    for (int o = 1; o <= 2; o <<= 1) {
      const float os0 = __shfl_xor_sync(0xffffffffu, bs0, o), ok0 = __shfl_xor_sync(0xffffffffu, best0, o);
      const int og0 = __shfl_xor_sync(0xffffffffu, gi0, o);
      if (os0 > bs0 || (os0 == bs0 && og0 < gi0)) { bs0 = os0; best0 = ok0; gi0 = og0; }
      const float os1 = __shfl_xor_sync(0xffffffffu, bs1, o), ok1 = __shfl_xor_sync(0xffffffffu, best1, o);
      const int og1 = __shfl_xor_sync(0xffffffffu, gi1, o);
      if (os1 > bs1 || (os1 == bs1 && og1 < gi1)) { bs1 = os1; best1 = ok1; gi1 = og1; }
    }
    // finisher: threads tq = 0, 2 take row r0, tq = 1, 3 row r1; tq = 0, 1 store
    {
      const int row = (tq & 1) ? r1 : r0;
      const int cr = row & 31;
      const float key = (tq & 1) ? best1 : best0;
      const int besti = (tq & 1) ? gi1 : gi0;
      const uint8_t* xr = sX + (row >> 5) * box_bytes;
      const bool euc = P.metric == TPQ_METRIC_EUCLIDEAN;
      float out;
      if (P.exact_values) {
        // exact fp32 similarity of the chosen centroid, e ascending (the exact kernel's arithmetic)
        const float* cr_g = P.ws + ((size_t)li * P.kpad + besti) * (d + 8);
        float acc1 = 0.f;
        for (int e = 0; e < d; ++e) {
          const float xv = *reinterpret_cast<const float*>(xr + box_off(e, cr));
          const float cv = __ldg(cr_g + e);
          if (euc) { const float dif = xv - cv; acc1 = fmaf(-dif, dif, acc1); }
          else acc1 = fmaf(xv, cv, acc1);
        }
        out = acc1;
      } else if (euc) {
        float x2 = 0.f;
        for (int e = 0; e < d; ++e) {
          const float xv = *reinterpret_cast<const float*>(xr + box_off(e, cr));
          x2 = fmaf(xv, xv, x2);
        }
        out = fmaf(2.f, key, -x2);                                      // -|x - c|^2 = 2 (<x,c> - |c|^2/2) - |x|^2
      } else {
        out = key;
      }
      const long long p = (long long)ti * AW_M + row;
      if (tq < 2 && p < P.n) {
        P.maxsims[(size_t)li * P.n + p] = out;
        P.labels[(size_t)li * P.n + p] = besti;
      }
    }
    mbar_arrive(xempty);                                                // this thread is done reading the point tile
  }
}

// ----------------------------------------------------------------------------- host
static int aw_map(CUtensorMap* map, const float* base, cuuint64_t d0, cuuint64_t d1, cuuint64_t d2, cuuint32_t b0,
                  cuuint32_t b1) {
  EncodeTiledFn enc = get_encode();
  if (!enc) { set_error("cuTensorMapEncodeTiled is not available from the driver"); return TPQ_ERR_CUDA; }
  cuuint64_t dims[3] = {d0, d1, d2};
  cuuint64_t strides[2] = {d0 * 4, d0 * d1 * 4};
  cuuint32_t box[3] = {b0, b1, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed (%d)", (int)r); return TPQ_ERR_CUDA; }
  return TPQ_OK;
}

static inline int aw_kpad(int k) { return (k + AW_N - 1) / AW_N * AW_N; }

bool assign_wide_shape(int d, int k) { return d >= 8 && d <= 256 && d % 8 == 0 && k >= 8 && k <= AW_K_MAX; }

size_t assign_wide_workspace_bytes(int l, int d, int k) {
  return assign_wide_shape(d, k) ? (size_t)l * aw_kpad(k) * (d + 8) * 4 : 0;
}

bool assign_wide_supported(int l, int d, long long n, int k, const void* data, const void* cent) {
  return l >= 1 && l <= 65535 && assign_wide_shape(d, k) && n >= 4 && n % 4 == 0 && n < (1ll << 31) - AW_M &&
         (reinterpret_cast<uintptr_t>(data) & 15) == 0 && (reinterpret_cast<uintptr_t>(cent) & 15) == 0;
}

int launch_assign_wide(const float* data, const float* cent, int l, int d, long long n, int k, int metric,
                       int exact_values, float* maxsims, int64_t* labels, void* ws, cudaStream_t st) {
  const int kpad = aw_kpad(k);
  float* wsf = static_cast<float*>(ws);
  aw_prepass_kernel<<<dim3((unsigned)((kpad + 255) / 256), (unsigned)l), 256, 0, st>>>(cent, d, k, kpad, metric, wsf);
  TPQ_LAUNCH_CHECK("aw_prepass_kernel");
  CUtensorMap mx, mc;
  if (int rc = aw_map(&mx, data, (cuuint64_t)n, (cuuint64_t)d, (cuuint64_t)l, 32, (cuuint32_t)d)) return rc;
  if (int rc = aw_map(&mc, wsf, (cuuint64_t)(d + 8), (cuuint64_t)kpad, (cuuint64_t)l, 32, AW_N)) return rc;
  AwParams P;
  P.l = l; P.n = (int)n; P.k = k; P.kpad = kpad; P.n_ntiles = kpad / AW_N;
  P.tiles_per_l = (int)((n + AW_M - 1) / AW_M);
  P.metric = metric; P.exact_values = exact_values;
  P.ws = wsf; P.maxsims = maxsims; P.labels = labels;
  const size_t x_bytes = (size_t)AW_M * d * 4;
  const size_t bar_bytes = (2 * AW_MAX_STAGES + 2) * 8;
  int stages = (int)((kSmemLimit - x_bytes - bar_bytes) / AW_STAGE);
  P.stages = stages > AW_MAX_STAGES ? AW_MAX_STAGES : stages;           // >= 6 at d = 256
  const size_t smem = x_bytes + (size_t)P.stages * AW_STAGE + (2 * P.stages + 2) * 8;
  const int sms = device_sm_count();
  const long long total = (long long)l * P.tiles_per_l;
  const int grid = (int)(total < sms ? total : sms);
  static void (*const kernels[32])(const CUtensorMap, const CUtensorMap, AwParams) = {
#define TPQ_AW4(b) assign_wide_kernel<b + 1>, assign_wide_kernel<b + 2>, assign_wide_kernel<b + 3>, assign_wide_kernel<b + 4>
      TPQ_AW4(0), TPQ_AW4(4), TPQ_AW4(8), TPQ_AW4(12), TPQ_AW4(16), TPQ_AW4(20), TPQ_AW4(24), TPQ_AW4(28)};
#undef TPQ_AW4
  const auto kern = kernels[d / 8 - 1];
  TPQ_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kern<<<grid, AW_THREADS, smem, st>>>(mx, mc, P);
  TPQ_LAUNCH_CHECK("assign_wide_kernel");
  return TPQ_OK;
}

}  // namespace tpq
