// The three small neighbours of the search path that the north-star names:
//
//   tpq_max_sim            MaxSimCuda / max_sim_tn     torchpq/kernels/MaxSimCuda.py:184-238,
//                          (MultiKMeans assignment)    kernels/cuda/max_sim.cu:182-309 (thread_nseuclidean :78-98,
//                                                      reduce_dim_2 :152-180); caller clustering/MultiKMeans.py:314-333
//   tpq_compute_centroids  ComputeCentroidsCuda        torchpq/kernels/ComputeCentroidsCuda.py:43-81,
//                          (k-means update)            kernels/cuda/compute_centroids.cu:9-86
//   tpq_pq_decode          PQDecodeCuda                torchpq/kernels/PQDecodeCuda.py:38-65, kernels/cuda/pq_decode.cu:7-53
//
// Round-1 versions: exact fp32 arithmetic in the reference's own order (parity first).  max_sim is a
// single pass with the arg-max kept in registers across centroid tiles -- no float atomicMax + racy label
// write as in the reference (max_sim.cu:173-178), so labels are deterministic (lowest index wins ties).
#include "common.cuh"

namespace tpq {

// ----------------------------------------------------------------------------- assignment: argmax_j sim(x_i, c_j)
// data [l, d, n], cent [l, d, k]; sim = sum_e -(x-c)^2 (euclidean, fmaf(-dif, dif, acc), e ascending), sum_e x*c
// (cosine, fmaf(x, c, acc)) or sum_e -|x-c| (manhattan, acc -= fabsf(x - c), max_sim.cu:100-120).
constexpr int MS_B = 128, MS_K = 8;
template <int METRIC>
__global__ void __launch_bounds__(256)
max_sim_kernel(const float* __restrict__ data, const float* __restrict__ cent, int d, int n, int k,
               float* __restrict__ maxsims, int64_t* __restrict__ labels) {
  __shared__ __align__(16) float As[MS_K][MS_B];
  __shared__ __align__(16) float Bs[MS_K][MS_B];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int l = blockIdx.y;
  const int i0 = blockIdx.x * MS_B;
  const float* X = data + (size_t)l * d * n;
  const float* Cn = cent + (size_t)l * d * k;
  float best[8]; int besti[8];
  #pragma unroll
  for (int i = 0; i < 8; ++i) { best[i] = -INFINITY; besti[i] = 0; }

  for (int j0 = 0; j0 < k; j0 += MS_B) {
    float acc[8][8];
    #pragma unroll
    for (int i = 0; i < 8; ++i)
      #pragma unroll
      for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
    for (int e0 = 0; e0 < d; e0 += MS_K) {
      #pragma unroll
      for (int r = 0; r < 4; ++r) {                         // 8 x 128 per operand / 256 threads = 4 each
        const int el = r * 256 + tid, ee = el >> 7, col = el & 127, ge = e0 + ee;
        As[ee][col] = (ge < d && i0 + col < n) ? X[(size_t)ge * n + i0 + col] : 0.f;
        Bs[ee][col] = (ge < d && j0 + col < k) ? Cn[(size_t)ge * k + j0 + col] : 0.f;
      }
      __syncthreads();
      const int kk_end = min(MS_K, d - e0);
      for (int kk = 0; kk < kk_end; ++kk) {
        const float4 a0 = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
        const float4 a1 = *reinterpret_cast<const float4*>(&As[kk][64 + ty * 4]);
        const float4 b0 = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
        const float4 b1 = *reinterpret_cast<const float4*>(&Bs[kk][64 + tx * 4]);
        const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
        const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
        #pragma unroll
        for (int i = 0; i < 8; ++i)
          #pragma unroll
          for (int j = 0; j < 8; ++j) {
            if (METRIC == TPQ_METRIC_EUCLIDEAN) { const float dif = a[i] - b[j]; acc[i][j] = fmaf(-dif, dif, acc[i][j]); }
            else if (METRIC == TPQ_METRIC_MANHATTAN) acc[i][j] -= fabsf(a[i] - b[j]);
            else acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
          }
      }
      __syncthreads();
    }
    // per point: best over this thread's 8 centroids, then over the 16 threads (tx) of the row group
    #pragma unroll
    for (int i = 0; i < 8; ++i) {
      float v = -INFINITY; int vi = 0x7fffffff;
      #pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int cj = j0 + (j < 4 ? tx * 4 + j : 64 + tx * 4 + (j - 4));
        if (cj < k && (acc[i][j] > v || (acc[i][j] == v && cj < vi))) { v = acc[i][j]; vi = cj; }
      }
      #pragma unroll
      for (int o = 1; o < 16; o <<= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, v, o);
        const int oi = __shfl_xor_sync(0xffffffffu, vi, o);
        if (ov > v || (ov == v && oi < vi)) { v = ov; vi = oi; }
      }
      if (v > best[i]) { best[i] = v; besti[i] = vi; }      // earlier tile (lower index) keeps ties
    }
  }
  if (tx == 0) {
    #pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int p = i0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
      if (p < n) { maxsims[(size_t)l * n + p] = best[i]; labels[(size_t)l * n + p] = besti[i]; }
    }
  }
}

// ----------------------------------------------------------------------------- centroid update, k > 1024
// One CTA = (block of CC_K clusters, block of CC_E features, l).  It walks ALL points in order, compacts the members of
// its clusters (order preserved) and warp w adds the members of clusters j = w (mod 8) one after the other into
// shared-memory sums: every sum is taken in point order, so the centroids do not depend on scheduling (shared and
// global float atomics made them, and everything trained from them, vary from run to run).
constexpr int CC_K = 256, CC_E = 32, CC_T = 1024;
__global__ void __launch_bounds__(256)
centroid_owner_kernel(const float* __restrict__ data, const int64_t* __restrict__ labels, int d, int n, int k,
                      float* __restrict__ cent) {
  __shared__ float sums[CC_K][CC_E + 1];
  __shared__ int cnt[CC_K];
  __shared__ int mem_p[CC_T];
  __shared__ uint8_t mem_j[CC_T];
  __shared__ int warp_n[8];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int j0 = blockIdx.x * CC_K, e0 = blockIdx.y * CC_E, l = blockIdx.z;
  const int kc = min(CC_K, k - j0);
  for (int i = tid; i < CC_K * (CC_E + 1); i += 256) (&sums[0][0])[i] = 0.f;
  for (int i = tid; i < CC_K; i += 256) cnt[i] = 0;
  const int64_t* lab = labels + (size_t)l * n;
  const bool has_e = e0 + lane < d;
  const float* x = data + ((size_t)l * d + e0 + (has_e ? lane : 0)) * n;
  for (int n0 = 0; n0 < n; n0 += CC_T) {
    int n_mem = 0;
    __syncthreads();                                               // previous tile's member list is consumed
    #pragma unroll 1
    for (int r = 0; r < CC_T / 256; ++r) {                         // order-preserving compaction, 256 points per round
      const int p = n0 + r * 256 + tid;
      int j = -1;
      if (p < n) { const long long v = lab[p]; if (v >= j0 && v < (long long)j0 + kc) j = (int)(v - j0); }
      const unsigned m = __ballot_sync(0xffffffffu, j >= 0);
      if (lane == 0) warp_n[warp] = __popc(m);
      __syncthreads();
      int base = n_mem;
      for (int w = 0; w < warp; ++w) base += warp_n[w];
      int total = n_mem;
      for (int w = 0; w < 8; ++w) total += warp_n[w];
      if (j >= 0) { const int at = base + __popc(m & ((1u << lane) - 1)); mem_p[at] = p; mem_j[at] = (uint8_t)j; }
      n_mem = total;
      __syncthreads();
    }
    // warp w owns clusters j = w (mod 8): its sums are added in point order
    for (int i0 = 0; i0 < n_mem; i0 += 8) {
      float v[8]; int jj[8];
      #pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int i = i0 + u;
        jj[u] = -1; v[u] = 0.f;
        if (i < n_mem && (mem_j[i] & 7) == warp) { jj[u] = mem_j[i]; v[u] = has_e ? __ldg(x + mem_p[i]) : 0.f; }
      }
      #pragma unroll
      for (int u = 0; u < 8; ++u) {
        if (jj[u] >= 0) {
          sums[jj[u]][lane] += v[u];
          if (lane == 0) cnt[jj[u]] += 1;
        }
      }
    }
  }
  __syncthreads();
  for (int i = tid; i < kc * CC_E; i += 256) {
    const int j = i % kc, e = i / kc;                              // consecutive threads: consecutive clusters (coalesced)
    if (e0 + e < d) {
      const float c = (float)cnt[j];
      cent[((size_t)l * d + e0 + e) * k + j0 + j] = cnt[j] == 0 ? 0.f : __fdiv_rn(sums[j][e], c);   // compute_centroids.cu:80
    }
  }
}

// Streaming update for k <= 1024 (the path C5 takes): one CTA owns (l, a block of CG_E * CG_G = 16 features) for ALL
// points, walks the points in tiles of CG_T, counting-sorts every tile by label once (shared-memory permutation), and
// for each group of 4 features stages the 4 rows as one float4 per point; thread j then walks the segment of cluster
// j (and j + 256, ...) with one LDS.128 gather per member and keeps the running sums of its clusters IN REGISTERS
// across the whole point stream.  No shared-memory atomics on the data, no global atomics at all, no memset and no
// finalize pass: the CTA knows its clusters' counts and writes sum / count itself.  (Round 1's centroid_sorted_kernel
// issued one global atomicAdd per (tile, feature, cluster) -- 128 M at C5 -- and two barriers per feature row.)
constexpr int CG_T = 4096, CG_E = 4, CG_G = 4;
template <int KJ>
__global__ void __launch_bounds__(256, 2)
centroid_stream_kernel(const float* __restrict__ data, const int64_t* __restrict__ labels,
                       int d, int n, int k, float* __restrict__ cent) {
  extern __shared__ __align__(16) uint8_t sm[];
  float4* xs = reinterpret_cast<float4*>(sm);                       // [CG_T] 4 features of one point
  uint16_t* perm = reinterpret_cast<uint16_t*>(xs + CG_T);          // [CG_T] point (within tile) at sorted position
  uint16_t* lab16 = perm + CG_T;                                    // [CG_T]
  int* seg = reinterpret_cast<int*>(lab16 + CG_T);                  // [k + 1] segment starts
  int* cur = seg + (k + 1);                                         // [k] histogram
  int* cw = cur + k;                                                // [8][k] per-warp scatter cursors
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int l = blockIdx.y, e_base = blockIdx.x * (CG_E * CG_G);
  float acc[KJ][CG_G][CG_E];
  int cnt[KJ];
  #pragma unroll
  for (int a = 0; a < KJ; ++a) {
    cnt[a] = 0;
    #pragma unroll
    for (int g = 0; g < CG_G; ++g)
      #pragma unroll
      for (int e = 0; e < CG_E; ++e) acc[a][g][e] = 0.f;
  }
  const int64_t* lab_l = labels + (size_t)l * n;
  constexpr int LPT = CG_T / 256;                                    // labels per thread per tile
  int lreg[LPT];                                                     // this tile's labels, loaded one tile ahead
  auto load_labels = [&](int n0) {
    #pragma unroll
    for (int u = 0; u < LPT; ++u) {
      const int p = n0 + u * 256 + tid;
      int j = 0xFFFF;
      if (p < n) { const long long v = __ldcs(reinterpret_cast<const long long*>(lab_l + p)); j = (v >= 0 && v < k) ? (int)v : 0xFFFF; }
      lreg[u] = j;                                                   // out-of-range labels are ignored (as the reference does)
    }
  };
  load_labels(0);
  for (int n0 = 0; n0 < n; n0 += CG_T) {
    const int np = min(CG_T, n - n0);
    for (int j = tid; j < k; j += 256) cur[j] = 0;
    __syncthreads();
    #pragma unroll
    for (int u = 0; u < LPT; ++u) {
      const int p = u * 256 + tid;
      if (p < np) { lab16[p] = (uint16_t)lreg[u]; if (lreg[u] != 0xFFFF) atomicAdd(&cur[lreg[u]], 1); }
    }
    if (n0 + CG_T < n) load_labels(n0 + CG_T);                       // in flight while this tile is summed
    __syncthreads();
    if (warp == 0) {                                                 // exclusive scan of the histogram
      int carry = 0;
      for (int j0 = 0; j0 < k; j0 += 32) {
        const int j = j0 + lane;
        const int c = j < k ? cur[j] : 0;
        const int incl = warp_inclusive_scan(c, lane);
        if (j < k) seg[j] = carry + incl - c;
        carry += __shfl_sync(0xffffffffu, incl, 31);
      }
      if (lane == 0) seg[k] = carry;
    }
    __syncthreads();
    // Stable scatter: warp w places the points [512 w, 512 w + 512) of the tile in order, after the members that warps
    // 0..w-1 place in the same segment, so every segment lists its points in point order and the sums below are taken
    // in a fixed order (an atomicAdd cursor made the order, and with it the rounding, vary from run to run).
    constexpr int PW = CG_T / 8;                                     // points per warp
    for (int i = tid; i < 8 * k; i += 256) cw[i] = 0;
    __syncthreads();
    #pragma unroll 1
    for (int r = 0; r < PW; r += 32) {                               // per-warp histogram (one leader per label group)
      const int p = warp * PW + r + lane;
      const int j = p < np ? (int)lab16[p] : 0xFFFF;
      const unsigned m = __match_any_sync(0xffffffffu, j);
      if (j != 0xFFFF && lane == __ffs(m) - 1) cw[warp * k + j] += __popc(m);
    }
    __syncthreads();
    #pragma unroll
    for (int a = 0; a < KJ; ++a) {
      const int j = tid + 256 * a;
      if (j < k) {
        cnt[a] += cur[j];
        int run = seg[j];
        for (int w = 0; w < 8; ++w) { const int t = cw[w * k + j]; cw[w * k + j] = run; run += t; }
      }
    }
    __syncthreads();
    #pragma unroll 1
    for (int r = 0; r < PW; r += 32) {
      const int p = warp * PW + r + lane;
      const int j = p < np ? (int)lab16[p] : 0xFFFF;
      const unsigned m = __match_any_sync(0xffffffffu, j);
      int at = 0;
      if (j != 0xFFFF) { at = cw[warp * k + j]; perm[at + __popc(m & ((1u << lane) - 1))] = (uint16_t)p; }
      __syncwarp();
      if (j != 0xFFFF && lane == __ffs(m) - 1) cw[warp * k + j] = at + __popc(m);
      __syncwarp();
    }
    // (the first staging barrier below also publishes perm)
    #pragma unroll
    for (int g = 0; g < CG_G; ++g) {
      const int e0 = e_base + g * CG_E;
      if (e0 >= d) break;                                            // CTA-uniform
      const float* x0 = data + ((size_t)l * d + e0) * n + n0;
      // 4 coalesced row reads -> one float4 per point.  All 32 loads of a batch are issued before the first shared-memory
      // store, so that many loads are in flight (with the 4 loads of one loop body alone in flight the kernel waited on
      // them).
      constexpr int SU = 8;
      const bool h1 = e0 + 1 < d, h2 = e0 + 2 < d, h3 = e0 + 3 < d;
      #pragma unroll 1
      for (int p0 = 0; p0 < np; p0 += 256 * SU) {
        float r[SU][4];
        #pragma unroll
        for (int u = 0; u < SU; ++u) {
          const int p = p0 + u * 256 + tid;
          const bool in = p < np;
          r[u][0] = in ? __ldcs(x0 + p) : 0.f;
          r[u][1] = (in && h1) ? __ldcs(x0 + (size_t)n + p) : 0.f;
          r[u][2] = (in && h2) ? __ldcs(x0 + 2 * (size_t)n + p) : 0.f;
          r[u][3] = (in && h3) ? __ldcs(x0 + 3 * (size_t)n + p) : 0.f;
        }
        #pragma unroll
        for (int u = 0; u < SU; ++u) {
          const int p = p0 + u * 256 + tid;
          if (p < np) xs[p] = make_float4(r[u][0], r[u][1], r[u][2], r[u][3]);
        }
      }
      __syncthreads();
      #pragma unroll
      for (int a = 0; a < KJ; ++a) {
        const int j = tid + 256 * a;
        if (j < k) {
          const int s1 = seg[j + 1];
          float4 t = make_float4(acc[a][g][0], acc[a][g][1], acc[a][g][2], acc[a][g][3]);
          for (int i = seg[j]; i < s1; ++i) {
            const float4 v = xs[perm[i]];
            t.x += v.x; t.y += v.y; t.z += v.z; t.w += v.w;
          }
          acc[a][g][0] = t.x; acc[a][g][1] = t.y; acc[a][g][2] = t.z; acc[a][g][3] = t.w;
        }
      }
      __syncthreads();
    }
  }
  #pragma unroll
  for (int a = 0; a < KJ; ++a) {
    const int j = tid + 256 * a;
    if (j >= k) continue;
    const float c = (float)cnt[a];
    #pragma unroll
    for (int g = 0; g < CG_G; ++g)
      #pragma unroll
      for (int e = 0; e < CG_E; ++e) {
        const int ee = e_base + g * CG_E + e;
        if (ee < d) cent[((size_t)l * d + ee) * k + j] = cnt[a] == 0 ? 0.f : __fdiv_rn(acc[a][g][e], c);   // compute_centroids.cu:80
      }
  }
}

// ----------------------------------------------------------------------------- PQ decode
// out[m*dsub + e, i] = codebook[m, e, code[m, i]]   (pq_decode.cu:7-53).  Write-bound: 4*d bytes per vector.
__global__ void __launch_bounds__(256)
pq_decode_kernel(const float* __restrict__ codebook, const uint8_t* __restrict__ code, int dsub, int64_t n,
                 bool vec, float* __restrict__ out) {
  extern __shared__ __align__(16) float tab[];             // [dsub][256]
  const int m = blockIdx.y;
  for (int i = threadIdx.x; i < dsub * 256; i += blockDim.x) tab[i] = codebook[(size_t)m * dsub * 256 + i];
  __syncthreads();
  const uint8_t* cm = code + (size_t)m * n;
  float* om = out + (size_t)m * dsub * n;
  for (int64_t i4 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4; i4 < n; i4 += (int64_t)gridDim.x * blockDim.x * 4) {
    if (vec) {
      const uint32_t w = *reinterpret_cast<const uint32_t*>(cm + i4);
      const int c0 = w & 0xff, c1 = (w >> 8) & 0xff, c2 = (w >> 16) & 0xff, c3 = w >> 24;
      for (int e = 0; e < dsub; ++e) {
        const float* t = tab + e * 256;
        __stcs(reinterpret_cast<float4*>(om + (size_t)e * n + i4), make_float4(t[c0], t[c1], t[c2], t[c3]));
      }
    } else {
      for (int u = 0; u < 4 && i4 + u < n; ++u) {
        const int c = cm[i4 + u];
        for (int e = 0; e < dsub; ++e) om[(size_t)e * n + i4 + u] = tab[e * 256 + c];
      }
    }
  }
}

}  // namespace tpq

namespace tpq {
bool assign_tc_supported(int l, int d, long long n, int k, const void* data, const void* cent);
int launch_assign_tc(const float* data, const float* cent, int l, int d, long long n, int k, int exact_values,
                     float* maxsims, int64_t* labels, cudaStream_t st);
bool assign_wide_supported(int l, int d, long long n, int k, const void* data, const void* cent);
size_t assign_wide_workspace_bytes(int l, int d, int k);
int launch_assign_wide(const float* data, const float* cent, int l, int d, long long n, int k, int metric,
                       int exact_values, float* maxsims, int64_t* labels, void* ws, cudaStream_t st);

// the exact SIMT kernel for one metric
static int launch_max_sim_exact(const float* data, const float* centroids, int l, int d, int64_t n, int k, int metric,
                                float* maxsims, int64_t* labels, cudaStream_t st) {
  dim3 grid((unsigned)((n + MS_B - 1) / MS_B), l);
  if (metric == TPQ_METRIC_EUCLIDEAN)
    max_sim_kernel<TPQ_METRIC_EUCLIDEAN><<<grid, 256, 0, st>>>(data, centroids, d, (int)n, k, maxsims, labels);
  else if (metric == TPQ_METRIC_MANHATTAN)
    max_sim_kernel<TPQ_METRIC_MANHATTAN><<<grid, 256, 0, st>>>(data, centroids, d, (int)n, k, maxsims, labels);
  else
    max_sim_kernel<TPQ_METRIC_COSINE><<<grid, 256, 0, st>>>(data, centroids, d, (int)n, k, maxsims, labels);
  TPQ_LAUNCH_CHECK("max_sim_kernel");
  return TPQ_OK;
}
}

using namespace tpq;

extern "C" int tpq_max_sim(const float* data, const float* centroids, int l, int d, int64_t n, int k, int metric,
                           int exact, float* maxsims, int64_t* labels, void* stream) {
  TPQ_REQUIRE(data && centroids && maxsims && labels, "tpq_max_sim: null pointer");
  TPQ_REQUIRE(l > 0 && d > 0 && n >= 0 && k > 0, "tpq_max_sim: bad sizes l=%d d=%d n=%lld k=%d", l, d, (long long)n, k);
  TPQ_REQUIRE(n <= 0x7fffffffll - MS_B && l <= 65535, "tpq_max_sim: n or l too large");
  TPQ_REQUIRE(metric == TPQ_METRIC_EUCLIDEAN || metric == TPQ_METRIC_COSINE || metric == TPQ_METRIC_MANHATTAN,
              "tpq_max_sim: unsupported metric %d", metric);
  if (n == 0) return TPQ_OK;
  if (exact != 1 && metric == TPQ_METRIC_EUCLIDEAN && assign_tc_supported(l, d, n, k, data, centroids))
    return launch_assign_tc(data, centroids, l, d, n, k, exact == 2 ? 1 : 0, maxsims, labels, (cudaStream_t)stream);
  return launch_max_sim_exact(data, centroids, l, d, n, k, metric, maxsims, labels, (cudaStream_t)stream);
}

extern "C" size_t tpq_kmeans_assign_workspace_bytes(int l, int d, int k) {
  return l > 0 && l <= 65535 ? assign_wide_workspace_bytes(l, d, k) : 0;
}

extern "C" int tpq_kmeans_assign(const float* data, const float* centroids, int l, int d, int64_t n, int k, int metric,
                                 int exact_values, float* maxsims, int64_t* labels, void* ws, size_t ws_bytes,
                                 void* stream) {
  TPQ_REQUIRE(data && centroids && maxsims && labels, "tpq_kmeans_assign: null pointer");
  TPQ_REQUIRE(l > 0 && d > 0 && n >= 0 && k > 0, "tpq_kmeans_assign: bad sizes l=%d d=%d n=%lld k=%d", l, d, (long long)n, k);
  TPQ_REQUIRE(n <= 0x7fffffffll - MS_B && l <= 65535, "tpq_kmeans_assign: n or l too large");
  TPQ_REQUIRE(metric == TPQ_METRIC_EUCLIDEAN || metric == TPQ_METRIC_COSINE || metric == TPQ_METRIC_MANHATTAN,
              "tpq_kmeans_assign: unsupported metric %d", metric);
  if (n == 0) return TPQ_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int ev = exact_values ? 1 : 0;
  if (metric == TPQ_METRIC_EUCLIDEAN && assign_tc_supported(l, d, n, k, data, centroids))
    return launch_assign_tc(data, centroids, l, d, n, k, ev, maxsims, labels, st);
  if (metric != TPQ_METRIC_MANHATTAN && assign_wide_supported(l, d, n, k, data, centroids)) {
    const size_t need = assign_wide_workspace_bytes(l, d, k);
    if (!ws || ws_bytes < need || (reinterpret_cast<uintptr_t>(ws) & 15) != 0) {
      set_error("tpq_kmeans_assign: workspace of %zu bytes at %p, need %zu bytes, 16-byte aligned", ws_bytes, ws, need);
      return TPQ_ERR_WORKSPACE;
    }
    return launch_assign_wide(data, centroids, l, d, n, k, metric, ev, maxsims, labels, ws, st);
  }
  return launch_max_sim_exact(data, centroids, l, d, n, k, metric, maxsims, labels, st);
}

// Both kernels keep their sums on chip: no workspace (the ABI keeps the argument).
extern "C" size_t tpq_compute_centroids_workspace_bytes(int l, int k) { (void)l; (void)k; return 0; }

extern "C" int tpq_compute_centroids(const float* data, const int64_t* labels, int l, int d, int64_t n, int k,
                                     float* centroids, void* ws, size_t ws_bytes, void* stream) {
  // (an empty tensor may have no storage: with n = 0 only the centroids are touched)
  TPQ_REQUIRE(centroids && (n == 0 || (data && labels)), "tpq_compute_centroids: null pointer");
  TPQ_REQUIRE(l > 0 && d > 0 && n >= 0 && k > 0 && n <= 0x7fffffffll && l <= 65535, "tpq_compute_centroids: bad sizes");
  (void)ws; (void)ws_bytes;
  cudaStream_t st = (cudaStream_t)stream;
  if (n > 0 && k <= 1024) {
    // streaming kernel: sums in registers, one launch, deterministic ownership of every output element
    const size_t smem = (size_t)CG_T * 16 + (size_t)CG_T * 2 * 2 + (size_t)(10 * k + 1) * 4;
    dim3 grid((unsigned)((d + CG_E * CG_G - 1) / (CG_E * CG_G)), l);
#define TPQ_CSTREAM(KJ)                                                                                              \
    do {                                                                                                             \
      TPQ_CUDA(cudaFuncSetAttribute(centroid_stream_kernel<KJ>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
      centroid_stream_kernel<KJ><<<grid, 256, smem, st>>>(data, labels, d, (int)n, k, centroids);                    \
    } while (0)
    if (k <= 256) TPQ_CSTREAM(1); else if (k <= 512) TPQ_CSTREAM(2); else TPQ_CSTREAM(4);
#undef TPQ_CSTREAM
    TPQ_LAUNCH_CHECK("centroid_stream_kernel");
    return TPQ_OK;
  }
  if (n == 0) {
    TPQ_CUDA(cudaMemsetAsync(centroids, 0, (size_t)l * d * k * 4, st));   // every cluster empty -> 0
    return TPQ_OK;
  }
  dim3 grid((unsigned)((k + CC_K - 1) / CC_K), (unsigned)((d + CC_E - 1) / CC_E), (unsigned)l);
  centroid_owner_kernel<<<grid, 256, 0, st>>>(data, labels, d, (int)n, k, centroids);
  TPQ_LAUNCH_CHECK("centroid_owner_kernel");
  return TPQ_OK;
}

extern "C" int tpq_pq_decode(const float* codebook, const uint8_t* code, int M, int dsub, int64_t n, float* out, void* stream) {
  TPQ_REQUIRE(codebook && code && out, "tpq_pq_decode: null pointer");
  TPQ_REQUIRE(M > 0 && dsub > 0 && n >= 0 && M <= 65535, "tpq_pq_decode: bad sizes");
  TPQ_REQUIRE((size_t)dsub * 1024 <= 200 * 1024, "tpq_pq_decode: d_subvector=%d too large", dsub);
  if (n == 0) return TPQ_OK;
  size_t smem = (size_t)dsub * 1024;
  TPQ_CUDA(cudaFuncSetAttribute(pq_decode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int64_t bx = (n + 1023) / 1024;
  const int64_t cap = (int64_t)device_sm_count() * 8;
  if (bx > cap) bx = cap;
  const bool vec = (n & 3) == 0 && (reinterpret_cast<uintptr_t>(code) & 3) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0;
  pq_decode_kernel<<<dim3((unsigned)bx, M), 256, smem, (cudaStream_t)stream>>>(codebook, code, dsub, n, vec, out);
  TPQ_LAUNCH_CHECK("pq_decode_kernel");
  return TPQ_OK;
}
