// Query preparation and coarse probing.
//
// Replaces, for IVFPQIndex.search (torchpq/index/IVFPQIndex.py:474-512):
//   util.normalize                          torchpq/util.py:38-43
//   metric.negative_squared_l2_distance     torchpq/metric.py:74-94   (cuBLAS sgemm + 4 elementwise passes)
//   fn.Topk -> top32_select / topk_select   torchpq/fn/Topk.py:43-67, kernels/cuda/top32_select.cu:483-636
//   smart probing                           torchpq/index/IVFPQIndex.py:499-512 (~8 torch launches)
// with three launches: squared norms, a tiled fp32 GEMM with the "*2 - |x|^2 - |c|^2"
// epilogue fused, and a warp-per-query top-n_probe select with smart probing fused.
#include "gemm_tile.cuh"

namespace tpq {

// Column reductions over a [d, n] matrix with row stride ld.  A CTA owns 32 columns; its 32 x 32 threads split the
// rows 32 ways (coalesced 128-byte row segments), partial sums meet in shared memory.  Row-group partials are combined
// in ascending group order, so the result is deterministic.  (32 row groups rather than round 1's 8: a 1000-query
// batch is only 32 CTAs, so at d = 960 the per-thread row loop was the whole latency of the cosine step.)
constexpr int CR_G = 32;    // row groups per CTA
__device__ __forceinline__ float col_sumsq(const float* __restrict__ x, int d, int64_t n, int64_t ld, int64_t j, int g,
                                           float (*part)[33], bool fma) {
  float s = 0.f;
  if (j < n) {
    for (int i = g; i < d; i += CR_G) {
      const float v = x[(size_t)i * ld + j];
      s = fma ? fmaf(v, v, s) : __fadd_rn(s, __fmul_rn(v, v));
    }
  }
  part[g][threadIdx.x & 31] = s;
  __syncthreads();
  float t = 0.f;
  #pragma unroll
  for (int r = 0; r < CR_G; ++r) t = __fadd_rn(t, part[r][threadIdx.x & 31]);
  return t;
}

// out[j] = sum_i x[i, j]^2   (torch's (a ** 2).sum(dim=-2): separately rounded squares)
__global__ void __launch_bounds__(32 * CR_G)
col_sqnorm_kernel(const float* __restrict__ x, int d, int64_t n, int64_t ld, float* __restrict__ out) {
  __shared__ float part[CR_G][33];
  const int64_t j = (int64_t)blockIdx.x * 32 + (threadIdx.x & 31);
  const int g = threadIdx.x >> 5;
  const float t = col_sumsq(x, d, n, ld, j, g, part, false);
  if (g == 0 && j < n) out[j] = t;
}

// out[j] = ||x[:, j]||_2 + eps, the divisor of normalize_columns_kernel
__global__ void __launch_bounds__(32 * CR_G)
col_norm_kernel(const float* __restrict__ x, int d, int64_t n, int64_t ld, float eps, float* __restrict__ out) {
  __shared__ float part[CR_G][33];
  const int64_t j = (int64_t)blockIdx.x * 32 + (threadIdx.x & 31);
  const int g = threadIdx.x >> 5;
  const float t = col_sumsq(x, d, n, ld, j, g, part, true);
  if (g == 0 && j < n) out[j] = __fadd_rn(sqrtf(t), eps);
}

// out[:, j] = x[:, j] / (||x[:, j]||_2 + eps)   (util.py:38-43 with eps 1e-9; metric.py:14-25 with eps 1e-8)
__global__ void __launch_bounds__(32 * CR_G)
normalize_columns_kernel(const float* __restrict__ x, int d, int n, float eps, float* __restrict__ out) {
  __shared__ float part[CR_G][33];
  const int j = blockIdx.x * 32 + (threadIdx.x & 31), g = threadIdx.x >> 5;
  const float t = col_sumsq(x, d, n, n, j, g, part, true);
  if (j >= n) return;
  const float nrm = __fadd_rn(sqrtf(t), eps);
  for (int i = g; i < d; i += CR_G) out[(size_t)i * n + j] = __fdiv_rn(x[(size_t)i * n + j], nrm);
}

static unsigned col_blocks(int64_t n) { return (unsigned)((n + 31) / 32); }

int col_sqnorms(const float* x, int d, int64_t n, int64_t ld, float* out, cudaStream_t st) {
  if (n == 0) return TPQ_OK;
  col_sqnorm_kernel<<<col_blocks(n), 32 * CR_G, 0, st>>>(x, d, n, ld, out);
  TPQ_LAUNCH_CHECK("col_sqnorm_kernel");
  return TPQ_OK;
}

int col_norms(const float* x, int d, int64_t n, int64_t ld, float eps, float* out, cudaStream_t st) {
  if (n == 0) return TPQ_OK;
  col_norm_kernel<<<col_blocks(n), 32 * CR_G, 0, st>>>(x, d, n, ld, eps, out);
  TPQ_LAUNCH_CHECK("col_norm_kernel");
  return TPQ_OK;
}

int normalize_columns(const float* x, int d, int n, float eps, float* out, cudaStream_t st) {
  if (n == 0) return TPQ_OK;
  normalize_columns_kernel<<<col_blocks(n), 32 * CR_G, 0, st>>>(x, d, n, eps, out);
  TPQ_LAUNCH_CHECK("normalize_columns_kernel");
  return TPQ_OK;
}

// sims[q, c] = ((2 * sum_i x[i,q] * cb[i,c]) - xn[q]) - cn[c]        (metric.py:75-94)
// The QT = 128 instance of the GEMM tile: a 128 x 128 tile per CTA.
__global__ void __launch_bounds__(256)
coarse_gemm_kernel(const float* __restrict__ x, const float* __restrict__ cb,
                   const float* __restrict__ xn, const float* __restrict__ cn,
                   int d, int nq, int C, float* __restrict__ sims) {
  using G = GemmTile<GB>;
  __shared__ __align__(16) G::Stages stages;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int q0 = blockIdx.y * GB, c0 = blockIdx.x * GB;
  float acc[8][8];
  G::run(x, nq, q0, cb + c0, C, C - c0, d, stages, acc);
  #pragma unroll
  for (int i = 0; i < 8; ++i) {
    int q = q0 + G::row(i, ty);
    if (q >= nq) continue;
    float a2 = xn[q];
    #pragma unroll
    for (int jh = 0; jh < 2; ++jh) {
      int c = c0 + jh * 64 + tx * 4;
      float o[4];
      #pragma unroll
      for (int j = 0; j < 4; ++j) {
        float y = __fmul_rn(acc[i][jh * 4 + j], 2.f);
        y = __fsub_rn(y, a2);
        o[j] = (c + j < C) ? __fsub_rn(y, cn[c + j]) : 0.f;
      }
      float* dst = sims + (size_t)q * C + c;
      if (c + 3 < C && (C & 3) == 0) *reinterpret_cast<float4*>(dst) = make_float4(o[0], o[1], o[2], o[3]);
      else for (int j = 0; j < 4 && c + j < C; ++j) dst[j] = o[j];
    }
  }
}

// One warp per query: top-n_probe of sims[q, :] (descending; ties -> lower cell index first),
// then the smart-probing entropy (IVFPQIndex.py:499-512).
__global__ void __launch_bounds__(128)
probe_select_kernel(const float* __restrict__ sims, int nq, int C, int n_probe, int kp,
                    int smart, float temperature,
                    float* __restrict__ probe_sims, int64_t* __restrict__ cells,
                    int64_t* __restrict__ n_probe_list) {
  extern __shared__ __align__(16) uint8_t smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int q = blockIdx.x * (blockDim.x >> 5) + warp;
  if (q >= nq) return;                                   // whole warp exits together
  uint64_t* base = reinterpret_cast<uint64_t*>(smem) + (size_t)warp * (kp + kTopkBuf);
  WarpTopK tk;
  tk.init(base, base + kp, kp, n_probe, lane);
  const float* row = sims + (size_t)q * C;
  uint64_t thr = 0;
  for (int c0 = 0; c0 < C; c0 += 128) {                  // four loads in flight per lane
    float v[4];
    #pragma unroll
    for (int u = 0; u < 4; ++u) { const int c = c0 + u * 32 + lane; v[u] = c < C ? __ldg(row + c) : 0.f; }
    #pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int c = c0 + u * 32 + lane;
      const bool ok = c < C;
      const uint64_t key = ok ? make_key(v[u], (uint32_t)c) : 0ull;
      if (tk.push(ok && key > thr, key, lane)) thr = tk.kth();
    }
  }
  tk.flush(lane);
  float* ps = probe_sims + (size_t)q * n_probe;
  int64_t* pc = cells + (size_t)q * n_probe;
  for (int j = lane; j < n_probe; j += 32) {
    uint64_t key = tk.list[j];
    ps[j] = key ? key_score(key) : -INFINITY;
    pc[j] = key ? (int64_t)key_addr(key) : 0;            // fewer cells than n_probe: reference pads index 0
  }
  if (!(smart && n_probe > 1)) {
    if (lane == 0) n_probe_list[q] = n_probe;            // IVFPQIndex.py:511-512
    return;
  }
  // p = softmax(-sqrt|s| / T);  H = -sum(p * log2 p / log2 n_probe);  n = ceil(H * n_probe)
  float mx = -INFINITY;
  for (int j = lane; j < n_probe; j += 32) {
    uint64_t key = tk.list[j];
    float s = key ? key_score(key) : -INFINITY;
    float z = __fdiv_rn(-sqrtf(fabsf(s)), temperature);
    mx = fmaxf(mx, z);
  }
  #pragma unroll
  for (int o = 16; o; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float sum = 0.f;
  for (int j = lane; j < n_probe; j += 32) {
    uint64_t key = tk.list[j];
    float s = key ? key_score(key) : -INFINITY;
    float z = __fdiv_rn(-sqrtf(fabsf(s)), temperature);
    sum += expf(z - mx);
  }
  #pragma unroll
  for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float lg = log2f((float)n_probe);
  float h = 0.f;
  for (int j = lane; j < n_probe; j += 32) {
    uint64_t key = tk.list[j];
    float s = key ? key_score(key) : -INFINITY;
    float z = __fdiv_rn(-sqrtf(fabsf(s)), temperature);
    float p = __fdiv_rn(expf(z - mx), sum);
    h += __fdiv_rn(__fmul_rn(p, log2f(p)), lg);          // 0 * -inf = NaN, as in the reference
  }
  #pragma unroll
  for (int o = 16; o; o >>= 1) h += __shfl_xor_sync(0xffffffffu, h, o);
  if (lane == 0) {
    float v = ceilf(__fmul_rn(-h, (float)n_probe));
    // CUDA's float->int64 conversion of NaN yields INT64_MIN, which is what the reference's
    // `.long()` produces on device; the scan then reads it as (int)0 -> one probe.
    n_probe_list[q] = isnan(v) ? (int64_t)0x8000000000000000ull : (int64_t)v;
  }
}

}  // namespace tpq

using namespace tpq;

extern "C" int tpq_normalize_columns(const float* x_dn, int d, int nq, float* out_dn, void* stream) {
  TPQ_REQUIRE(x_dn && out_dn && d > 0 && nq >= 0, "tpq_normalize_columns: bad argument");
  return normalize_columns(x_dn, d, nq, 1e-9f, out_dn, (cudaStream_t)stream);
}

extern "C" size_t tpq_coarse_workspace_bytes(int d, int nq, int n_cells) {
  (void)d;
  return align_up((size_t)nq * n_cells * 4, 256) + align_up((size_t)nq * 4, 256) + align_up((size_t)n_cells * 4, 256);
}

extern "C" int tpq_coarse_probe(const float* x_dn, const float* vq_codebook, int d, int nq, int n_cells,
                                int n_probe, int smart, float temperature,
                                float* probe_sims, int64_t* cells, int64_t* n_probe_list,
                                void* ws, size_t ws_bytes, void* stream) {
  TPQ_REQUIRE(x_dn && vq_codebook && probe_sims && cells && n_probe_list, "tpq_coarse_probe: null pointer");
  TPQ_REQUIRE(d > 0 && nq >= 0 && n_cells > 0, "tpq_coarse_probe: bad sizes d=%d nq=%d C=%d", d, nq, n_cells);
  TPQ_REQUIRE(n_probe >= 1 && n_probe <= n_cells, "n_probe=%d must be in [1, n_cells=%d]", n_probe, n_cells);
  if (n_probe > 1024) { set_error("n_probe=%d > 1024 is not supported", n_probe); return TPQ_ERR_UNSUPPORTED; }
  if (ws_bytes < tpq_coarse_workspace_bytes(d, nq, n_cells) || !ws) {
    set_error("tpq_coarse_probe: workspace too small (%zu < %zu)", ws_bytes, tpq_coarse_workspace_bytes(d, nq, n_cells));
    return TPQ_ERR_WORKSPACE;
  }
  if (nq == 0) return TPQ_OK;
  cudaStream_t st = (cudaStream_t)stream;
  uint8_t* w = reinterpret_cast<uint8_t*>(ws);
  float* sims = reinterpret_cast<float*>(w);  w += align_up((size_t)nq * n_cells * 4, 256);
  float* xn = reinterpret_cast<float*>(w);    w += align_up((size_t)nq * 4, 256);
  float* cn = reinterpret_cast<float*>(w);
  if (int rc = col_sqnorms(x_dn, d, nq, nq, xn, st)) return rc;
  if (int rc = col_sqnorms(vq_codebook, d, n_cells, n_cells, cn, st)) return rc;
  dim3 grid((n_cells + GB - 1) / GB, (nq + GB - 1) / GB);
  coarse_gemm_kernel<<<grid, 256, 0, st>>>(x_dn, vq_codebook, xn, cn, d, nq, n_cells, sims);
  TPQ_LAUNCH_CHECK("coarse_gemm_kernel");
  const int kp = list_capacity(n_probe);
  const int wpb = 4;
  size_t smem = (size_t)wpb * (kp + kTopkBuf) * sizeof(uint64_t);
  TPQ_CUDA(cudaFuncSetAttribute(probe_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  probe_select_kernel<<<(nq + wpb - 1) / wpb, wpb * 32, smem, st>>>(sims, nq, n_cells, n_probe, kp, smart, temperature,
                                                                   probe_sims, cells, n_probe_list);
  TPQ_LAUNCH_CHECK("probe_select_kernel");
  return TPQ_OK;
}
