// Exact brute-force k-NN over a flat fp32 store (FlatIndex.search, torchpq/index/FlatIndex.py:46-101).
//
// One fused kernel streams the exact fp32 distance GEMM tile by tile and keeps per-query top-k lists in shared memory,
// so the [nq, n] score matrix never reaches HBM (10 k queries x 1 M vectors would be 40 GB).  Each CTA owns QT queries
// and one slice of the base columns; it writes its queries' sorted top-k keys to ws[slice, q, :], and
// tpq_merge_topk merges the slices and decodes values, addresses and ids.
#include "fused_scan.cuh"

extern "C" int tpq_merge_topk(const uint64_t* keys_in, int nq, int n_parts, int k, const int64_t* address2id,
                              int64_t capacity, float* values, int64_t* ids, int64_t* address, void* stream);

namespace tpq {

constexpr float kFlatEps = 1e-8f;     // metric.cosine_similarity's `norm + 1e-8` (metric.py:14-25)

// The plan, read by the workspace size and the launch; k == 0 is the range search's, with no lists and no keys.
//   QT: the smallest of 16, 32, 64 that holds the batch (a 1-query batch does not pay for 64 rows of GEMM), halved
//       while the CTA's shared memory exceeds 227 KB.  k <= 256 keeps 64 (kp = 256: 24 + 32 + 128 + 4 = 188 KB),
//       k = 512 gives 32 (20 + 16 + 128 + 4 = 168 KB), k = 1024 gives 16 (18 + 8 + 128 + 4 = 158 KB).  64 is the
//       largest: a 128-query tile would halve the lists' room (k <= 128) for a GEMM that is already 64 x 128.
//   S:  slices of the columns, enough that the grid (query tiles x slices) covers the SMs twice, at most one per
//       128-column tile; each slice is a whole number of tiles.  The workspace holds S * nq * k keys: S * nq is at most
//       2 * SMs * QT + nq, whatever n is.
struct FlatPlan {
  int qt, kp, qtiles, S;
  int64_t slice_cols;
  size_t smem, keys, xn, xq, total;     // keys / xn / xq: offsets into the workspace
};

static FlatPlan plan_flat(int d, int nq, int64_t n, int k) {
  FlatPlan P{};
  P.kp = k ? list_capacity(k) : 0;
  P.qt = 16;
  while (P.qt < 64 && P.qt < nq) P.qt *= 2;
  while (P.qt > 16 && fused_smem_bytes(P.qt, P.kp) > kSmemLimit) P.qt /= 2;
  P.smem = fused_smem_bytes(P.qt, P.kp);
  P.qtiles = (nq + P.qt - 1) / P.qt;
  const int64_t tiles = (n + GB - 1) / GB;
  int64_t S = (2 * (int64_t)device_sm_count() + P.qtiles - 1) / P.qtiles;
  S = S < 1 ? 1 : (tiles > 0 && S > tiles ? tiles : S);
  const int64_t per = tiles > 0 ? (tiles + S - 1) / S : 1;          // tiles per slice
  P.S = tiles > 0 ? (int)((tiles + per - 1) / per) : 1;             // no empty slice
  P.slice_cols = per * GB;
  P.keys = 0;
  P.xn = align_up((size_t)P.S * nq * k * 8, 256);
  P.xq = P.xn + align_up((size_t)nq * 4, 256);
  P.total = P.xq + align_up((size_t)d * nq * 4, 256);
  return P;
}

// grid (query tiles, slices), 256 threads.  METRIC: euclidean ((acc * 2) - xn[q]) - norms[c] with norms = ||b||^2;
// cosine acc / norms[c] with norms = ||b|| + 1e-8 and x normalised; inner acc.  Two CTAs per SM: at most 128
// registers (without the bound ptxas gave QT = 64 143 and QT = 32 inner 64 with a spill).
template <int QT, int METRIC>
__global__ void __launch_bounds__(256, 2)
flat_search_kernel(const float* __restrict__ x, int d, int nq, const float* __restrict__ base, int64_t ld, int64_t n,
                   const float* __restrict__ norms, const float* __restrict__ xn, int k, int kp, int64_t slice_cols,
                   uint64_t* __restrict__ keys_out) {
  using G = GemmTile<QT>;
  extern __shared__ __align__(16) uint8_t smem[];
  auto& stages = *reinterpret_cast<typename G::Stages*>(smem);
  float (*S)[GB] = reinterpret_cast<float (*)[GB]>(smem + sizeof(typename G::Stages));
  uint64_t* lists = reinterpret_cast<uint64_t*>(smem + sizeof(typename G::Stages) + (size_t)QT * GB * 4);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, tx = tid & 15, ty = tid >> 4;
  uint64_t* wbuf = lists + (size_t)QT * kp + (size_t)warp * kTopkBuf;
  const int q0 = blockIdx.x * QT;
  const int64_t c_begin = (int64_t)blockIdx.y * slice_cols;
  const int64_t c_end = c_begin + slice_cols < n ? c_begin + slice_cols : n;
  for (int i = tid; i < QT * kp; i += 256) lists[i] = 0ull;
  // (the barrier after G::run's first stash orders these stores before the first selection, and each selection
  //  before the next tile's score stores)
  for (int64_t c0 = c_begin; c0 < c_end; c0 += GB) {
    float acc[G::MI][8];
    G::run(x, nq, q0, base + c0, ld, (int)(c_end - c0 < GB ? c_end - c0 : GB), d, stages, acc);
    float nc[8];
    #pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int64_t c = c0 + G::col(j, tx);
      nc[j] = (METRIC != TPQ_METRIC_INNER && c < c_end) ? norms[c] : 1.f;
    }
    #pragma unroll
    for (int i = 0; i < G::MI; ++i) {
      const int r = G::row(i, ty);
      const float a2 = (METRIC == TPQ_METRIC_EUCLIDEAN && q0 + r < nq) ? xn[q0 + r] : 0.f;
      float o[8];
      #pragma unroll
      for (int j = 0; j < 8; ++j) {
        if (METRIC == TPQ_METRIC_EUCLIDEAN) o[j] = __fsub_rn(__fsub_rn(__fmul_rn(acc[i][j], 2.f), a2), nc[j]);
        else if (METRIC == TPQ_METRIC_COSINE) o[j] = __fdiv_rn(acc[i][j], nc[j]);
        else o[j] = acc[i][j];
      }
      *reinterpret_cast<float4*>(&S[r][tx * 4]) = make_float4(o[0], o[1], o[2], o[3]);
      *reinterpret_cast<float4*>(&S[r][64 + tx * 4]) = make_float4(o[4], o[5], o[6], o[7]);
    }
    __syncthreads();
    // warp w owns rows w, w + 8, ...: filter each against its query's k-th key, stage the survivors, flush per row
    for (int r = warp; r < QT && q0 + r < nq; r += kFusedWarps) {
      WarpTopK tk{lists + (size_t)r * kp, wbuf, kp, k, 0};
      uint64_t thr = tk.kth();
      #pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int64_t c = c0 + u * 32 + lane;
        const bool ok = c < c_end;
        const uint64_t key = ok ? make_key(S[r][u * 32 + lane], (uint32_t)c) : 0ull;
        if (tk.push(ok && key > thr, key, lane)) thr = tk.kth();
      }
      tk.flush(lane);
    }
  }
  __syncthreads();                                     // the lists were last written by their own warps
  for (int r = warp; r < QT && q0 + r < nq; r += kFusedWarps) {
    uint64_t* dst = keys_out + ((size_t)blockIdx.y * nq + q0 + r) * k;
    for (int i = lane; i < k; i += 32) dst[i] = lists[(size_t)r * kp + i];
  }
}

// grid (query tiles, slices), 256 threads.  flat_search_kernel's GEMM and epilogue, then every score > thr (strict, in
// fp32; NaN never passes) of a live column goes to the match buffer as (query, key); at most `cap` of them are written
// to keys_out / q_out, and *total counts them all.
template <int QT, int METRIC>
__global__ void __launch_bounds__(256, 2)
flat_range_kernel(const float* __restrict__ x, int d, int nq, const float* __restrict__ base, int64_t ld, int64_t n,
                  const float* __restrict__ norms, const float* __restrict__ xn, float thr, int64_t slice_cols,
                  uint64_t* __restrict__ keys_out, int32_t* __restrict__ q_out, int64_t cap,
                  unsigned long long* __restrict__ total) {
  using G = GemmTile<QT>;
  extern __shared__ __align__(16) uint8_t smem[];
  auto& stages = *reinterpret_cast<typename G::Stages*>(smem);
  RangeBuf& mb = *reinterpret_cast<RangeBuf*>(smem + sizeof(typename G::Stages));
  const int tid = threadIdx.x, lane = tid & 31, tx = tid & 15, ty = tid >> 4;
  const int q0 = blockIdx.x * QT;
  const int64_t c_begin = (int64_t)blockIdx.y * slice_cols;
  const int64_t c_end = c_begin + slice_cols < n ? c_begin + slice_cols : n;
  auto query = [&](int r) { return q0 + r; };
  if (tid == 0) mb.cnt = 0;                            // ordered before the first append by G::run's first barrier
  for (int64_t c0 = c_begin; c0 < c_end; c0 += GB) {
    float acc[G::MI][8];
    G::run(x, nq, q0, base + c0, ld, (int)(c_end - c0 < GB ? c_end - c0 : GB), d, stages, acc);
    float nc[8];
    #pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int64_t c = c0 + G::col(j, tx);
      nc[j] = (METRIC != TPQ_METRIC_INNER && c < c_end) ? norms[c] : 1.f;
    }
    uint32_t pass = 0;
    #pragma unroll
    for (int i = 0; i < G::MI; ++i) {
      const int r = G::row(i, ty);
      const float a2 = (METRIC == TPQ_METRIC_EUCLIDEAN && q0 + r < nq) ? xn[q0 + r] : 0.f;
      #pragma unroll
      for (int j = 0; j < 8; ++j) {
        float o;
        if (METRIC == TPQ_METRIC_EUCLIDEAN) o = __fsub_rn(__fsub_rn(__fmul_rn(acc[i][j], 2.f), a2), nc[j]);
        else if (METRIC == TPQ_METRIC_COSINE) o = __fdiv_rn(acc[i][j], nc[j]);
        else o = acc[i][j];
        acc[i][j] = o;
        if (q0 + r < nq && c0 + G::col(j, tx) < c_end && o > thr) pass |= 1u << (i * 8 + j);
      }
    }
    range_append(mb, pass, acc, [&](int i) { return G::row(i, ty); },
                 [&](int j) { return (uint32_t)(c0 + G::col(j, tx)); }, lane);
    __syncthreads();                                   // the appends, and this tile's last reads of the stages
    if (mb.cnt > kRangeBuf - QT * GB) range_flush(mb, total, cap, keys_out, q_out, query);
  }
  __syncthreads();
  range_flush(mb, total, cap, keys_out, q_out, query);
}

static bool flat_metric(int metric) {
  return metric == TPQ_METRIC_EUCLIDEAN || metric == TPQ_METRIC_COSINE || metric == TPQ_METRIC_INNER;
}

// The checks of tpq_flat_search and tpq_flat_range_search on the sizes.
static int flat_check(const char* name, int d, int nq, int64_t n, int64_t ld) {
  TPQ_REQUIRE(d > 0 && nq >= 0 && n >= 0 && ld >= n, "%s: bad sizes d=%d nq=%d n=%lld ld=%lld", name, d, nq,
              (long long)n, (long long)ld);
  TPQ_REQUIRE(n < (int64_t(1) << 32), "%s: n=%lld exceeds the 32-bit address of a key", name, (long long)n);
  return TPQ_OK;
}

// The rest of both searches up to the launch, for nq > 0: the query, base and norm pointers, the plan P (k == 0: the
// range search's) and the workspace, then the queries the GEMM reads, xq: x_dn with |x|^2 at P.xn (euclidean), or the
// normalised queries at P.xq (cosine).  n == 0 reads no query.
static int flat_prepare(const char* name, const float* x_dn, int d, int nq, const float* base, int64_t n,
                        const float* norms, int metric, int k, void* ws, size_t ws_bytes, cudaStream_t st,
                        FlatPlan& P, const float*& xq) {
  TPQ_REQUIRE(x_dn, "%s: null query pointer", name);
  TPQ_REQUIRE(n == 0 || (base && (norms || metric == TPQ_METRIC_INNER)), "%s: null base or norms", name);
  P = plan_flat(d, nq, n, k);
  if (!ws || ws_bytes < P.total) {
    set_error("%s: workspace too small (%zu < %zu)", name, ws_bytes, P.total);
    return TPQ_ERR_WORKSPACE;
  }
  xq = x_dn;
  uint8_t* w = reinterpret_cast<uint8_t*>(ws);
  if (n == 0) return TPQ_OK;
  if (metric == TPQ_METRIC_EUCLIDEAN) return col_sqnorms(x_dn, d, nq, nq, reinterpret_cast<float*>(w + P.xn), st);
  if (metric == TPQ_METRIC_COSINE) {
    xq = reinterpret_cast<float*>(w + P.xq);
    return normalize_columns(x_dn, d, nq, kFlatEps, reinterpret_cast<float*>(w + P.xq), st);
  }
  return TPQ_OK;
}

}  // namespace tpq

using namespace tpq;

extern "C" int tpq_flat_norms(const float* base, int64_t ld, int d, int64_t n, int metric, float* norms, void* stream) {
  TPQ_REQUIRE(flat_metric(metric), "tpq_flat_norms: unsupported metric %d", metric);
  TPQ_REQUIRE(d > 0 && n >= 0 && ld >= n, "tpq_flat_norms: bad sizes d=%d n=%lld ld=%lld", d, (long long)n, (long long)ld);
  TPQ_REQUIRE(n < (int64_t(1) << 32), "tpq_flat_norms: n=%lld exceeds the 32-bit address of a key", (long long)n);
  if (metric == TPQ_METRIC_INNER || n == 0) return TPQ_OK;           // inner products need no table
  TPQ_REQUIRE(base && norms, "tpq_flat_norms: null pointer");
  if (metric == TPQ_METRIC_EUCLIDEAN) return col_sqnorms(base, d, n, ld, norms, (cudaStream_t)stream);
  return col_norms(base, d, n, ld, kFlatEps, norms, (cudaStream_t)stream);
}

extern "C" size_t tpq_flat_workspace_bytes(int d, int nq, int64_t n, int k) {
  if (d <= 0 || nq <= 0 || n < 0 || k <= 0 || k > 1024) return 0;
  return plan_flat(d, nq, n, k).total;
}

extern "C" int tpq_flat_search(const float* x_dn, int d, int nq, const float* base, int64_t ld, int64_t n,
                               const float* norms, int metric, int k, const int64_t* address2id,
                               float* values, int64_t* ids, int64_t* address, void* ws, size_t ws_bytes,
                               void* stream) {
  TPQ_REQUIRE(k > 0, "k must be in (0, 1024], got %d", k);
  if (k > 1024) { set_error("k=%d > 1024 is not supported", k); return TPQ_ERR_UNSUPPORTED; }
  if (!flat_metric(metric)) { set_error("tpq_flat_search: unsupported metric %d", metric); return TPQ_ERR_UNSUPPORTED; }
  if (int rc = flat_check("tpq_flat_search", d, nq, n, ld)) return rc;
  TPQ_REQUIRE(values && ids && (address2id || n == 0), "tpq_flat_search: null output or address2id");
  if (nq == 0) return TPQ_OK;
  cudaStream_t st = (cudaStream_t)stream;
  FlatPlan P;
  const float* xq;
  if (int rc = flat_prepare("tpq_flat_search", x_dn, d, nq, base, n, norms, metric, k, ws, ws_bytes, st, P, xq))
    return rc;
  uint64_t* keys = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(ws) + P.keys);
  const float* xn = reinterpret_cast<const float*>(reinterpret_cast<uint8_t*>(ws) + P.xn);
  if (int rc = fused_launch<true>("flat_search_kernel", P.qt, metric, dim3(P.qtiles, P.S), P.smem, st,
                                  [](auto q, auto m) { return flat_search_kernel<decltype(q)::value, decltype(m)::value>; },
                                  xq, d, nq, base, ld, n, norms, xn, k, P.kp, P.slice_cols, keys))
    return rc;
  // n == 0: every key is empty and the id table (capacity 0) is never read, so any non-null pointer will do
  return tpq_merge_topk(keys, nq, P.S, k, n ? address2id : reinterpret_cast<const int64_t*>(keys), n, values, ids,
                        address, stream);
}

extern "C" size_t tpq_flat_range_workspace_bytes(int d, int nq, int64_t n) {
  if (d <= 0 || nq <= 0 || n < 0) return 0;
  return plan_flat(d, nq, n, 0).total;
}

extern "C" int tpq_flat_range_search(const float* x_dn, int d, int nq, const float* base, int64_t ld, int64_t n,
                                     const float* norms, int metric, float threshold, uint64_t* match_keys,
                                     int32_t* match_query, int64_t cap, uint64_t* total, void* ws, size_t ws_bytes,
                                     void* stream) {
  if (!flat_metric(metric)) {
    set_error("tpq_flat_range_search: unsupported metric %d", metric);
    return TPQ_ERR_UNSUPPORTED;
  }
  TPQ_REQUIRE(threshold == threshold, "tpq_flat_range_search: the threshold is NaN");
  TPQ_REQUIRE(cap >= 0, "tpq_flat_range_search: bad sizes d=%d nq=%d n=%lld ld=%lld cap=%lld", d, nq, (long long)n,
              (long long)ld, (long long)cap);
  if (int rc = flat_check("tpq_flat_range_search", d, nq, n, ld)) return rc;
  TPQ_REQUIRE(total && (cap == 0 || (match_keys && match_query)), "tpq_flat_range_search: null total or match buffer");
  if (nq == 0) return TPQ_OK;
  cudaStream_t st = (cudaStream_t)stream;
  FlatPlan P;
  const float* xq;
  if (int rc = flat_prepare("tpq_flat_range_search", x_dn, d, nq, base, n, norms, metric, 0, ws, ws_bytes, st, P, xq))
    return rc;
  TPQ_CUDA(cudaMemsetAsync(total, 0, sizeof(uint64_t), st));
  if (n == 0) return TPQ_OK;
  const float* xn = reinterpret_cast<const float*>(reinterpret_cast<uint8_t*>(ws) + P.xn);
  return fused_launch<true>("flat_range_kernel", P.qt, metric, dim3(P.qtiles, P.S), P.smem, st,
                            [](auto q, auto m) { return flat_range_kernel<decltype(q)::value, decltype(m)::value>; },
                            xq, d, nq, base, ld, n, norms, xn, threshold, P.slice_cols, match_keys, match_query, cap,
                            reinterpret_cast<unsigned long long*>(total));
}
