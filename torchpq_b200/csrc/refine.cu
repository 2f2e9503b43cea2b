// Exact re-rank of any index's candidates on stored fp32 vectors: the second pass of RefineFlatIndex.search.
//
// The base index returns k1 candidate ids per query; the host maps them to addresses of a row-major store
// vectors [n, d] (-1 = none).  This pass scores every candidate exactly against the query and keeps the k best:
//   euclidean  acc = fmaf(-dif, dif, acc), dif = x_e - y_e, e ascending from +0   (max_sim_kernel, kmeans.cu)
//   cosine     acc = fmaf(x_e, y_e, acc) on x / (||x|| + 1e-9) (normalize_columns); y as stored
// so a candidate's value equals tpq_max_sim(x_q, y) bit for bit, the same arithmetic as tpq_rerank.  Keys are
// make_key(score, address): ties go to the lower address; missing slots are (-inf, -1).
//
// Kernel: a CTA of 256 threads takes a tile of up to 8 queries at a time (persistent grid), as rerank_kernel does
// (query_tile.cuh: load the tile's x, then one warp per query selects).  The scoring differs: a candidate is 4·d
// contiguous bytes, so rather than one thread gathering its own candidate, each warp takes 32 candidates at a time and
// stages their rows into shared memory in chunks of 32 elements with cp.async, one row chunk (128 contiguous bytes,
// whole sectors) per warp-wide copy.  Two chunk buffers per warp: the next chunk is in flight while lane j runs
// candidate j's chain over the current one, serially from e = 0, so the chain above holds for any d.  Rows are padded
// to 33 floats, so the 32 lanes reading element e of 32 different rows hit 32 different banks.
#include "gemm_tile.cuh"
#include "query_tile.cuh"

extern "C" int tpq_merge_topk(const uint64_t* keys_in, int nq, int n_parts, int k, const int64_t* address2id,
                              int64_t capacity, float* values, int64_t* ids, int64_t* address, void* stream);

namespace tpq {

constexpr int kRfThreads = 256, kRfWarps = kRfThreads / 32;
constexpr int kRfChunk = 32;                          // row elements per staged chunk
constexpr int kRfRow = kRfChunk + 1;                  // padded row stride of a chunk buffer, in floats
constexpr int kRfBuf = 32 * kRfRow;                   // one chunk buffer: 32 rows

struct RefineArgs {
  const float* x; int d, nq;
  const int64_t* cand; int k1;
  const float* vectors; int64_t n;
  int k, kp, qt;
  size_t x_off, keys_off, lists_off, rows_off;        // shared-memory offsets
  uint64_t* keys_out;
};

// The plan, read by the workspace size and the launch.  QT: 8 queries per tile (one per warp for the selection), halved
// while the tile's shared memory exceeds the limit.  The chunk buffers (2 per warp, 67.6 KB) do not depend on d.
struct RefinePlan {
  RefineArgs a;
  size_t smem, ws_x, total;
  bool ok;
};

static RefinePlan plan_refine(int d, int nq, int k1, int k) {
  RefinePlan P{};
  RefineArgs& a = P.a;
  a.d = d; a.nq = nq; a.k1 = k1; a.k = k;
  a.kp = list_capacity(k);
  const size_t rows = (size_t)kRfWarps * 2 * kRfBuf * 4;
  auto tile = [&](int qt) {
    return align_up((size_t)qt * d * 4, 16) + (size_t)qt * k1 * 8 + (size_t)qt * a.kp * 8 + rows;
  };
  a.qt = kRfWarps;
  while (a.qt > 1 && tile(a.qt) > kSmemLimit) a.qt /= 2;
  a.x_off = 0;
  a.keys_off = align_up((size_t)a.qt * d * 4, 16);
  a.lists_off = a.keys_off + (size_t)a.qt * k1 * 8;
  a.rows_off = a.lists_off + (size_t)a.qt * a.kp * 8;
  P.smem = a.rows_off + rows;
  P.ok = P.smem <= kSmemLimit;
  P.ws_x = align_up((size_t)nq * k * 8, 256);                       // keys [nq, k] | normalised x [d, nq] (cosine)
  P.total = P.ws_x + align_up((size_t)d * nq * 4, 256);
  return P;
}

__device__ __forceinline__ void cp_async4(float* dst, const float* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"((uint32_t)__cvta_generic_to_shared(dst)), "l"(src)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory"); }

template <int METRIC>
__global__ void __launch_bounds__(kRfThreads)
refine_kernel(const RefineArgs A) {
  extern __shared__ __align__(16) uint8_t smem[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int d = A.d, k1 = A.k1;
  float* xs = reinterpret_cast<float*>(smem + A.x_off);
  uint64_t* keys = reinterpret_cast<uint64_t*>(smem + A.keys_off);
  uint64_t* lists = reinterpret_cast<uint64_t*>(smem + A.lists_off);
  float* rows = reinterpret_cast<float*>(smem + A.rows_off) + (size_t)warp * 2 * kRfBuf;   // this warp's two buffers
  const int nch = (d + kRfChunk - 1) / kRfChunk;
  const int tiles = (A.nq + A.qt - 1) / A.qt;
  for (int t = blockIdx.x; t < tiles; t += gridDim.x) {
    const int q0 = t * A.qt, nqt = min(A.qt, A.nq - q0);
    __syncthreads();                                                         // the previous tile's x and lists are read
    load_query_tile<kRfThreads>(A, xs, d, q0, nqt, tid);
    __syncthreads();
    // warp w's steps s = 0, 1, ...: group g = w + 8·(s / nch) of 32 candidates (pairs 32g .. 32g + 31 of the tile),
    // chunk c = s % nch of their rows
    const int np = nqt * k1, groups = (np + 31) / 32;
    const int steps = groups > warp ? (groups - warp + kRfWarps - 1) / kRfWarps * nch : 0;
    const int64_t* cand = A.cand + (size_t)q0 * k1;
    auto address = [&](int p) {                                              // pair p's store address, -1 = none
      const int64_t a = p < np ? __ldg(cand + p) : -1;
      return a >= 0 && a < A.n ? a : (int64_t)-1;
    };
    auto stage = [&](int s) {                                                // step s's chunk into buffer s & 1
      const int g = warp + kRfWarps * (s / nch), c = s % nch, e = c * kRfChunk + lane;
      const int64_t a = address(g * 32 + lane);
      float* buf = rows + (s & 1) * kRfBuf + lane;
      #pragma unroll 8
      for (int r = 0; r < 32; ++r) {
        const int64_t ar = __shfl_sync(0xffffffffu, a, r);
        if (ar >= 0 && e < d) cp_async4(buf + r * kRfRow, A.vectors + ar * d + e);
      }
      cp_async_commit();
    };
    float acc = 0.f;
    if (steps > 0) stage(0);
    for (int s = 0; s < steps; ++s) {
      if (s + 1 < steps) { stage(s + 1); cp_async_wait<1>(); }
      else cp_async_wait<0>();
      __syncwarp();                                                          // every lane's copies of step s have landed
      const int g = warp + kRfWarps * (s / nch), c = s % nch, p = g * 32 + lane;
      if (c == 0) acc = 0.f;
      if (p < np) {
        const float* y = rows + (s & 1) * kRfBuf + lane * kRfRow;
        const float* xq = xs + (p / k1) * d + c * kRfChunk;
        const int ne = min(kRfChunk, d - c * kRfChunk);
        #pragma unroll 8
        for (int e = 0; e < ne; ++e) {
          if (METRIC == TPQ_METRIC_EUCLIDEAN) { const float dif = __fsub_rn(xq[e], y[e]); acc = fmaf(-dif, dif, acc); }
          else acc = fmaf(xq[e], y[e], acc);
        }
        if (c == nch - 1) {
          const int64_t a = address(p);
          keys[p] = a >= 0 ? make_key(acc, (uint32_t)a) : 0ull;
        }
      }
      __syncwarp();                                                          // buffer s & 1 is read before step s + 2
    }
    __syncthreads();
    select_query_tile(A, keys, lists, k1, nqt, q0, warp, lane);
  }
}

template <int METRIC>
static int launch_refine(const RefinePlan& P, cudaStream_t st) {
  auto kern = refine_kernel<METRIC>;
  TPQ_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)P.smem));
  int per_sm = 0;
  TPQ_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kRfThreads, P.smem));
  const int tiles = (P.a.nq + P.a.qt - 1) / P.a.qt;
  const int grid = min(tiles, device_sm_count() * (per_sm > 0 ? per_sm : 1));
  kern<<<grid, kRfThreads, P.smem, st>>>(P.a);
  TPQ_LAUNCH_CHECK("refine_kernel");
  return TPQ_OK;
}

}  // namespace tpq

using namespace tpq;

extern "C" size_t tpq_refine_flat_workspace_bytes(int d, int nq, int k) {
  if (d <= 0 || nq <= 0 || k <= 0) return 0;
  return align_up((size_t)nq * k * 8, 256) + align_up((size_t)d * nq * 4, 256);
}

extern "C" int tpq_refine_flat(const float* x_dn, int d, int nq, const int64_t* candidates, int k1,
                               const float* vectors, int64_t n, int metric, int k, const int64_t* address2id,
                               float* values, int64_t* ids, int64_t* address, void* ws, size_t ws_bytes, void* stream) {
  TPQ_REQUIRE(metric == TPQ_METRIC_EUCLIDEAN || metric == TPQ_METRIC_COSINE,
              "tpq_refine_flat: unsupported metric %d (euclidean and cosine only)", metric);
  TPQ_REQUIRE(0 < k && k <= k1 && k1 <= 1024, "tpq_refine_flat: need 0 < k <= k1 <= 1024, got k=%d k1=%d", k, k1);
  TPQ_REQUIRE(d > 0 && nq >= 0 && n >= 0 && n <= 0xFFFFFFFFll, "tpq_refine_flat: bad sizes d=%d nq=%d n=%lld", d, nq,
              (long long)n);
  if (nq == 0) return TPQ_OK;
  TPQ_REQUIRE(x_dn && candidates && (vectors || n == 0) && address2id && values && ids,
              "tpq_refine_flat: null pointer");
  const RefinePlan P = plan_refine(d, nq, k1, k);
  if (!P.ok) { set_error("tpq_refine_flat: d=%d, k1=%d need more shared memory than one CTA has", d, k1); return TPQ_ERR_UNSUPPORTED; }
  if (!ws || ws_bytes < P.total) { set_error("tpq_refine_flat: workspace too small (%zu < %zu)", ws_bytes, P.total); return TPQ_ERR_WORKSPACE; }
  cudaStream_t st = (cudaStream_t)stream;
  uint8_t* w = reinterpret_cast<uint8_t*>(ws);
  RefinePlan L = P;
  L.a.keys_out = reinterpret_cast<uint64_t*>(w);
  L.a.x = x_dn;
  if (metric == TPQ_METRIC_COSINE) {
    float* xn = reinterpret_cast<float*>(w + P.ws_x);
    if (int rc = normalize_columns(x_dn, d, nq, 1e-9f, xn, st)) return rc;
    L.a.x = xn;
  }
  L.a.cand = candidates;
  L.a.vectors = vectors;
  L.a.n = n;
  const int rc = metric == TPQ_METRIC_EUCLIDEAN ? launch_refine<TPQ_METRIC_EUCLIDEAN>(L, st)
                                                : launch_refine<TPQ_METRIC_COSINE>(L, st);
  if (rc) return rc;
  return tpq_merge_topk(L.a.keys_out, nq, 1, k, address2id, n, values, ids, address, stream);
}
