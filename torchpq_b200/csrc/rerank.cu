// Re-rank of IVFPQ candidates on a second, finer PQ code: the second pass of IVFPQRIndex.search.
//
// The first pass is the ordinary IVFPQ scan on the first M code bytes of every item; it returns k1 candidate addresses
// per query.  This pass reads each candidate's codes from the reference-layout `_storage` ([(M + Mr)/4, cap, 4]: the
// first M/4 word planes are the scanned code, the next Mr/4 the re-rank code), reconstructs the vector, scores it
// exactly against the query and keeps the k best:
//   reconstruction  y_e = y2_e + y1_e with use_residual (y1: first-level codebook entry, y2: re-rank codebook entry of
//                   the candidate's codes for dimension e), else y_e = y2_e
//   euclidean       acc = fmaf(-dif, dif, acc), dif = x_e - y_e, e ascending from +0   (max_sim_kernel, kmeans.cu)
//   cosine          acc = fmaf(x_e, y_e, acc) on x / (||x|| + 1e-9) (normalize_columns, as the search), y not normalised
// so a candidate's value equals tpq_max_sim(x_q, decode(codes)) bit for bit.  Keys are make_key(score, address): ties
// go to the lower address, as in every other top-k here; missing slots are (-inf, -1).
//
// Kernel: a CTA of 256 threads takes a tile of up to 8 queries at a time (persistent grid, one tile after another).
//   1. its queries' x go to shared memory;
//   2. one thread per (query, candidate) pair: the candidate's code words are gathered from `_storage` into the
//      thread's own column of a shared array (all loads in flight together: each word is its own 32-byte sector), then
//      the thread runs the d-long fmaf chain, its codebook lookups `cb[e * 256 + code]` gathered from shared memory;
//   3. warp w sorts query w's k1 keys, 64 at a time, into a kp-slot list (merge_staged + warp_merge_run) and writes its
//      first k keys; tpq_merge_topk with one part decodes them into values, addresses and ids.
// Steps 1 and 3 are query_tile.cuh's, shared with refine.cu.
// Codebooks: each is d * 1 KB (128 KB at d = 128), so at d = 128 only one fits in shared memory beside the tile.  The
// re-rank codebook is staged first because every score reads it; the first-level one only with use_residual.  A
// codebook that does not fit is read through the read-only cache.  CTAs persist across tiles so that the staging is paid
// once per CTA, not once per tile.
#include "gemm_tile.cuh"
#include "query_tile.cuh"

extern "C" int tpq_merge_topk(const uint64_t* keys_in, int nq, int n_parts, int k, const int64_t* address2id,
                              int64_t capacity, float* values, int64_t* ids, int64_t* address, void* stream);

namespace tpq {

constexpr int kRrThreads = 256, kRrWarps = kRrThreads / 32;

struct RerankArgs {
  const float* x; int d, nq;
  const int64_t* cand; int k1;
  const uint32_t* storage; int64_t cap;
  int M, Mr;
  const float* cb1; const float* cb2;
  int k, kp, qt;
  size_t x_off, codes_off, keys_off, lists_off, cb1_off, cb2_off;     // shared-memory offsets; cb*_off == 0: not staged
  uint64_t* keys_out;
};

// The plan, read by the workspace size and the launch.  QT: 8 queries per tile (one per warp for the selection), halved
// while the tile's shared memory exceeds the limit.  Then the codebooks are staged while they fit.
struct RerankPlan {
  RerankArgs a;
  size_t smem, ws_x, total;
  bool ok;
};

static RerankPlan plan_rerank(int d, int nq, int k1, int M, int Mr, int residual, int k) {
  RerankPlan P{};
  RerankArgs& a = P.a;
  a.d = d; a.nq = nq; a.k1 = k1; a.M = M; a.Mr = Mr; a.k = k;
  a.kp = list_capacity(k);
  const int W = (residual ? M / 4 : 0) + Mr / 4;                   // code words read per candidate
  auto tile = [&](int qt) {
    return align_up((size_t)qt * d * 4, 16) + (size_t)W * kRrThreads * 4 + (size_t)qt * k1 * 8 + (size_t)qt * a.kp * 8;
  };
  a.qt = kRrWarps;
  while (a.qt > 1 && tile(a.qt) > kSmemLimit) a.qt /= 2;
  a.x_off = 0;
  a.codes_off = align_up((size_t)a.qt * d * 4, 16);
  a.keys_off = a.codes_off + (size_t)W * kRrThreads * 4;
  a.lists_off = a.keys_off + (size_t)a.qt * k1 * 8;
  P.smem = a.lists_off + (size_t)a.qt * a.kp * 8;
  P.ok = P.smem <= kSmemLimit;
  const size_t cb = (size_t)d * 256 * 4;
  if (P.smem + cb <= kSmemLimit) { a.cb2_off = P.smem; P.smem += cb; }
  if (residual && P.smem + cb <= kSmemLimit) { a.cb1_off = P.smem; P.smem += cb; }
  P.ws_x = align_up((size_t)nq * k * 8, 256);                       // keys [nq, k] | normalised x [d, nq] (cosine)
  P.total = P.ws_x + align_up((size_t)d * nq * 4, 256);
  return P;
}

__device__ __forceinline__ uint32_t code_byte(const uint32_t* col, int m) {
  return (col[(m >> 2) * kRrThreads] >> (8 * (m & 3))) & 0xFFu;
}

template <bool RESIDUAL, int METRIC>
__global__ void __launch_bounds__(kRrThreads)
rerank_kernel(const RerankArgs A) {
  extern __shared__ __align__(16) uint8_t smem[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int d = A.d, k1 = A.k1, M = A.M, Mr = A.Mr;
  float* xs = reinterpret_cast<float*>(smem + A.x_off);
  uint32_t* col = reinterpret_cast<uint32_t*>(smem + A.codes_off) + tid;     // this thread's column of code words
  uint64_t* keys = reinterpret_cast<uint64_t*>(smem + A.keys_off);
  uint64_t* lists = reinterpret_cast<uint64_t*>(smem + A.lists_off);
  const float* cb1 = A.cb1;
  const float* cb2 = A.cb2;
  if (A.cb2_off) {
    float* s = reinterpret_cast<float*>(smem + A.cb2_off);
    for (int i = tid; i < d * 256; i += kRrThreads) s[i] = __ldg(A.cb2 + i);
    cb2 = s;
  }
  if (RESIDUAL && A.cb1_off) {
    float* s = reinterpret_cast<float*>(smem + A.cb1_off);
    for (int i = tid; i < d * 256; i += kRrThreads) s[i] = __ldg(A.cb1 + i);
    cb1 = s;
  }
  const int W1 = RESIDUAL ? M / 4 : 0, W = W1 + Mr / 4;
  const int g0 = RESIDUAL ? 0 : M / 4;                                       // first word plane read
  const int dsub1 = RESIDUAL ? d / M : 1, dsub2 = d / Mr;
  const int tiles = (A.nq + A.qt - 1) / A.qt;
  for (int t = blockIdx.x; t < tiles; t += gridDim.x) {
    const int q0 = t * A.qt, nqt = min(A.qt, A.nq - q0);
    __syncthreads();                                                         // the previous tile's x and lists are read
    load_query_tile<kRrThreads>(A, xs, d, q0, nqt, tid);
    __syncthreads();
    for (int p = tid; p < nqt * k1; p += kRrThreads) {
      const int q = p / k1;
      const int64_t a = A.cand[(size_t)q0 * k1 + p];
      uint64_t key = 0ull;
      if (a >= 0 && a < A.cap) {
        #pragma unroll 8
        for (int w = 0; w < W; ++w) col[w * kRrThreads] = __ldg(A.storage + (size_t)(g0 + w) * A.cap + a);
        const float* xq = xs + q * d;
        float acc = 0.f;
        int m1 = 0, i1 = 0, m2 = 0, i2 = 0;
        uint32_t c1 = RESIDUAL ? code_byte(col, 0) : 0u, c2 = code_byte(col + W1 * kRrThreads, 0);
        for (int e = 0; e < d; ++e) {
          float y = cb2[e * 256 + c2];
          if (RESIDUAL) y = __fadd_rn(y, cb1[e * 256 + c1]);
          if (METRIC == TPQ_METRIC_EUCLIDEAN) { const float dif = __fsub_rn(xq[e], y); acc = fmaf(-dif, dif, acc); }
          else acc = fmaf(xq[e], y, acc);
          if (++i2 == dsub2 && e + 1 < d) { i2 = 0; c2 = code_byte(col + W1 * kRrThreads, ++m2); }
          if (RESIDUAL && ++i1 == dsub1 && e + 1 < d) { i1 = 0; c1 = code_byte(col, ++m1); }
        }
        key = make_key(acc, (uint32_t)a);
      }
      keys[p] = key;
    }
    __syncthreads();
    select_query_tile(A, keys, lists, k1, nqt, q0, warp, lane);
  }
}

template <bool RESIDUAL, int METRIC>
static int launch_rerank(const RerankPlan& P, cudaStream_t st) {
  auto kern = rerank_kernel<RESIDUAL, METRIC>;
  TPQ_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)P.smem));
  int per_sm = 0;
  TPQ_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kRrThreads, P.smem));
  const int tiles = (P.a.nq + P.a.qt - 1) / P.a.qt;
  const int grid = min(tiles, device_sm_count() * (per_sm > 0 ? per_sm : 1));
  kern<<<grid, kRrThreads, P.smem, st>>>(P.a);
  TPQ_LAUNCH_CHECK("rerank_kernel");
  return TPQ_OK;
}

}  // namespace tpq

using namespace tpq;

extern "C" size_t tpq_rerank_workspace_bytes(int d, int nq, int k) {
  if (d <= 0 || nq <= 0 || k <= 0) return 0;
  return align_up((size_t)nq * k * 8, 256) + align_up((size_t)d * nq * 4, 256);
}

extern "C" int tpq_rerank(const float* x_dn, int d, int nq, const int64_t* candidates, int k1,
                          const uint8_t* storage, int64_t capacity, int M, int Mr,
                          const float* pq_codebook, const float* pq_rerank_codebook, int use_residual, int metric,
                          int k, const int64_t* address2id, float* values, int64_t* ids, int64_t* address,
                          void* ws, size_t ws_bytes, void* stream) {
  TPQ_REQUIRE(metric == TPQ_METRIC_EUCLIDEAN || metric == TPQ_METRIC_COSINE,
              "tpq_rerank: unsupported metric %d (euclidean and cosine only)", metric);
  TPQ_REQUIRE(0 < k && k <= k1 && k1 <= 1024, "tpq_rerank: need 0 < k <= k1 <= 1024, got k=%d k1=%d", k, k1);
  TPQ_REQUIRE(M > 0 && M % 4 == 0 && Mr > 0 && Mr % 4 == 0,
              "tpq_rerank: n_subvectors=%d and n_subvectors_rerank=%d must be positive multiples of 4", M, Mr);
  TPQ_REQUIRE(d > 0 && d % M == 0 && d % Mr == 0, "tpq_rerank: d=%d must be a multiple of M=%d and Mr=%d", d, M, Mr);
  TPQ_REQUIRE(nq >= 0 && capacity >= 0 && capacity <= 0xFFFFFFFFll, "tpq_rerank: bad sizes nq=%d capacity=%lld", nq,
              (long long)capacity);
  if (nq == 0) return TPQ_OK;
  TPQ_REQUIRE(x_dn && candidates && storage && pq_rerank_codebook && (pq_codebook || !use_residual) && address2id &&
              values && ids, "tpq_rerank: null pointer");
  const RerankPlan P = plan_rerank(d, nq, k1, M, Mr, use_residual, k);
  if (!P.ok) { set_error("tpq_rerank: d=%d, M + Mr=%d, k1=%d need more shared memory than one CTA has", d, M + Mr, k1); return TPQ_ERR_UNSUPPORTED; }
  if (!ws || ws_bytes < P.total) { set_error("tpq_rerank: workspace too small (%zu < %zu)", ws_bytes, P.total); return TPQ_ERR_WORKSPACE; }
  cudaStream_t st = (cudaStream_t)stream;
  uint8_t* w = reinterpret_cast<uint8_t*>(ws);
  RerankPlan L = P;
  L.a.keys_out = reinterpret_cast<uint64_t*>(w);
  L.a.x = x_dn;
  if (metric == TPQ_METRIC_COSINE) {
    float* xn = reinterpret_cast<float*>(w + P.ws_x);
    if (int rc = normalize_columns(x_dn, d, nq, 1e-9f, xn, st)) return rc;
    L.a.x = xn;
  }
  L.a.cand = candidates;
  L.a.storage = reinterpret_cast<const uint32_t*>(storage);
  L.a.cap = capacity;
  L.a.cb1 = pq_codebook; L.a.cb2 = pq_rerank_codebook;
  int rc;
  if (use_residual) rc = metric == TPQ_METRIC_EUCLIDEAN ? launch_rerank<true, TPQ_METRIC_EUCLIDEAN>(L, st)
                                                        : launch_rerank<true, TPQ_METRIC_COSINE>(L, st);
  else rc = metric == TPQ_METRIC_EUCLIDEAN ? launch_rerank<false, TPQ_METRIC_EUCLIDEAN>(L, st)
                                           : launch_rerank<false, TPQ_METRIC_COSINE>(L, st);
  if (rc) return rc;
  return tpq_merge_topk(L.a.keys_out, nq, 1, k, address2id, capacity, values, ids, address, stream);
}
