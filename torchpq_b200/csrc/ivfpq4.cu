// IVFPQ4Index.search: inverted-file search over 4-bit PQ codes (16 codewords per sub-quantizer).
//
// The store is IVFPQ's cell container read in place, with no scan layout: storage [M/8, capacity] 32-bit words, word g
// of a slot holding sub-quantizers 8 g .. 8 g + 7, code m in bits 4 (m & 7) .. 4 (m & 7) + 3 (nibble m & 1 of byte
// m >> 1, low nibble first); is_empty marks holes; cell c scans [cell_start[c], cell_start[c] + cell_size[c]).
//
// One CTA per (query, slice of its probed tiles), query-major like ivfpq_range_kernel:
//   * prologue: warp 0 lays out the query's probe entries (probe_count / probe_visits, scan_layout.cuh) as runs of
//     32-slot tiles, while the CTA builds the query's LUT [M][16] fp32 in shared memory from pq_codebook [M, dsub, 16]
//     with lut.cuh's entry arithmetic.  At most 16 KB (M = 256): no table goes through global memory.
//   * lookups: row m is 16 consecutive words, so the 32 lanes of a warp reading row m touch at most 16 banks and lanes
//     with the same code broadcast: every LDS is conflict-free without the lane rotation of the 8-bit scan layout.
//   * streaming: lanes own consecutive slots, so a warp's load of word g is 128 contiguous bytes of _storage.  Per word
//     (w << 2) & 0x3C3C3C3C and (w >> 2) & 0x3C3C3C3C put 4 * code of the even and odd sub-quantizers in bytes; one PRMT
//     then zero-extends a byte into the LDS address, whose row offset 64 m is an immediate.  A lookup is PRMT + LDS + FADD.
//   * residual: the query half part1 = 2 dot is built once; on entering each cell the CTA forms the LUT as
//     part1 + part2[cell] (one fp32 add per entry, the 8-bit residual path's association).
//   * score: acc = LUT[0][code_0] + LUT[1][code_1] + ... added in ascending m from +0, one rounding per add; the value
//     is base + acc, base = the cell's coarse similarity (residual) or +0.
//   * selection: CtaTopK (common.cuh); each slice's sorted keys go to the workspace and tpq_merge_topk merges the slices.
//     Keys order by score descending, then address ascending, so the answer depends neither on slicing nor on chunking.
#include "lut.cuh"

extern "C" int tpq_merge_topk(const uint64_t* keys_in, int nq, int n_parts, int k, const int64_t* address2id,
                              int64_t capacity, float* values, int64_t* ids, int64_t* address, void* stream);

namespace tpq {

constexpr int kPq4NW = 8;                 // warps of a scan CTA
constexpr int kPq4MinB = 4;               // CTAs per SM the registers are sized for
constexpr int kPq4MaxM = 256;             // sub-quantizers: a 16 KB LUT
constexpr int kPq4Chunk = 8192;           // queries per scan launch
constexpr int kPq4MaxSlices = 64;

struct Pq4Args {
  const uint32_t* words;                  // storage as [M / 8, capacity] words
  const uint8_t* is_empty; const int64_t* cell_start; const int64_t* cell_size;
  int64_t capacity; int n_cells;
  const float* x; int ldx;                // queries [d, ldx] (normalised for cosine by the coarse stage)
  const float* pq;                        // [M, dsub, 16]
  const float* part2;                     // residual: [n_cells, M, 16]
  const int64_t* cells; const int64_t* npl; const float* base_sims;   // [nq, n_probe], [nq], [nq, n_probe]
  int M, dsub, metric, n_probe;
  int q_base, n, k, kp, S;
  uint64_t* keys;                         // [S][n][k] of this chunk
  int lut2, seg_a0, seg_n, seg_cell, seg_prefix, next, topk;   // shared-memory offsets (bytes)
};

__device__ __forceinline__ uint32_t prmt4(uint32_t a, uint32_t sel) {
  uint32_t d;
  asm("prmt.b32 %0, %1, 0, %2;" : "=r"(d) : "r"(a), "r"(sel));
  return d;
}

// The LUT [M][16] of query q (RES: the query half 2 dot), built by every thread of the CTA; entry e = 16 m + code.
template <bool RES>
__device__ __forceinline__ void build_lut4(float* out, const Pq4Args& A, int q) {
  const int kind = RES ? kLutPart1 : A.metric;
  for (int e = threadIdx.x; e < A.M * 16; e += blockDim.x) {
    const int m = e >> 4, c = e & 15;
    float dot = 0.f, a2 = 0.f, b2 = 0.f;
    for (int i = 0; i < A.dsub; ++i) {
      const float xv = __ldg(A.x + (size_t)(m * A.dsub + i) * A.ldx + q);
      const float p = __ldg(A.pq + ((size_t)m * A.dsub + i) * 16 + c);
      dot = dot_step(dot, xv, p); a2 = sq_step(a2, xv); b2 = sq_step(b2, p);
    }
    out[e] = lut_entry(kind, dot, a2, b2);
  }
}

// acc over the MW = M / 8 words of slot `a`, m ascending from +0.  MWP: MW rounded up to a power of two (the unroll).
template <int MWP>
__device__ __forceinline__ float adc4(const uint32_t* __restrict__ words, int64_t cap, uint32_t a, const float* lut, int MW) {
  float acc = 0.f;
  const uint8_t* base = reinterpret_cast<const uint8_t*>(lut);
  #pragma unroll
  for (int g0 = 0; g0 < MWP; g0 += 8) {
    constexpr int U = MWP < 8 ? MWP : 8;                 // words in flight
    uint32_t w[U];
    #pragma unroll
    for (int u = 0; u < U; ++u) w[u] = (g0 + u < MW) ? __ldg(words + (size_t)(g0 + u) * cap + a) : 0u;
    #pragma unroll
    for (int u = 0; u < U; ++u) {
      if (g0 + u >= MW) break;
      const uint32_t lo = (w[u] << 2) & 0x3C3C3C3Cu, hi = (w[u] >> 2) & 0x3C3C3C3Cu;
      const uint8_t* row = base + (g0 + u) * 8 * 64;
      #pragma unroll
      for (int b = 0; b < 4; ++b) {
        acc = __fadd_rn(acc, *reinterpret_cast<const float*>(row + (2 * b) * 64 + prmt4(lo, 0x4440u | b)));
        acc = __fadd_rn(acc, *reinterpret_cast<const float*>(row + (2 * b + 1) * 64 + prmt4(hi, 0x4440u | b)));
      }
    }
  }
  return acc;
}

// The tiles [lo, hi) of the query's probed runs, handed out to the warps by the CTA's cursor (which starts at 0).
// seg: this warp's current run; tiles only increase, within a call and from one call to the next.
template <int MWP>
__device__ __forceinline__ void scan_tiles(const Pq4Args& A, const uint8_t* smem, CtaTopK& tk, int* next, int& seg,
                                           int lo, int hi, float base, int lane) {
  const float* lut = reinterpret_cast<const float*>(smem);
  const uint32_t* seg_a0 = reinterpret_cast<const uint32_t*>(smem + A.seg_a0);
  const uint32_t* seg_n = reinterpret_cast<const uint32_t*>(smem + A.seg_n);
  const int32_t* seg_prefix = reinterpret_cast<const int32_t*>(smem + A.seg_prefix);
  const int MW = A.M >> 3;
  for (;;) {
    int b = 0;
    if (lane == 0) b = atomicAdd(next, 1);
    b = lo + __shfl_sync(0xffffffffu, b, 0);
    if (b >= hi) break;
    while (b >= seg_prefix[seg + 1]) ++seg;
    const uint32_t slot = (uint32_t)(b - seg_prefix[seg]) * 32u + lane;
    const uint32_t a = seg_a0[seg] + slot;
    const bool live = slot < seg_n[seg] && A.is_empty[a] == 0;
    const float s = __fadd_rn(base, adc4<MWP>(A.words, A.capacity, live ? a : 0u, lut, MW));
    const uint64_t key = make_key(s, a);
    tk.push(live && key > tk.threshold(), key, lane);
  }
}

template <int MWP, bool RES>
__global__ void __launch_bounds__(kPq4NW * 32, kPq4MinB)
ivfpq4_scan_kernel(const __grid_constant__ Pq4Args A) {
  extern __shared__ __align__(16) uint8_t smem[];
  float* lut = reinterpret_cast<float*>(smem);
  float* part1 = reinterpret_cast<float*>(smem + A.lut2);
  uint32_t* seg_a0 = reinterpret_cast<uint32_t*>(smem + A.seg_a0);
  uint32_t* seg_n = reinterpret_cast<uint32_t*>(smem + A.seg_n);
  int32_t* seg_cell = reinterpret_cast<int32_t*>(smem + A.seg_cell);
  int32_t* seg_prefix = reinterpret_cast<int32_t*>(smem + A.seg_prefix);
  int* next = reinterpret_cast<int*>(smem + A.next);
  const int qi = blockIdx.x / A.S, slice = blockIdx.x % A.S, q = A.q_base + qi;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int P = probe_count<RES>(A.npl[q], A.n_probe);
  if (warp == 0) {                                           // the visited entries as runs of 32-slot tiles
    const int64_t* cq = A.cells + (size_t)q * A.n_probe;
    int carry = 0;
    if (lane == 0) seg_prefix[0] = 0;
    for (int j0 = 0; j0 < P; j0 += 32) {
      const int j = j0 + lane;
      int nt = 0;
      if (j < P) {
        int64_t s;
        const bool visit = probe_visits(cq, j, A.n_cells, A.cell_start, s);
        const int64_t c = visit ? cq[j] : 0;
        const int64_t n = visit ? A.cell_size[c] : 0;
        nt = (int)((n + 31) >> 5);
        seg_a0[j] = (uint32_t)(visit ? s : 0);
        seg_n[j] = (uint32_t)n;
        if (RES) seg_cell[j] = (int32_t)c;
      }
      const int incl = warp_inclusive_scan(nt, lane);
      if (j < P) seg_prefix[j + 1] = carry + incl;
      carry += __shfl_sync(0xffffffffu, incl, 31);
    }
  }
  build_lut4<RES>(RES ? part1 : lut, A, q);
  CtaTopK tk;
  tk.init(smem + A.topk, kPq4NW, warp, A.kp, A.k);
  if (tid == 0) *next = 0;
  __syncthreads();
  const int total = seg_prefix[P];
  const int b_begin = (int)(((int64_t)total * slice) / A.S), b_end = (int)(((int64_t)total * (slice + 1)) / A.S);
  int seg = 0;
  if constexpr (RES) {
    for (int j = 0; j < P; ++j) {
      const int b0 = max(seg_prefix[j], b_begin), b1 = min(seg_prefix[j + 1], b_end);
      if (b1 <= b0) continue;                                // skipped entry, empty cell, another slice's tiles
      __syncthreads();                                       // every warp is done with the previous cell's LUT
      if (tid == 0) *next = 0;
      const float* p2 = A.part2 + (size_t)seg_cell[j] * A.M * 16;
      for (int e = tid; e < A.M * 16; e += blockDim.x) lut[e] = __fadd_rn(part1[e], __ldg(p2 + e));
      __syncthreads();
      scan_tiles<MWP>(A, smem, tk, next, seg, b0, b1, A.base_sims[(size_t)q * A.n_probe + j], lane);
    }
  } else {
    scan_tiles<MWP>(A, smem, tk, next, seg, b_begin, b_end, 0.f, lane);
  }
  tk.cta_drain(lane, warp);
  uint64_t* out = A.keys + ((size_t)slice * A.n + qi) * A.k;
  for (int i = tid; i < A.k; i += blockDim.x) out[i] = tk.list[i];
}

using Pq4Kernel = void (*)(Pq4Args);
template <bool RES>
static Pq4Kernel pq4_kernel_r(int M) {
  const int mw = M / 8;
  if (mw <= 1) return ivfpq4_scan_kernel<1, RES>;
  if (mw <= 2) return ivfpq4_scan_kernel<2, RES>;
  if (mw <= 4) return ivfpq4_scan_kernel<4, RES>;
  if (mw <= 8) return ivfpq4_scan_kernel<8, RES>;
  if (mw <= 16) return ivfpq4_scan_kernel<16, RES>;
  return ivfpq4_scan_kernel<32, RES>;
}

// What a search runs, from the sizes alone.  The workspace holds the coarse stage of the whole batch (as
// tpq_ivfpq_search's) and the slices' keys of one chunk of queries.
struct Pq4Plan {
  int S, chunk, kp;
  size_t coarse, coarse_bytes, sims, cells, npl, xn, keys, total;
};

static Pq4Plan plan_pq4(int d, int nq, int n_cells, int n_probe, int k) {
  Pq4Plan P{};
  P.kp = list_capacity(k);
  const int want = device_sm_count() * 8;                    // two waves of four CTAs per SM
  P.S = nq >= want ? 1 : ((want + nq - 1) / nq > kPq4MaxSlices ? kPq4MaxSlices : (want + nq - 1) / nq);
  P.chunk = nq < kPq4Chunk ? nq : kPq4Chunk;
  size_t o = 0;
  auto take = [&](size_t bytes) { const size_t at = o; o += align_up(bytes, 256); return at; };
  P.coarse_bytes = tpq_coarse_workspace_bytes(d, nq, n_cells);
  P.coarse = take(P.coarse_bytes);
  P.sims = take((size_t)nq * n_probe * 4);
  P.cells = take((size_t)nq * n_probe * 8);
  P.npl = take((size_t)nq * 8);
  P.xn = take((size_t)nq * d * 4);
  P.keys = take((size_t)P.S * P.chunk * k * 8);
  P.total = o;
  return P;
}

// Shared memory of a scan CTA: LUT, the residual query half, the probe runs, the cursor, then CtaTopK's.
static size_t pq4_smem(Pq4Args& A, int n_probe, bool residual) {
  size_t o = 0;
  auto take = [&](size_t bytes) { const size_t at = o; o += align_up(bytes, 16); return (int)at; };
  take((size_t)A.M * 64);
  A.lut2 = take(residual ? (size_t)A.M * 64 : 0);
  A.seg_a0 = take((size_t)n_probe * 4);
  A.seg_n = take((size_t)n_probe * 4);
  A.seg_cell = take(residual ? (size_t)n_probe * 4 : 0);
  A.seg_prefix = take(((size_t)n_probe + 1) * 4);
  A.next = take(8);
  A.topk = take(CtaTopK::bytes(kPq4NW, A.kp));
  return o;
}

}  // namespace tpq

using namespace tpq;

extern "C" size_t tpq_ivfpq4_workspace_bytes(int d, int nq, int n_cells, int n_probe, int k) {
  if (d <= 0 || nq <= 0 || n_cells <= 0 || n_probe <= 0 || k <= 0 || k > 1024) return 0;
  return plan_pq4(d, nq, n_cells, n_probe, k).total;
}

extern "C" int tpq_ivfpq4_search(const float* x_dn, int d, int M, int nq, int metric, const uint8_t* storage,
                                 const uint8_t* is_empty, const int64_t* cell_start, const int64_t* cell_size,
                                 const int64_t* address2id, int64_t capacity, int n_cells, const float* vq_codebook,
                                 const float* pq_codebook, const float* part2, const int64_t* cells,
                                 const int64_t* n_probe_list, const float* base_sims, int n_probe, int smart,
                                 float temperature, int k, float* values, int64_t* ids, int64_t* address, void* ws,
                                 size_t ws_bytes, void* stream) {
  const char* name = "tpq_ivfpq4_search";
  if (metric != TPQ_METRIC_EUCLIDEAN && metric != TPQ_METRIC_COSINE) {
    set_error("%s: unsupported metric %d (euclidean and cosine only)", name, metric);
    return TPQ_ERR_UNSUPPORTED;
  }
  TPQ_REQUIRE(k > 0, "%s: k must be in (0, 1024], got %d", name, k);
  if (k > 1024) { set_error("%s: k=%d > 1024 is not supported", name, k); return TPQ_ERR_UNSUPPORTED; }
  TPQ_REQUIRE(M > 0 && M % 8 == 0, "%s: n_subvectors=%d must be a positive multiple of 8", name, M);
  if (M > kPq4MaxM) { set_error("%s: n_subvectors=%d > %d is not supported", name, M, kPq4MaxM); return TPQ_ERR_UNSUPPORTED; }
  TPQ_REQUIRE(d > 0 && d % M == 0, "%s: d=%d must be a positive multiple of n_subvectors=%d", name, d, M);
  TPQ_REQUIRE(nq >= 0 && n_cells > 0 && n_probe >= 1 && capacity >= 0, "%s: bad sizes nq=%d n_cells=%d n_probe=%d "
              "capacity=%lld", name, nq, n_cells, n_probe, (long long)capacity);
  TPQ_REQUIRE(capacity < (int64_t(1) << 32), "%s: capacity=%lld exceeds the 32-bit address of a key", name,
              (long long)capacity);
  TPQ_REQUIRE((cells == nullptr) == (n_probe_list == nullptr), "%s: cells and n_probe_list go together", name);
  if (!cells) {
    TPQ_REQUIRE(n_probe <= n_cells, "%s: n_probe=%d must be in [1, n_cells=%d]", name, n_probe, n_cells);
    if (n_probe > 1024) { set_error("%s: n_probe=%d > 1024 is not supported", name, n_probe); return TPQ_ERR_UNSUPPORTED; }
  }
  const bool residual = part2 != nullptr;
  TPQ_REQUIRE(!residual || metric == TPQ_METRIC_EUCLIDEAN, "%s: residual IVFPQ is defined for the euclidean metric", name);
  TPQ_REQUIRE(!residual || !cells || base_sims, "%s: a residual search over given cells needs base_sims", name);
  TPQ_REQUIRE(values && ids, "%s: null output", name);
  if (nq == 0) return TPQ_OK;
  TPQ_REQUIRE(x_dn && pq_codebook && cell_start && cell_size && (cells || vq_codebook), "%s: null query, codebook or "
              "cell table", name);
  TPQ_REQUIRE(capacity == 0 || (storage && is_empty && address2id), "%s: null store", name);
  TPQ_REQUIRE(reinterpret_cast<uintptr_t>(storage) % 4 == 0, "%s: storage must be 4-byte aligned", name);
  const Pq4Plan P = plan_pq4(d, nq, n_cells, n_probe, k);
  Pq4Args A{};
  A.M = M; A.kp = P.kp;
  const size_t smem = pq4_smem(A, n_probe, residual);
  if (smem > kSmemLimit) {
    set_error("%s: M=%d n_probe=%d k=%d needs %zu B of shared memory (> 227 KB)", name, M, n_probe, k, smem);
    return TPQ_ERR_UNSUPPORTED;
  }
  if (!ws || ws_bytes < P.total) {
    set_error("%s: workspace too small (%zu < %zu)", name, ws_bytes, P.total);
    return TPQ_ERR_WORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  uint8_t* w = reinterpret_cast<uint8_t*>(ws);
  const float* xs = x_dn;
  if (!cells) {                                              // tpq_ivfpq_search's coarse stage
    if (metric == TPQ_METRIC_COSINE) {
      float* xn = reinterpret_cast<float*>(w + P.xn);
      if (int rc = tpq_normalize_columns(x_dn, d, nq, xn, stream)) return rc;
      xs = xn;
    }
    float* sims = reinterpret_cast<float*>(w + P.sims);
    int64_t *cw = reinterpret_cast<int64_t*>(w + P.cells), *nw = reinterpret_cast<int64_t*>(w + P.npl);
    if (int rc = tpq_coarse_probe(xs, vq_codebook, d, nq, n_cells, n_probe, smart, temperature, sims, cw, nw,
                                  w + P.coarse, P.coarse_bytes, stream))
      return rc;
    cells = cw; n_probe_list = nw; base_sims = sims;
  }
  A.words = reinterpret_cast<const uint32_t*>(storage); A.is_empty = is_empty;
  A.cell_start = cell_start; A.cell_size = cell_size; A.capacity = capacity; A.n_cells = n_cells;
  A.x = xs; A.ldx = nq; A.pq = pq_codebook; A.part2 = part2;
  A.cells = cells; A.npl = n_probe_list; A.base_sims = base_sims;
  A.dsub = d / M; A.metric = metric; A.n_probe = n_probe; A.k = k; A.S = P.S;
  A.keys = reinterpret_cast<uint64_t*>(w + P.keys);
  const Pq4Kernel kern = residual ? pq4_kernel_r<true>(M) : pq4_kernel_r<false>(M);
  TPQ_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  // capacity == 0: every key is empty and the id table is never read, so any non-null pointer will do
  const int64_t* a2i = capacity ? address2id : reinterpret_cast<const int64_t*>(A.keys);
  for (int q0 = 0; q0 < nq; q0 += P.chunk) {
    const int n = nq - q0 < P.chunk ? nq - q0 : P.chunk;
    A.q_base = q0; A.n = n;
    kern<<<(unsigned)n * P.S, kPq4NW * 32, smem, st>>>(A);
    TPQ_LAUNCH_CHECK("ivfpq4_scan_kernel");
    if (int rc = tpq_merge_topk(A.keys, n, P.S, k, a2i, capacity, values + (size_t)q0 * k, ids + (size_t)q0 * k,
                                address ? address + (size_t)q0 * k : nullptr, stream))
      return rc;
  }
  return TPQ_OK;
}
