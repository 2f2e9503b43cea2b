// IVFFlatIndex.search: inverted-file search with exact fp32 distances over a flat store.
//
// The store is IVFPQ's cell container with fp32 columns: _storage [d, capacity] (tpq_store_codes with code_size = 4 d
// bytes), cell c holding slots [cell_start[c], cell_start[c] + cell_capacity[c]) of which [start, start + cell_size) are
// scanned, holes marked in is_empty.  A query visits the cells of its probe list by the IVFPQ rule (probe_count and
// probe_visits, scan_layout.cuh) and scores every live vector there with flat.cu's GEMM tile and epilogues, so a score
// is FlatIndex's bit for bit.
//
// Cell-major: the (query, probe entry) pairs are grouped by cell and each cell becomes a small GEMM -- the queries that
// probe it times its vectors -- so a probed cell is read once per chunk of queries, not once per query.  Per chunk:
//   1. the chunk's queries are copied to a [d, n] matrix; cells == NULL: the coarse probe of tpq_ivfpq_search on it;
//   2. ivfflat_pairs_count_kernel: the visited pairs per cell, and each pair's rank in its cell;
//   3. ivfflat_plan_kernel: each cell's pairs padded to the query tile QT, and the work items (cell, query tile, column
//      slice), largest slice first;
//   4. ivfflat_pairs_scatter_kernel + ivfflat_gather_kernel: the pairs' queries as one [d, pad_cap] matrix with zero
//      columns for the padding, which GemmTile<QT>::run reads unmodified;
//   5. ivfflat_scan_kernel: per item, GEMM + epilogue + is_empty mask + one WarpTopK per pair over the slice's 128-column
//      tiles -> keys[j * S + slice][q][:] for the pair (query q, entry j); parts no pair writes stay zero (empty);
//   6. tpq_merge_topk over the n_probe * S parts of every query -> values, ids, address.
// The key order is total (score descending, address ascending) and every part is an exact top-k of its columns, so the
// answer does not depend on QT, S or the chunk.
// IVFSQIndex.search (tpq_ivfsq_search) is the same search over an SQCodec-coded store (word planes of 8-bit codes or
// fp16): its scan instances read the codes through gemm_tile.cuh's BLoadSQ8 / BLoadSQ16, which decode them as the tile
// stages them, so its scores are this search's over the decoded store, bit for bit.
#include "fused_scan.cuh"
#include "scan_layout.cuh"

extern "C" int tpq_merge_topk(const uint64_t* keys_in, int nq, int n_parts, int k, const int64_t* address2id,
                              int64_t capacity, float* values, int64_t* ids, int64_t* address, void* stream);

namespace tpq {

constexpr float kIvfFlatEps = 1e-8f;            // flat.cu's kFlatEps: metric.cosine_similarity's `norm + 1e-8`
constexpr size_t kIvfFlatKeyBytes = size_t(256) << 20;   // the chunk's keys [n_probe * S, n, k] stay within 256 MB
constexpr int kIvfFlatMaxChunk = 16384;         // and a chunk holds at most this many queries
constexpr size_t kIvfRangeXgBytes = size_t(256) << 20;   // the range search's gathered pair queries stay within 256 MB
constexpr int kIvfFlatBuckets = 128;            // classes of the largest-first item order (4 per octave)
constexpr int kIvfFlatMaxSlices = 128;          // n_probe * S parts per query at most (n_probe permitting)

// The plan, read by the workspace size and the search.  Every size is known before the search, from (d, nq, n_cells,
// n_probe, k) alone; k == 0 is the range search's, with no lists and no keys:
//   chunk0: queries per chunk when S = 1: the most whose keys fit kIvfFlatKeyBytes (k == 0: whose n_probe pair columns
//           of d floats fit kIvfRangeXgBytes), at most kIvfFlatMaxChunk;
//   QT:     16, 32 or 64: the smallest that holds a cell's expected pairs (chunk0 * n_probe / n_cells), halved while the
//           shared memory exceeds 227 KB (k = 1024 gives 16, as in flat.cu);
//   S:      column slices per (cell, query tile), enough for two CTAs per SM when the pairs make fewer tiles, with
//           n_probe * S <= max(n_probe, 128) parts per query;
//   chunk:  queries per chunk with S slices (k == 0: chunk0).
// Per chunk of n queries: pairs = n * n_probe slots; the padded pair columns pad_cap = pairs + min(n_cells, pairs) *
// (QT - 1) bound sum over cells of round_up(pairs of the cell, QT), and items = S * pad_cap / QT bounds the work items.
// Past one chunk the workspace stops growing with nq.
struct IvfFlatPlan {
  int qt, kp, S, chunk;
  int64_t pairs, pad_cap, items;
  size_t smem;
  size_t keys, xc, xs, xp, xn, coarse, coarse_bytes, sims, cells, npl, cnt, off, slot, pq, pj, itm, xg, total;
};

static IvfFlatPlan plan_ivfflat(int d, int nq, int n_cells, int n_probe, int k) {
  IvfFlatPlan P{};
  P.kp = k ? list_capacity(k) : 0;
  auto chunk_of = [&](size_t budget, size_t per_query) {
    size_t c = budget / per_query;
    c = c < (size_t)kIvfFlatMaxChunk ? c : (size_t)kIvfFlatMaxChunk;
    return (int)(c < 1 ? 1 : (c > (size_t)nq ? (size_t)nq : c));
  };
  const size_t keys_per_query = (size_t)n_probe * k * 8;
  const int chunk0 = k ? chunk_of(kIvfFlatKeyBytes, keys_per_query) : chunk_of(kIvfRangeXgBytes, (size_t)n_probe * d * 4);
  const int64_t per_cell = ((int64_t)chunk0 * n_probe + n_cells - 1) / n_cells;
  P.qt = 16;
  while (P.qt < 64 && P.qt < per_cell) P.qt *= 2;
  while (P.qt > 16 && fused_smem_bytes(P.qt, P.kp) > kSmemLimit) P.qt /= 2;
  P.smem = fused_smem_bytes(P.qt, P.kp);
  const int64_t tiles = ((int64_t)chunk0 * n_probe + P.qt - 1) / P.qt;
  const int64_t want = 2 * (int64_t)device_sm_count();
  const int smax = n_probe >= kIvfFlatMaxSlices ? 1 : kIvfFlatMaxSlices / n_probe;
  int64_t S = tiles >= want ? 1 : (want + tiles - 1) / tiles;
  P.S = (int)(S > smax ? smax : S);
  P.chunk = k ? chunk_of(kIvfFlatKeyBytes, keys_per_query * P.S) : chunk0;
  P.pairs = (int64_t)P.chunk * n_probe;
  P.pad_cap = P.pairs + (P.pairs < n_cells ? P.pairs : n_cells) * (P.qt - 1);
  P.items = P.S * (P.pad_cap / P.qt);
  const size_t n = (size_t)P.chunk;
  size_t o = 0;
  auto take = [&](size_t bytes) { const size_t at = o; o += align_up(bytes, 256); return at; };
  P.keys = take((size_t)n_probe * P.S * n * k * 8);
  P.xc = take((size_t)d * n * 4);                      // the chunk's queries
  P.xs = take((size_t)d * n * 4);                      // cosine: normalize_columns(xc, 1e-8), what the GEMM reads
  P.xp = take((size_t)d * n * 4);                      // cosine: tpq_normalize_columns(xc), what the probe reads
  P.xn = take(n * 4);                                  // euclidean: |x|^2
  P.coarse_bytes = tpq_coarse_workspace_bytes(d, (int)n, n_cells);
  P.coarse = take(P.coarse_bytes);
  P.sims = take(n * n_probe * 4);
  P.cells = take(n * n_probe * 8);
  P.npl = take(n * 8);
  P.cnt = take(((size_t)n_cells + 2) * 4);             // pairs per cell, then [n_cells] = items, [n_cells + 1] = columns
  P.off = take((size_t)n_cells * 4);                   // each cell's first padded pair column
  P.slot = take((size_t)P.pairs * 4);
  P.pq = take((size_t)P.pad_cap * 4);                  // chunk-local query of each padded pair column (-1: padding)
  P.pj = take((size_t)P.pad_cap * 4);                  // probe entry of each padded pair column
  P.itm = take((size_t)P.items * 16);
  P.xg = take((size_t)d * P.pad_cap * 4);
  P.total = o;
  return P;
}

// thread per (query, entry) of the chunk: the visited pairs counted per cell; slot = the pair's rank in its cell (-1: none)
__global__ void ivfflat_pairs_count_kernel(const int64_t* __restrict__ cells, const int64_t* __restrict__ npl, int n,
                                           int n_probe, int n_cells, const int64_t* __restrict__ cell_start,
                                           const int64_t* __restrict__ cell_size, int* __restrict__ cell_cnt,
                                           int* __restrict__ slot) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (int64_t)n * n_probe) return;
  const int qi = (int)(t / n_probe), j = (int)(t % n_probe);
  int pos = -1;
  int64_t s;
  if (j < probe_count<false>(npl[qi], n_probe) && probe_visits(cells + (size_t)qi * n_probe, j, n_cells, cell_start, s)) {
    const int64_t c = cells[t];
    if (cell_size[c] > 0) pos = atomicAdd(cell_cnt + c, 1);
  }
  slot[t] = pos;
}

// One CTA: off[c] = exclusive prefix of round_up(cnt[c], qt); cnt[n_cells] = items, cnt[n_cells + 1] = padded columns.
// Items: the ceil(cnt / qt) query tiles x S slices of every cell with pairs, ordered by the slice's column tiles
// descending in classes of 4 per octave.
__global__ void __launch_bounds__(1024) ivfflat_plan_kernel(int* __restrict__ cnt, const int64_t* __restrict__ cell_size,
                                                            int n_cells, int qt, int S, int* __restrict__ off,
                                                            int4* __restrict__ items) {
  __shared__ int hist[kIvfFlatBuckets], base[kIvfFlatBuckets], wsum[32], carry;
  const int tid = threadIdx.x;
  for (int i = tid; i < kIvfFlatBuckets; i += 1024) hist[i] = 0;
  if (tid == 0) carry = 0;
  __syncthreads();
  auto bucket_of = [&](int c) {
    const int64_t per = ((cell_size[c] + GB - 1) / GB + S - 1) / S;             // column tiles of the largest slice
    const uint32_t w = (uint32_t)(per < 1 ? 1 : (per > 0x7fffffff ? 0x7fffffff : per));
    const int lg = 31 - __clz(w);
    const int sub = lg >= 2 ? (int)((w >> (lg - 2)) & 3u) : (int)((w << (2 - lg)) & 3u);
    return kIvfFlatBuckets - 1 - min(kIvfFlatBuckets - 1, 4 * lg + sub);       // more work -> smaller bucket index
  };
  for (int c0 = 0; c0 < n_cells; c0 += 1024) {
    const int c = c0 + tid;
    const int v = c < n_cells ? cnt[c] : 0;
    const int tiles = (v + qt - 1) / qt;
    const int incl = cta_inclusive_scan(tiles * qt, wsum, carry);
    if (c < n_cells) {
      off[c] = incl - tiles * qt;
      if (tiles) atomicAdd(&hist[bucket_of(c)], tiles * S);
    }
  }
  __syncthreads();
  if (tid == 0) {
    int s = 0;
    for (int b = 0; b < kIvfFlatBuckets; ++b) { base[b] = s; s += hist[b]; }
    cnt[n_cells] = s;
    cnt[n_cells + 1] = carry;
  }
  __syncthreads();
  for (int c = tid; c < n_cells; c += 1024) {
    const int tiles = (cnt[c] + qt - 1) / qt;
    if (!tiles) continue;
    const int pos = atomicAdd(&base[bucket_of(c)], tiles * S);
    for (int i = 0; i < tiles * S; ++i) items[pos + i] = make_int4(c, i / S, i % S, 0);
  }
}

__global__ void ivfflat_pairs_scatter_kernel(const int64_t* __restrict__ cells, int n, int n_probe,
                                             const int* __restrict__ slot, const int* __restrict__ off,
                                             int* __restrict__ pair_q, int* __restrict__ pair_j) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (int64_t)n * n_probe) return;
  const int s = slot[t];
  if (s < 0) return;
  const int p = off[cells[t]] + s;
  pair_q[p] = (int)(t / n_probe);
  pair_j[p] = (int)(t % n_probe);
}

// xg[g, p] = x[g, pair_q[p]] for the padded pair columns p < cnt[n_cells + 1]; padding columns are zero
__global__ void ivfflat_gather_kernel(const float* __restrict__ x, int d, int n, const int* __restrict__ pair_q,
                                      const int* __restrict__ n_cols, int64_t pad_cap, float* __restrict__ xg) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= *n_cols) return;
  const int q = pair_q[p];
  for (int g = blockIdx.y; g < d; g += gridDim.y) xg[(size_t)g * pad_cap + p] = q >= 0 ? x[(size_t)g * n + q] : 0.f;
}

// One CTA per work item (cell, query tile, slice), 256 threads; the CTAs past the chunk's item count return at once.
// The slice's columns run in 128-column tiles: GemmTile<QT> over the tile's QT pair columns of xg, flat.cu's epilogue
// (euclidean ((acc * 2) - |x|^2) - norms[a] with norms = |b|^2; cosine acc / norms[a] with norms = |b| + 1e-8 and x
// normalised), then per pair row a filter against its k-th key and a WarpTopK that never takes an is_empty slot.
// Two CTAs per SM, as flat_search_kernel.  BL is the store's B loader (gemm_tile.cuh): BLoadF32 for IVFFlatIndex's fp32
// columns, BLoadSQ8 / BLoadSQ16 for IVFSQIndex's code words, decoded as the tile stages them, so that an SQ store scores
// exactly as its decoded fp32 image would.  base [*, ld] is the store, `extra` the loader's own pointers (SQ8: lower,
// range), last so that the fp32 instances keep IVFFlatIndex's parameter list.
template <int QT, int METRIC, class BL, class... Extra>
__global__ void __launch_bounds__(256, 2)
ivfflat_scan_kernel(const float* __restrict__ xg, int d, int pad_cap, const int* __restrict__ pair_q,
                    const int* __restrict__ pair_j, const int4* __restrict__ items, const int* __restrict__ cnt,
                    int n_cells, const int* __restrict__ off, const typename BL::T* __restrict__ base, int64_t ld,
                    const uint8_t* __restrict__ is_empty, const int64_t* __restrict__ cell_start,
                    const int64_t* __restrict__ cell_size, const float* __restrict__ norms, const float* __restrict__ xn,
                    int n, int S, int k, int kp, uint64_t* __restrict__ keys_out, Extra... extra) {
  using G = GemmTile<QT, BL>;
  if ((int)blockIdx.x >= cnt[n_cells]) return;
  const int4 it = items[blockIdx.x];
  const int cell = it.x, sl = it.z;
  const int64_t size = cell_size[cell], start = cell_start[cell];
  const int64_t T = (size + GB - 1) / GB;
  const int64_t c_begin = start + T * sl / S * GB;
  const int64_t c_end = start + (T * (sl + 1) / S * GB < size ? T * (sl + 1) / S * GB : size);
  if (c_begin >= c_end) return;                        // a slice without columns: its parts stay empty
  const int p0 = off[cell] + it.y * QT;
  const int rows = cnt[cell] - it.y * QT < QT ? cnt[cell] - it.y * QT : QT;
  extern __shared__ __align__(16) uint8_t smem[];
  auto& stages = *reinterpret_cast<typename G::Stages*>(smem);
  float (*Sc)[GB] = reinterpret_cast<float (*)[GB]>(smem + sizeof(typename G::Stages));
  uint64_t* lists = reinterpret_cast<uint64_t*>(smem + sizeof(typename G::Stages) + (size_t)QT * GB * 4);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, tx = tid & 15, ty = tid >> 4;
  uint64_t* wbuf = lists + (size_t)QT * kp + (size_t)warp * kTopkBuf;
  float a2[G::MI];
  #pragma unroll
  for (int i = 0; i < G::MI; ++i) {
    const int r = G::row(i, ty);
    a2[i] = (METRIC == TPQ_METRIC_EUCLIDEAN && r < rows) ? xn[pair_q[p0 + r]] : 0.f;
  }
  for (int i = tid; i < QT * kp; i += 256) lists[i] = 0ull;
  // (the barrier after G::run's first stash orders these stores before the first selection, and each selection
  //  before the next tile's score stores)
  for (int64_t c0 = c_begin; c0 < c_end; c0 += GB) {
    const int cols = (int)(c_end - c0 < GB ? c_end - c0 : GB);
    float acc[G::MI][8];
    G::run(xg, pad_cap, p0, BL{base + c0, ld, extra...}, cols, d, stages, acc);
    float nc[8];
    #pragma unroll
    for (int j = 0; j < 8; ++j) nc[j] = G::col(j, tx) < cols ? norms[c0 + G::col(j, tx)] : 1.f;
    #pragma unroll
    for (int i = 0; i < G::MI; ++i) {
      const int r = G::row(i, ty);
      float o[8];
      #pragma unroll
      for (int j = 0; j < 8; ++j) {
        if (METRIC == TPQ_METRIC_EUCLIDEAN) o[j] = __fsub_rn(__fsub_rn(__fmul_rn(acc[i][j], 2.f), a2[i]), nc[j]);
        else o[j] = __fdiv_rn(acc[i][j], nc[j]);
      }
      *reinterpret_cast<float4*>(&Sc[r][tx * 4]) = make_float4(o[0], o[1], o[2], o[3]);
      *reinterpret_cast<float4*>(&Sc[r][64 + tx * 4]) = make_float4(o[4], o[5], o[6], o[7]);
    }
    __syncthreads();
    bool live[4];
    #pragma unroll
    for (int u = 0; u < 4; ++u) live[u] = u * 32 + lane < cols && is_empty[c0 + u * 32 + lane] == 0;
    for (int r = warp; r < rows; r += kFusedWarps) {
      WarpTopK tk{lists + (size_t)r * kp, wbuf, kp, k, 0};
      uint64_t thr = tk.kth();
      #pragma unroll
      for (int u = 0; u < 4; ++u) {
        const uint64_t key = live[u] ? make_key(Sc[r][u * 32 + lane], (uint32_t)(c0 + u * 32 + lane)) : 0ull;
        if (tk.push(live[u] && key > thr, key, lane)) thr = tk.kth();
      }
      tk.flush(lane);
    }
  }
  __syncthreads();                                     // the lists were last written by their own warps
  for (int r = warp; r < rows; r += kFusedWarps) {
    const int p = p0 + r;
    uint64_t* dst = keys_out + (((size_t)pair_j[p] * S + sl) * n + pair_q[p]) * k;
    for (int i = lane; i < k; i += 32) dst[i] = lists[(size_t)r * kp + i];
  }
}

// One CTA per work item, as ivfflat_scan_kernel: the same GEMM, epilogue and is_empty mask, then every score > thr
// (strict, in fp32; NaN never passes) goes to the match buffer as (pair row, key); a flush maps the row to its query,
// q_base + pair_q[row], writes at most `cap` matches to keys_out / q_out and counts them all in *total.
template <int QT, int METRIC, class BL, class... Extra>
__global__ void __launch_bounds__(256, 2)
ivfflat_range_kernel(const float* __restrict__ xg, int d, int pad_cap, const int* __restrict__ pair_q,
                     const int4* __restrict__ items, const int* __restrict__ cnt, int n_cells,
                     const int* __restrict__ off, const typename BL::T* __restrict__ base, int64_t ld,
                     const uint8_t* __restrict__ is_empty, const int64_t* __restrict__ cell_start,
                     const int64_t* __restrict__ cell_size, const float* __restrict__ norms,
                     const float* __restrict__ xn, int S, float thr, int q_base, uint64_t* __restrict__ keys_out,
                     int32_t* __restrict__ q_out, int64_t cap, unsigned long long* __restrict__ total,
                     Extra... extra) {
  using G = GemmTile<QT, BL>;
  if ((int)blockIdx.x >= cnt[n_cells]) return;
  const int4 it = items[blockIdx.x];
  const int cell = it.x, sl = it.z;
  const int64_t size = cell_size[cell], start = cell_start[cell];
  const int64_t T = (size + GB - 1) / GB;
  const int64_t c_begin = start + T * sl / S * GB;
  const int64_t c_end = start + (T * (sl + 1) / S * GB < size ? T * (sl + 1) / S * GB : size);
  if (c_begin >= c_end) return;
  const int p0 = off[cell] + it.y * QT;
  const int rows = cnt[cell] - it.y * QT < QT ? cnt[cell] - it.y * QT : QT;
  extern __shared__ __align__(16) uint8_t smem[];
  auto& stages = *reinterpret_cast<typename G::Stages*>(smem);
  RangeBuf& mb = *reinterpret_cast<RangeBuf*>(smem + sizeof(typename G::Stages));
  const int tid = threadIdx.x, lane = tid & 31, tx = tid & 15, ty = tid >> 4;
  float a2[G::MI];
  #pragma unroll
  for (int i = 0; i < G::MI; ++i) {
    const int r = G::row(i, ty);
    a2[i] = (METRIC == TPQ_METRIC_EUCLIDEAN && r < rows) ? xn[pair_q[p0 + r]] : 0.f;
  }
  auto query = [&](int r) { return q_base + pair_q[p0 + r]; };
  if (tid == 0) mb.cnt = 0;                            // ordered before the first append by G::run's first barrier
  for (int64_t c0 = c_begin; c0 < c_end; c0 += GB) {
    const int cols = (int)(c_end - c0 < GB ? c_end - c0 : GB);
    float acc[G::MI][8];
    G::run(xg, pad_cap, p0, BL{base + c0, ld, extra...}, cols, d, stages, acc);
    float nc[8];
    bool live[8];
    #pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int c = G::col(j, tx);
      live[j] = c < cols && is_empty[c0 + c] == 0;
      nc[j] = c < cols ? norms[c0 + c] : 1.f;
    }
    uint32_t pass = 0;
    #pragma unroll
    for (int i = 0; i < G::MI; ++i) {
      const bool row_ok = G::row(i, ty) < rows;
      #pragma unroll
      for (int j = 0; j < 8; ++j) {
        float o;
        if (METRIC == TPQ_METRIC_EUCLIDEAN) o = __fsub_rn(__fsub_rn(__fmul_rn(acc[i][j], 2.f), a2[i]), nc[j]);
        else o = __fdiv_rn(acc[i][j], nc[j]);
        acc[i][j] = o;
        if (row_ok && live[j] && o > thr) pass |= 1u << (i * 8 + j);
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

}  // namespace tpq

using namespace tpq;

extern "C" size_t tpq_ivfflat_workspace_bytes(int d, int nq, int n_cells, int n_probe, int k) {
  if (d <= 0 || nq <= 0 || n_cells <= 0 || n_probe <= 0 || k <= 0 || k > 1024) return 0;
  return plan_ivfflat(d, nq, n_cells, n_probe, k).total;
}

// The chunk's part of the workspace, at the plan's offsets.
struct IvfChunk {
  float *xc, *xs, *xp, *xn, *xg;
  int *cnt, *off, *slot, *pair_q, *pair_j;
  int4* items;
};

static IvfChunk ivf_chunk_ws(const IvfFlatPlan& P, uint8_t* w) {
  IvfChunk W;
  W.xc = reinterpret_cast<float*>(w + P.xc); W.xs = reinterpret_cast<float*>(w + P.xs);
  W.xp = reinterpret_cast<float*>(w + P.xp); W.xn = reinterpret_cast<float*>(w + P.xn);
  W.xg = reinterpret_cast<float*>(w + P.xg);
  W.cnt = reinterpret_cast<int*>(w + P.cnt); W.off = reinterpret_cast<int*>(w + P.off);
  W.slot = reinterpret_cast<int*>(w + P.slot); W.pair_q = reinterpret_cast<int*>(w + P.pq);
  W.pair_j = reinterpret_cast<int*>(w + P.pj);
  W.items = reinterpret_cast<int4*>(w + P.itm);
  return W;
}

// Steps 1-4 of ivf_chunks for the chunk [q0, q0 + n) of the batch.
static int ivf_chunk_pairs(const IvfFlatPlan& P, uint8_t* w, const IvfChunk& W, const float* x_dn, int d, int nq, int q0,
                           int n, const float* vq_codebook, int n_cells, const int64_t* cells,
                           const int64_t* n_probe_list, int n_probe, int smart, float temperature, int metric,
                           const int64_t* cell_start, const int64_t* cell_size, cudaStream_t st) {
  void* stream = st;
  float *xc = W.xc, *xs = W.xs, *xp = W.xp, *xn = W.xn;
  TPQ_CUDA(cudaMemcpy2DAsync(xc, (size_t)n * 4, x_dn + q0, (size_t)nq * 4, (size_t)n * 4, d, cudaMemcpyDeviceToDevice, st));
  const int64_t *cq = cells ? cells + (size_t)q0 * n_probe : nullptr, *npl = cells ? n_probe_list + q0 : nullptr;
  if (!cells) {                                        // tpq_ivfpq_search's coarse stage, on the chunk
    const float* xprobe = xc;
    if (metric == TPQ_METRIC_COSINE) {
      if (int rc = tpq_normalize_columns(xc, d, n, xp, stream)) return rc;
      xprobe = xp;
    }
    int64_t *cw = reinterpret_cast<int64_t*>(w + P.cells), *nw = reinterpret_cast<int64_t*>(w + P.npl);
    if (int rc = tpq_coarse_probe(xprobe, vq_codebook, d, n, n_cells, n_probe, smart, temperature,
                                  reinterpret_cast<float*>(w + P.sims), cw, nw, w + P.coarse, P.coarse_bytes, stream))
      return rc;
    cq = cw; npl = nw;
  }
  const float* xq = xc;
  if (metric == TPQ_METRIC_EUCLIDEAN) {
    if (int rc = col_sqnorms(xc, d, n, n, xn, st)) return rc;
  } else {
    if (int rc = normalize_columns(xc, d, n, kIvfFlatEps, xs, st)) return rc;
    xq = xs;
  }
  const int64_t nt = (int64_t)n * n_probe;
  const unsigned pgrid = (unsigned)((nt + 255) / 256);
  TPQ_CUDA(cudaMemsetAsync(W.cnt, 0, ((size_t)n_cells + 2) * 4, st));
  TPQ_CUDA(cudaMemsetAsync(W.pair_q, 0xFF, (size_t)P.pad_cap * 4, st));
  ivfflat_pairs_count_kernel<<<pgrid, 256, 0, st>>>(cq, npl, n, n_probe, n_cells, cell_start, cell_size, W.cnt, W.slot);
  TPQ_LAUNCH_CHECK("ivfflat_pairs_count_kernel");
  ivfflat_plan_kernel<<<1, 1024, 0, st>>>(W.cnt, cell_size, n_cells, P.qt, P.S, W.off, W.items);
  TPQ_LAUNCH_CHECK("ivfflat_plan_kernel");
  ivfflat_pairs_scatter_kernel<<<pgrid, 256, 0, st>>>(cq, n, n_probe, W.slot, W.off, W.pair_q, W.pair_j);
  TPQ_LAUNCH_CHECK("ivfflat_pairs_scatter_kernel");
  const dim3 ggrid((unsigned)((P.pad_cap + 255) / 256), (unsigned)(d < 64 ? d : 64));
  ivfflat_gather_kernel<<<ggrid, 256, 0, st>>>(xq, d, n, W.pair_q, W.cnt + n_cells + 1, P.pad_cap, W.xg);
  TPQ_LAUNCH_CHECK("ivfflat_gather_kernel");
  return TPQ_OK;
}

// The batch in chunks of P.chunk queries, shared by the search and the range search.  For each chunk [q0, q0 + n):
// steps 1-4 -- the chunk's queries, its probe lists (the caller's, or the coarse probe's), |x|^2 (euclidean) or the
// normalised queries (cosine), the visited pairs grouped by cell, the work items and the pairs' queries gathered into
// W.xg -- then scan(q0, n).
template <class Scan>
static int ivf_chunks(const IvfFlatPlan& P, uint8_t* w, const IvfChunk& W, const float* x_dn, int d, int nq,
                      const float* vq_codebook, int n_cells, const int64_t* cells, const int64_t* n_probe_list,
                      int n_probe, int smart, float temperature, int metric, const int64_t* cell_start,
                      const int64_t* cell_size, cudaStream_t st, Scan scan) {
  for (int q0 = 0; q0 < nq; q0 += P.chunk) {
    const int n = nq - q0 < P.chunk ? nq - q0 : P.chunk;
    if (int rc = ivf_chunk_pairs(P, w, W, x_dn, d, nq, q0, n, vq_codebook, n_cells, cells, n_probe_list, n_probe, smart,
                                 temperature, metric, cell_start, cell_size, st))
      return rc;
    if (int rc = scan(q0, n)) return rc;
  }
  return TPQ_OK;
}

// The checks of the search and the range search on the metric, the sizes and the probe lists.
static int ivf_check(const char* name, int d, int nq, int n_cells, int n_probe, int64_t capacity, int metric,
                     const int64_t* cells, const int64_t* n_probe_list) {
  if (metric != TPQ_METRIC_EUCLIDEAN && metric != TPQ_METRIC_COSINE) {
    set_error("%s: unsupported metric %d (euclidean and cosine only)", name, metric);
    return TPQ_ERR_UNSUPPORTED;
  }
  TPQ_REQUIRE(d > 0 && nq >= 0 && n_cells > 0 && n_probe >= 1 && capacity >= 0,
              "%s: bad sizes d=%d nq=%d n_cells=%d n_probe=%d capacity=%lld", name, d, nq, n_cells, n_probe,
              (long long)capacity);
  TPQ_REQUIRE(capacity < (int64_t(1) << 32), "%s: capacity=%lld exceeds the 32-bit address of a key", name,
              (long long)capacity);
  TPQ_REQUIRE((cells == nullptr) == (n_probe_list == nullptr), "%s: cells and n_probe_list go together", name);
  if (!cells) {
    TPQ_REQUIRE(n_probe <= n_cells, "n_probe=%d must be in [1, n_cells=%d]", n_probe, n_cells);
    if (n_probe > 1024) { set_error("n_probe=%d > 1024 is not supported", n_probe); return TPQ_ERR_UNSUPPORTED; }
  }
  return TPQ_OK;
}

// The body of tpq_ivfflat_search and tpq_ivfsq_search: `name` prefixes the messages, BL reads the store (storage
// [*, capacity] words) and `extra` are its own pointers, checked by the caller.
template <class BL, class... Extra>
static int ivf_search(const char* name, const float* x_dn, int d, int nq, const float* vq_codebook, int n_cells,
                      const typename BL::T* storage, int64_t capacity, const uint8_t* is_empty,
                      const int64_t* cell_start, const int64_t* cell_size, const float* norms, int metric,
                      const int64_t* cells, const int64_t* n_probe_list, int n_probe, int smart, float temperature,
                      int k, const int64_t* address2id, float* values, int64_t* ids, int64_t* address, void* ws,
                      size_t ws_bytes, void* stream, Extra... extra) {
  TPQ_REQUIRE(k > 0, "k must be in (0, 1024], got %d", k);
  if (k > 1024) { set_error("k=%d > 1024 is not supported", k); return TPQ_ERR_UNSUPPORTED; }
  if (int rc = ivf_check(name, d, nq, n_cells, n_probe, capacity, metric, cells, n_probe_list)) return rc;
  TPQ_REQUIRE(values && ids, "%s: null output", name);
  if (nq == 0) return TPQ_OK;
  TPQ_REQUIRE(x_dn && cell_start && cell_size && (cells || vq_codebook), "%s: null query or cell table", name);
  TPQ_REQUIRE(capacity == 0 || (storage && is_empty && norms && address2id), "%s: null store", name);
  const IvfFlatPlan P = plan_ivfflat(d, nq, n_cells, n_probe, k);
  if (!ws || ws_bytes < P.total) {
    set_error("%s: workspace too small (%zu < %zu)", name, ws_bytes, P.total);
    return TPQ_ERR_WORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  uint8_t* w = reinterpret_cast<uint8_t*>(ws);
  uint64_t* keys = reinterpret_cast<uint64_t*>(w + P.keys);
  const IvfChunk W = ivf_chunk_ws(P, w);
  // capacity == 0: every key is empty and the id table is never read, so any non-null pointer will do
  const int64_t* a2i = capacity ? address2id : reinterpret_cast<const int64_t*>(keys);
  return ivf_chunks(P, w, W, x_dn, d, nq, vq_codebook, n_cells, cells, n_probe_list, n_probe, smart, temperature, metric,
                    cell_start, cell_size, st, [&](int q0, int n) {
    TPQ_CUDA(cudaMemsetAsync(keys, 0, (size_t)n_probe * P.S * n * k * 8, st));
    if (int rc = fused_launch<false>(
            "ivfflat_scan_kernel", P.qt, metric, dim3((unsigned)P.items), P.smem, st,
            [](auto q, auto m) { return ivfflat_scan_kernel<decltype(q)::value, decltype(m)::value, BL, Extra...>; },
            W.xg, d, (int)P.pad_cap, W.pair_q, W.pair_j, W.items, W.cnt, n_cells, W.off, storage, capacity, is_empty,
            cell_start, cell_size, norms, W.xn, n, P.S, k, P.kp, keys, extra...))
      return rc;
    return tpq_merge_topk(keys, n, n_probe * P.S, k, a2i, capacity, values + (size_t)q0 * k, ids + (size_t)q0 * k,
                          address ? address + (size_t)q0 * k : nullptr, stream);
  });
}

// The checks of tpq_ivfsq_search and tpq_ivfsq_range_search on the code width, d and the 8-bit codec's lower and range,
// then body(BLoadSQ16{}) or body(BLoadSQ8{}, lower, range): the loader and its own pointers.
template <class Body>
static int ivf_sq(const char* name, int bits, int d, const float* lower, const float* range, Body body) {
  if (bits != 8 && bits != 16) {
    set_error("%s: bits=%d is not supported (8 and 16 only)", name, bits);
    return TPQ_ERR_UNSUPPORTED;
  }
  TPQ_REQUIRE(d > 0 && d % (bits == 8 ? 4 : 2) == 0, "%s: d=%d must be a positive multiple of %d for %d bits", name, d,
              bits == 8 ? 4 : 2, bits);
  if (bits == 16) return body(BLoadSQ16{});
  TPQ_REQUIRE(lower && range, "%s: null lower or range (8 bits)", name);
  TPQ_REQUIRE((reinterpret_cast<uintptr_t>(lower) | reinterpret_cast<uintptr_t>(range)) % 16 == 0,
              "%s: lower and range must be 16-byte aligned", name);
  return body(BLoadSQ8{}, lower, range);
}

extern "C" int tpq_ivfflat_search(const float* x_dn, int d, int nq, const float* vq_codebook, int n_cells,
                                  const float* storage, int64_t capacity, const uint8_t* is_empty,
                                  const int64_t* cell_start, const int64_t* cell_size, const float* norms, int metric,
                                  const int64_t* cells, const int64_t* n_probe_list, int n_probe, int smart,
                                  float temperature, int k, const int64_t* address2id, float* values, int64_t* ids,
                                  int64_t* address, void* ws, size_t ws_bytes, void* stream) {
  return ivf_search<BLoadF32>("tpq_ivfflat_search", x_dn, d, nq, vq_codebook, n_cells, storage, capacity, is_empty,
                              cell_start, cell_size, norms, metric, cells, n_probe_list, n_probe, smart, temperature,
                              k, address2id, values, ids, address, ws, ws_bytes, stream);
}

extern "C" int tpq_ivfsq_search(const float* x_dn, int d, int nq, const float* vq_codebook, int n_cells,
                                const uint8_t* storage, int bits, const float* lower, const float* range,
                                int64_t capacity, const uint8_t* is_empty, const int64_t* cell_start,
                                const int64_t* cell_size, const float* norms, int metric, const int64_t* cells,
                                const int64_t* n_probe_list, int n_probe, int smart, float temperature, int k,
                                const int64_t* address2id, float* values, int64_t* ids, int64_t* address, void* ws,
                                size_t ws_bytes, void* stream) {
  const uint32_t* words = reinterpret_cast<const uint32_t*>(storage);
  return ivf_sq("tpq_ivfsq_search", bits, d, lower, range, [&](auto bl, auto... extra) {
    return ivf_search<decltype(bl)>("tpq_ivfsq_search", x_dn, d, nq, vq_codebook, n_cells, words, capacity, is_empty,
                                    cell_start, cell_size, norms, metric, cells, n_probe_list, n_probe, smart,
                                    temperature, k, address2id, values, ids, address, ws, ws_bytes, stream, extra...);
  });
}

// ----------------------------------------------------------------------------- range search
extern "C" size_t tpq_ivfflat_range_workspace_bytes(int d, int nq, int n_cells, int n_probe) {
  if (d <= 0 || nq <= 0 || n_cells <= 0 || n_probe <= 0) return 0;
  return plan_ivfflat(d, nq, n_cells, n_probe, 0).total;
}

// The body of tpq_ivfflat_range_search and tpq_ivfsq_range_search, as ivf_search is of the searches.
template <class BL, class... Extra>
static int ivf_range(const char* name, const float* x_dn, int d, int nq, const float* vq_codebook, int n_cells,
                     const typename BL::T* storage, int64_t capacity, const uint8_t* is_empty,
                     const int64_t* cell_start, const int64_t* cell_size, const float* norms, int metric,
                     const int64_t* cells, const int64_t* n_probe_list, int n_probe, int smart, float temperature,
                     float threshold, uint64_t* match_keys, int32_t* match_query, int64_t cap, uint64_t* total,
                     void* ws, size_t ws_bytes, void* stream, Extra... extra) {
  if (int rc = ivf_check(name, d, nq, n_cells, n_probe, capacity, metric, cells, n_probe_list)) return rc;
  TPQ_REQUIRE(threshold == threshold, "%s: the threshold is NaN", name);
  TPQ_REQUIRE(cap >= 0, "%s: cap=%lld is negative", name, (long long)cap);
  TPQ_REQUIRE(total && (cap == 0 || (match_keys && match_query)), "%s: null total or match buffer", name);
  if (nq == 0) return TPQ_OK;
  TPQ_REQUIRE(x_dn && cell_start && cell_size && (cells || vq_codebook), "%s: null query or cell table", name);
  TPQ_REQUIRE(capacity == 0 || (storage && is_empty && norms), "%s: null store", name);
  const IvfFlatPlan P = plan_ivfflat(d, nq, n_cells, n_probe, 0);
  if (!ws || ws_bytes < P.total) {
    set_error("%s: workspace too small (%zu < %zu)", name, ws_bytes, P.total);
    return TPQ_ERR_WORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  TPQ_CUDA(cudaMemsetAsync(total, 0, sizeof(uint64_t), st));
  if (capacity == 0) return TPQ_OK;                    // nothing to score
  uint8_t* w = reinterpret_cast<uint8_t*>(ws);
  const IvfChunk W = ivf_chunk_ws(P, w);
  return ivf_chunks(P, w, W, x_dn, d, nq, vq_codebook, n_cells, cells, n_probe_list, n_probe, smart, temperature, metric,
                    cell_start, cell_size, st, [&](int q0, int) {
    return fused_launch<false>(
        "ivfflat_range_kernel", P.qt, metric, dim3((unsigned)P.items), P.smem, st,
        [](auto q, auto m) { return ivfflat_range_kernel<decltype(q)::value, decltype(m)::value, BL, Extra...>; },
        W.xg, d, (int)P.pad_cap, W.pair_q, W.items, W.cnt, n_cells, W.off, storage, capacity, is_empty, cell_start,
        cell_size, norms, W.xn, P.S, threshold, q0, match_keys, match_query, cap,
        reinterpret_cast<unsigned long long*>(total), extra...);
  });
}

extern "C" int tpq_ivfflat_range_search(const float* x_dn, int d, int nq, const float* vq_codebook, int n_cells,
                                        const float* storage, int64_t capacity, const uint8_t* is_empty,
                                        const int64_t* cell_start, const int64_t* cell_size, const float* norms,
                                        int metric, const int64_t* cells, const int64_t* n_probe_list, int n_probe,
                                        int smart, float temperature, float threshold, uint64_t* match_keys,
                                        int32_t* match_query, int64_t cap, uint64_t* total, void* ws, size_t ws_bytes,
                                        void* stream) {
  return ivf_range<BLoadF32>("tpq_ivfflat_range_search", x_dn, d, nq, vq_codebook, n_cells, storage, capacity,
                             is_empty, cell_start, cell_size, norms, metric, cells, n_probe_list, n_probe, smart,
                             temperature, threshold, match_keys, match_query, cap, total, ws, ws_bytes, stream);
}

extern "C" int tpq_ivfsq_range_search(const float* x_dn, int d, int nq, const float* vq_codebook, int n_cells,
                                      const uint8_t* storage, int bits, const float* lower, const float* range,
                                      int64_t capacity, const uint8_t* is_empty, const int64_t* cell_start,
                                      const int64_t* cell_size, const float* norms, int metric, const int64_t* cells,
                                      const int64_t* n_probe_list, int n_probe, int smart, float temperature,
                                      float threshold, uint64_t* match_keys, int32_t* match_query, int64_t cap,
                                      uint64_t* total, void* ws, size_t ws_bytes, void* stream) {
  const uint32_t* words = reinterpret_cast<const uint32_t*>(storage);
  return ivf_sq("tpq_ivfsq_range_search", bits, d, lower, range, [&](auto bl, auto... extra) {
    return ivf_range<decltype(bl)>("tpq_ivfsq_range_search", x_dn, d, nq, vq_codebook, n_cells, words, capacity,
                                   is_empty, cell_start, cell_size, norms, metric, cells, n_probe_list, n_probe, smart,
                                   temperature, threshold, match_keys, match_query, cap, total, ws, ws_bytes, stream,
                                   extra...);
  });
}
