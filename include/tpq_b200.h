/*
 * tpq_b200 -- C ABI of the H100-native IVFPQ search path.
 *
 * Drop-in boundary for torchpq.index.IVFPQIndex.search() (reference
 * torchpq/index/IVFPQIndex.py:469-524) and the ops below it.  Every entry point
 * takes plain DEVICE pointers, sizes and a cudaStream_t (passed as void*); the
 * caller (PyTorch host code) owns every buffer, the library never allocates,
 * frees or keeps caller memory, never synchronises the host, and launches only
 * on the stream it is given.  Return value: 0 on success, negative tpq_status
 * on error (tpq_last_error() gives the message for the calling thread).
 *
 * All kernels are hand-written CUDA compiled ahead of time for sm_90a.
 */
#ifndef TPQ_B200_H
#define TPQ_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
  TPQ_OK = 0,
  TPQ_ERR_BAD_ARG = -1,      /* mirrors the reference's Python asserts (shape / dtype / range) */
  TPQ_ERR_UNSUPPORTED = -2,  /* valid in the reference but not built here (says which) */
  TPQ_ERR_WORKSPACE = -3,    /* caller workspace too small */
  TPQ_ERR_CUDA = -4          /* a CUDA runtime call failed (message carries cudaGetErrorString) */
} tpq_status;

/* MANHATTAN exists for k-means assignment only (tpq_max_sim, tpq_kmeans_assign, exact kernel) and INNER for the flat
 * search only (tpq_flat_*); every IVFPQ, LUT and relayout entry point rejects both: the IVFPQ index is defined for
 * euclidean and cosine. */
enum { TPQ_METRIC_EUCLIDEAN = 0, TPQ_METRIC_COSINE = 1, TPQ_METRIC_MANHATTAN = 2, TPQ_METRIC_INNER = 3 };

/* Index state read by search.  Field-for-field the buffers of the reference's
 * CellContainer / BaseContainer / codecs (container/CellContainer.py:46-81,
 * container/BaseContainer.py:32-38, codec/VQCodec.py:15-17, codec/PQCodec.py:36-46),
 * followed by the scan ("shadow") layout derived from them by tpq_relayout_*. */
typedef struct tpq_index {
  int32_t d_vector;          /* d */
  int32_t n_subvectors;      /* M, M % 4 == 0 (contiguous_size 4, IVFPQIndex.py:41) */
  int32_t n_cells;           /* C */
  int32_t metric;            /* TPQ_METRIC_* (reference `distance`) */
  int64_t capacity;          /* address slots = _address2id.shape[0] */
  const float*   vq_codebook;   /* [d, C]        vq_codec.codebook */
  const float*   pq_codebook;   /* [M, d/M, 256] pq_codec.codebook */
  const uint8_t* storage;       /* [code_size/4, capacity, 4] _storage (may be NULL once the scan layout exists) */
  const uint8_t* is_empty;      /* [capacity] _is_empty */
  const int64_t* cell_start;    /* [C] _cell_start */
  const int64_t* cell_size;     /* [C] _cell_size */
  const int64_t* address2id;    /* [capacity] _address2id */
  /* ---- scan layout (all NULL / 0 until tpq_relayout_codes has run) ---- */
  int32_t m_pad;                /* M rounded up to a multiple of 32 */
  int32_t shard_rank;           /* this shard owns cells c with c % shard_world == shard_rank */
  int32_t shard_world;
  int32_t mean_cell_live;       /* live vectors per cell of this shard, rounded down (0 = unknown); selects the scan */
  int64_t n_blocks;             /* 32-vector blocks in codes_scan */
  const uint8_t*  codes_scan;   /* [n_blocks, m_pad/16, 32 lanes, 16 B], lane-rotated (DESIGN.md) */
  const uint32_t* block_valid;  /* [n_blocks] bit l set = vector l of the block is live */
  const int32_t*  cell_block_start; /* [C+1] first block of each cell (exclusive prefix; [C] = n_blocks) */
  const float*    pq_codebook_t;    /* [256, m_pad, d/M] transposed PQ codebook (zero rows for padding) */
  const float*    pq_norm_t;        /* [256, m_pad] squared norms of the sub-centroids (0 for cosine) */
  /* ---- residual IVFPQ (pq_use_residual=True, IVFPQIndex.py:48-55,160-170); NULL / 0 otherwise ---- */
  const float*    part2_scan;       /* [C, m_pad/64 groups, 256, 64]: -2 <c_cell,m , p_m,code> - |p_m,code|^2 in LUT layout */
  int32_t         residual;         /* 1 = codes are PQ codes of x - vq_centroid(cell) */
  /* ---- bytes of code per item in storage: 0 means n_subvectors.  IVFPQRIndex stores M + Mr (its re-rank code after
   *      the scanned one); the scan, relayout and search read only the first M/4 word planes.  Only tpq_store_codes
   *      reads this field: it writes code_size/4 planes and puts the first M/4 in the scan layout. ---- */
  int32_t         code_size;
} tpq_index;

/* ------------------------------------------------------------------ misc */
int         tpq_version(void);
const char* tpq_last_error(void);
/* 1 if the library was compiled for the device's architecture (sm_90a) */
int         tpq_device_supported(int device);

/* ------------------------------------------------------------------ query preparation
 * cosine pre-normalisation x / (||x||_2 + 1e-9) per column  (util.py:38-43, IVFPQIndex.py:474-475) */
int tpq_normalize_columns(const float* x_dn, int d, int nq, float* out_dn, void* stream);

/* ------------------------------------------------------------------ coarse probe
 * Replaces metric.negative_squared_l2_distance + fn.Topk + the smart-probing block
 * (metric.py:74-94, fn/Topk.py:43-67, IVFPQIndex.py:485-512).
 *   x_dn [d, nq] (already normalised for cosine), vq_codebook [d, C]
 *   -> probe_sims [nq, n_probe] f32 descending, cells [nq, n_probe] i64,
 *      n_probe_list [nq] i64 (ceil(H * n_probe) when smart != 0, else n_probe).
 * ws: at least tpq_coarse_workspace_bytes(d, nq, C) bytes. */
size_t tpq_coarse_workspace_bytes(int d, int nq, int n_cells);
int tpq_coarse_probe(const float* x_dn, const float* vq_codebook, int d, int nq, int n_cells,
                     int n_probe, int smart, float temperature,
                     float* probe_sims, int64_t* cells, int64_t* n_probe_list,
                     void* ws, size_t ws_bytes, void* stream);

/* ------------------------------------------------------------------ ADC look-up table
 * Replaces PQCodec.precompute_adc (codec/PQCodec.py:62-75; MultiKMeans.py:183-223).
 * -> lut [M, nq, 256] f32, the reference's `precomputed` layout. */
int tpq_build_lut(const float* x_dn, const float* pq_codebook, int d, int M, int nq, int metric,
                  float* lut_mqk, void* stream);

/* ------------------------------------------------------------------ fused list scan + top-k, reference layout
 * Exact drop-in for fn.IVFPQTopk.topk / IVFPQTopkCuda.topk (fn/IVFPQTopk.py:54-104,
 * kernels/IVFPQTopkCuda.py:81-142, kernels/cuda/ivfpq_topk.cu:822-971): same argument
 * list, reads the reference's own storage layout and `precomputed` LUT, accumulates in
 * the reference's order (fp32, m ascending from 0.f).
 *   data [M/4, n_data, 4] u8, precomputed [M, nq, 256] f32, is_empty [n_data] u8,
 *   cell_start/cell_size [nq, n_probe] i64 (already gathered), n_probe_list [nq] i64
 *   -> values [nq, k] f32 descending (-inf padded), address [nq, k] i64 (-1 padded). */
size_t tpq_ivfpq_topk_workspace_bytes(int nq, int k);
int tpq_ivfpq_topk(const uint8_t* data, const float* precomputed, const uint8_t* is_empty,
                   const int64_t* cell_start, const int64_t* cell_size, const int64_t* n_probe_list,
                   int64_t n_data, int M, int nq, int n_probe, int k,
                   float* values, int64_t* address, void* ws, size_t ws_bytes, void* stream);

/* ------------------------------------------------------------------ scan layout
 * tpq_relayout_plan: cell_block_start[c] = sum_{c'<c, owned} ceil(cell_extent[c']/32); [C] = total.  The caller passes
 * the cells' CAPACITIES (blocks exist for every slot a cell can hold, so that tpq_store_codes can add items in place;
 * the scan reads only the first ceil(cell_size/32) of them).  Cells not owned by (rank, world) get zero blocks. */
int tpq_relayout_plan(const int64_t* cell_extent, int n_cells, int shard_rank, int shard_world,
                      int32_t* cell_block_start /* [C+1] */, void* stream);
/* Bytes of codes_scan for n_blocks blocks of an M-subvector index. */
size_t tpq_codes_scan_bytes(int M, int64_t n_blocks);
/* Fill codes_scan / block_valid from the reference buffers (index->storage, is_empty,
 * cell_start, cell_size) for the blocks planned in cell_block_start. */
int tpq_relayout_codes(const tpq_index* index, uint8_t* codes_scan, uint32_t* block_valid, void* stream);
/* Residual IVFPQ: the per-cell half of the LUT (IVFPQIndex.precompute_part2, IVFPQIndex.py:160-170) in LUT layout. */
size_t tpq_part2_scan_bytes(int M, int n_cells);
int tpq_relayout_part2(const float* vq_codebook, const float* pq_codebook, int d, int M, int n_cells,
                       float* part2_scan, void* stream);
/* Transposed PQ codebook + norms used by the in-kernel LUT build. */
int tpq_relayout_codebook(const float* pq_codebook, int d, int M, int metric,
                          float* pq_codebook_t, float* pq_norm_t, void* stream);

/* ------------------------------------------------------------------ full search
 * IVFPQIndex.search (IVFPQIndex.py:469-524): x [d, nq] f32 -> values [nq,k] f32 (desc),
 * ids [nq,k] i64, address [nq,k] i64 (nullable).  Needs the scan layout in `index`.
 * keys_out (nullable, [nq,k] u64): packed (score,address) keys for the cross-shard merge. */
size_t tpq_search_workspace_bytes(const tpq_index* index, int nq, int n_probe, int k);
int tpq_ivfpq_search(const tpq_index* index, const float* x_dn, int nq, int n_probe, int k,
                     int smart, float temperature,
                     float* values, int64_t* ids, int64_t* address, uint64_t* keys_out,
                     void* ws, size_t ws_bytes, void* stream);

/* search over given probe lists (IVFPQIndex.search_cells non-residual branch, IVFPQIndex.py:407-467) */
int tpq_ivfpq_search_cells(const tpq_index* index, const float* x_dn, const int64_t* cells,
                           const float* base_sims /* [nq, n_probe], required when index->residual */,
                           const int64_t* n_probe_list, int nq, int n_probe, int k,
                           float* values, int64_t* ids, int64_t* address, uint64_t* keys_out,
                           void* ws, size_t ws_bytes, void* stream);

/* ------------------------------------------------------------------ flat (exact brute-force) search
 * FlatIndex.search (FlatIndex.py:46-101) over base [d, ld] f32 (row stride ld = the store's capacity), columns
 * [0, n) live, n < 2^32.  Scores, exact fp32 (one fmaf chain over i ascending per dot product):
 *   EUCLIDEAN ((2 x.b) - |x|^2) - |b|^2      COSINE (x / (|x| + 1e-8)).b / (|b| + 1e-8)      INNER x.b
 * tpq_flat_norms: the per-column table search reads, norms [n] f32 (|b|^2 squares separately rounded, or |b| + 1e-8;
 *   nothing for INNER, whose norms may be NULL).  Compute it once per store state.
 * tpq_flat_search: x_dn [d, nq] -> values [nq, k] f32 descending (-inf padded), ids [nq, k] i64
 *   (address2id[address], -1 padded), address [nq, k] i64 (nullable, -1 padded).  Order: score descending, then address
 *   ascending.  The [nq, n] score matrix is never stored: one fused GEMM + top-k kernel, then tpq_merge_topk.
 *   k > 1024 and metrics other than the three above: TPQ_ERR_UNSUPPORTED.  ws: at least
 *   tpq_flat_workspace_bytes(d, nq, n, k) bytes (bounded in n). */
int tpq_flat_norms(const float* base, int64_t ld, int d, int64_t n, int metric, float* norms, void* stream);
size_t tpq_flat_workspace_bytes(int d, int nq, int64_t n, int k);
int tpq_flat_search(const float* x_dn, int d, int nq, const float* base, int64_t ld, int64_t n,
                    const float* norms, int metric, int k, const int64_t* address2id,
                    float* values, int64_t* ids, int64_t* address, void* ws, size_t ws_bytes, void* stream);

/* ------------------------------------------------------------------ IVF search with exact fp32 distances (IVFFlatIndex)
 * The store is the IVFPQ cell container with fp32 columns: storage [d, capacity] f32 (tpq_store_codes with code_size =
 * 4 d bytes), is_empty [capacity], cell_start / cell_size [n_cells]; capacity < 2^32.  norms [capacity]: tpq_flat_norms
 * of every slot (|b|^2 for EUCLIDEAN, |b| + 1e-8 for COSINE), valid for the current store.
 * cells == NULL: the coarse probe of tpq_ivfpq_search runs inside (x normalised by tpq_normalize_columns for COSINE;
 *   n_probe <= n_cells, n_probe > 1024 TPQ_ERR_UNSUPPORTED); else cells [nq, n_probe] i64 and n_probe_list [nq] i64 as
 *   for tpq_ivfpq_search_cells (smart and temperature unused).
 * Visited: the first probe_count(n_probe_list[q], n_probe) = max(1, min((int)n_probe_list[q], n_probe)) entries, skipping
 *   cells outside [0, n_cells) and an entry whose cell_start equals the previous entry's; a visited cell's live slots of
 *   [cell_start, cell_start + cell_size) are scored.  Scores are tpq_flat_search's, bit for bit:
 *   EUCLIDEAN ((2 x.b) - |x|^2) - |b|^2      COSINE (x / (|x| + 1e-8)).b / (|b| + 1e-8)
 * -> values [nq, k] f32 descending (-inf padded), ids [nq, k] i64 (address2id[address], -1 padded), address [nq, k] i64
 *   (nullable, -1 padded).  Order: score descending, then address ascending; independent of the batch and its chunking.
 *   k > 1024 and metrics other than the two above: TPQ_ERR_UNSUPPORTED.  Arguments are checked before any launch;
 *   nq == 0 returns at once.  ws: at least tpq_ivfflat_workspace_bytes(d, nq, n_cells, n_probe, k) bytes, which stops
 *   growing with nq past one chunk of queries (the most whose n_probe * k keys fit 256 MB, at most 16 384). */
size_t tpq_ivfflat_workspace_bytes(int d, int nq, int n_cells, int n_probe, int k);
int tpq_ivfflat_search(const float* x_dn, int d, int nq, const float* vq_codebook, int n_cells,
                       const float* storage, int64_t capacity, const uint8_t* is_empty,
                       const int64_t* cell_start, const int64_t* cell_size, const float* norms, int metric,
                       const int64_t* cells, const int64_t* n_probe_list, int n_probe, int smart, float temperature,
                       int k, const int64_t* address2id, float* values, int64_t* ids, int64_t* address,
                       void* ws, size_t ws_bytes, void* stream);

/* ------------------------------------------------------------------ IVF search over 4-bit PQ codes (IVFPQ4Index)
 * The store is the IVFPQ cell container read in place (no scan layout): storage [M/8, capacity, 4] u8, 4-byte aligned,
 * code m of a slot in nibble m & 1 (low first) of byte m >> 1, so word g holds sub-quantizers 8g .. 8g+7; is_empty
 * [capacity], cell_start / cell_size [n_cells], address2id [capacity]; capacity < 2^32.  vq_codebook [d, n_cells],
 * pq_codebook [M, d/M, 16]; M a multiple of 8, at most 256 (TPQ_ERR_UNSUPPORTED beyond).
 * part2 (nullable; EUCLIDEAN only): residual IVFPQ, [n_cells, M, 16] f32, the cell half of each cell's LUT,
 *   (c_m . p * -2) - nrm * nrm (lut.cuh's part 2 entry).
 * cells == NULL: the coarse probe of tpq_ivfpq_search runs inside (x normalised by tpq_normalize_columns for COSINE;
 *   n_probe <= n_cells, n_probe > 1024 TPQ_ERR_UNSUPPORTED; residual base = the probe similarities); else cells
 *   [nq, n_probe] i64, n_probe_list [nq] i64 and, residual, base_sims [nq, n_probe] f32 as for tpq_ivfpq_search_cells
 *   (x used as given; smart and temperature unused).
 * Visited: tpq_ivfpq_search's rule, the first max(1, min((int)n_probe_list[q], n_probe)) entries (residual: max(0, ...)),
 *   skipping cells outside [0, n_cells) and an entry whose cell_start equals the previous entry's; a visited cell's live
 *   slots of [cell_start, cell_start + cell_size) are scored.  LUT [M][16] per query (lut.cuh's entries, from +0 fmaf
 *   chains over the d/M dimensions):  EUCLIDEAN ((2 dot) - |x_m|^2) - |p|^2   COSINE dot   residual: (2 dot) + part2[cell]
 *   (one fp32 add per entry).  Score = base + acc, acc = LUT[m][code_m] summed over m ascending from +0 in fp32, base =
 *   the cell's coarse similarity (residual) or +0.
 * -> values [nq, k] f32 descending (-inf padded), ids [nq, k] i64 (address2id[address], -1 padded), address [nq, k] i64
 *   (nullable, -1 padded).  Order: score descending, then address ascending; independent of the batch and its slicing.
 *   Arguments are checked before any launch; nq == 0 returns at once.  ws: at least
 *   tpq_ivfpq4_workspace_bytes(d, nq, n_cells, n_probe, k) bytes. */
size_t tpq_ivfpq4_workspace_bytes(int d, int nq, int n_cells, int n_probe, int k);
int tpq_ivfpq4_search(const float* x_dn, int d, int M, int nq, int metric, const uint8_t* storage,
                      const uint8_t* is_empty, const int64_t* cell_start, const int64_t* cell_size,
                      const int64_t* address2id, int64_t capacity, int n_cells, const float* vq_codebook,
                      const float* pq_codebook, const float* part2, const int64_t* cells,
                      const int64_t* n_probe_list, const float* base_sims, int n_probe, int smart,
                      float temperature, int k, float* values, int64_t* ids, int64_t* address, void* ws,
                      size_t ws_bytes, void* stream);

/* ------------------------------------------------------------------ scalar quantization (SQCodec, IVFSQIndex)
 * tpq_sq_encode: x_dn [d, n] f32 -> out [d, n]: u8 for bits 8, fp16 for bits 16, f32 (a copy) for bits 32.
 * tpq_sq_decode: codes [d, n] in the same types -> out_dn [d, n] f32.  lower / range [d] f32 (bits 8 only, NULL
 *   otherwise allowed): the codec's trained bounds, range = upper - lower + 1e-8.  Bit for bit the reference's torch ops:
 *   encode 8  clamp(rint(((x - lower) / range) * 256), 0, 255)    (each op rounded, rint half to even; NaN -> 0)
 *   decode 8  ((code / 256) * range) + lower                       (two roundings, no fma)
 *   16 bits   __float2half_rn / __half2float (beyond +-65504: +-inf)
 *   bits other than 8, 16, 32: TPQ_ERR_UNSUPPORTED.  n == 0 returns at once.  Inputs are never written.
 * tpq_ivfsq_search: tpq_ivfflat_search over an SQ-coded store, scored on the decoded vectors: storage is
 *   [code_size / 4, capacity, 4] u8 as tpq_index.storage (word planes, row stride capacity words) with code_size = d
 *   (bits 8, d % 4 == 0) or 2 d (bits 16, d % 2 == 0); byte j of an item is the code of dimension j (bits 8), bytes
 *   2 j, 2 j + 1 the fp16 code of dimension j (bits 16).  lower / range: as above, 16-byte aligned, read for bits 8.
 *   norms: tpq_flat_norms of the decoded store.  Values, ids and addresses are tpq_ivfflat_search's on the decoded
 *   store [d, capacity] f32, bit for bit; the workspace is tpq_ivfflat_workspace_bytes's.  bits other than 8 and 16:
 *   TPQ_ERR_UNSUPPORTED; every other argument is checked as by tpq_ivfflat_search, before any launch. */
int tpq_sq_encode(const float* x_dn, int d, int64_t n, int bits, const float* lower, const float* range, void* out,
                  void* stream);
int tpq_sq_decode(const void* codes, int d, int64_t n, int bits, const float* lower, const float* range, float* out_dn,
                  void* stream);
int tpq_ivfsq_search(const float* x_dn, int d, int nq, const float* vq_codebook, int n_cells,
                     const uint8_t* storage, int bits, const float* lower, const float* range, int64_t capacity,
                     const uint8_t* is_empty, const int64_t* cell_start, const int64_t* cell_size, const float* norms,
                     int metric, const int64_t* cells, const int64_t* n_probe_list, int n_probe, int smart,
                     float temperature, int k, const int64_t* address2id, float* values, int64_t* ids,
                     int64_t* address, void* ws, size_t ws_bytes, void* stream);

/* ------------------------------------------------------------------ range search (FlatIndex, IVFFlatIndex, IVFSQIndex, IVFPQIndex)
 * Every scored item whose score is above the threshold: the same items and scores as the searches above (tpq_flat_search's
 * columns [0, n); the IVF searches' live slots of the visited cells), matched when score > threshold, strictly, in fp32
 * (a NaN score never matches; +-inf thresholds are allowed, a NaN threshold is TPQ_ERR_BAD_ARG).
 * -> match_keys [cap] u64 and match_query [cap] i32, unordered: one entry per match, match_query its query and match_keys
 *   (order-preserving image of the fp32 score << 32) | (0xFFFFFFFF - address), the key every top-k here sorts by (key
 *   descending = score descending, then address ascending; the image of f is bits(f) | 2^31 for f >= +0 and ~bits(f)
 *   below).  *total (one u64 on the device) receives the exact count of matches; at most cap are written, the first
 *   cap in no defined order, and nothing past cap.  A caller whose *total exceeds cap runs the call again with
 *   cap >= *total; the result does not depend on the plan, the chunking or the batch.  cap == 0 counts only, and the
 *   match arrays may then be NULL.  Arguments are checked before any launch; nq == 0 returns at once without writing
 *   *total; n == 0 (capacity == 0) sets *total = 0.
 * tpq_flat_range_search: over tpq_flat_search's store, metrics EUCLIDEAN, COSINE, INNER.  ws: at least
 *   tpq_flat_range_workspace_bytes(d, nq, n) bytes.
 * tpq_ivfflat_range_search / tpq_ivfsq_range_search: over tpq_ivfflat_search's / tpq_ivfsq_search's store, probe and
 *   visiting rule, metrics EUCLIDEAN and COSINE.  A cell is visited at most once per query when cells == NULL (the
 *   coarse probe returns distinct cells).  ws: at least tpq_ivfflat_range_workspace_bytes(d, nq, n_cells, n_probe)
 *   bytes, which stops growing with nq past one chunk of queries (the most whose gathered pair queries, n_probe * d
 *   floats each, fit 256 MB, at most 16 384).
 * tpq_ivfpq_range_search: over the IVFPQ scan of tpq_ivfpq_search (cells == NULL: its coarse stage runs inside, with
 *   cosine normalisation and smart probing, and a cell is visited at most once per query) or of tpq_ivfpq_search_cells
 *   (cells / n_probe_list given, smart and temperature unused; base_sims [nq, n_probe] required for a residual index).
 *   The scored items and their scores are those searches', bit for bit: the live slots of the visited cells, ADC sums in
 *   the scan's order (plus the cell's coarse similarity for a residual index).  On a cell shard (shard_world > 1) only
 *   the shard's cells are scanned, with global addresses.  Metrics EUCLIDEAN and COSINE (residual: EUCLIDEAN); an index
 *   without blocks (n_blocks == 0) sets *total = 0.  ws: at least tpq_ivfpq_range_workspace_bytes(index, nq, n_probe)
 *   bytes. */
size_t tpq_flat_range_workspace_bytes(int d, int nq, int64_t n);
int tpq_flat_range_search(const float* x_dn, int d, int nq, const float* base, int64_t ld, int64_t n,
                          const float* norms, int metric, float threshold, uint64_t* match_keys, int32_t* match_query,
                          int64_t cap, uint64_t* total, void* ws, size_t ws_bytes, void* stream);
size_t tpq_ivfflat_range_workspace_bytes(int d, int nq, int n_cells, int n_probe);
int tpq_ivfflat_range_search(const float* x_dn, int d, int nq, const float* vq_codebook, int n_cells,
                             const float* storage, int64_t capacity, const uint8_t* is_empty,
                             const int64_t* cell_start, const int64_t* cell_size, const float* norms, int metric,
                             const int64_t* cells, const int64_t* n_probe_list, int n_probe, int smart,
                             float temperature, float threshold, uint64_t* match_keys, int32_t* match_query,
                             int64_t cap, uint64_t* total, void* ws, size_t ws_bytes, void* stream);
int tpq_ivfsq_range_search(const float* x_dn, int d, int nq, const float* vq_codebook, int n_cells,
                           const uint8_t* storage, int bits, const float* lower, const float* range, int64_t capacity,
                           const uint8_t* is_empty, const int64_t* cell_start, const int64_t* cell_size,
                           const float* norms, int metric, const int64_t* cells, const int64_t* n_probe_list,
                           int n_probe, int smart, float temperature, float threshold, uint64_t* match_keys,
                           int32_t* match_query, int64_t cap, uint64_t* total, void* ws, size_t ws_bytes,
                           void* stream);
size_t tpq_ivfpq_range_workspace_bytes(const tpq_index* index, int nq, int n_probe);
int tpq_ivfpq_range_search(const tpq_index* index, const float* x_dn, const int64_t* cells, const float* base_sims,
                           const int64_t* n_probe_list, int nq, int n_probe, int smart, float temperature,
                           float threshold, uint64_t* match_keys, int32_t* match_query, int64_t cap,
                           uint64_t* total, void* ws, size_t ws_bytes, void* stream);

/* ------------------------------------------------------------------ row-wise top-k (fn.Topk, fn/Topk.py:43-67)
 * x [m, n] row-major, contiguous, fp32 or fp16 (dtype TPQ_DTYPE_*) -> the k best entries of every row: values [m, k]
 * f32 (an fp16 value widened exactly), indices [m, k] i64 (the column).  Order: value descending, then column
 * ascending; +0 ranks above -0 and every NaN, of either sign, above +inf (returned as a NaN, payload not kept).  A row
 * with fewer than k entries is padded with (-inf, -1).  1 <= k <= 1024 and n < 2^32 (TPQ_ERR_UNSUPPORTED beyond);
 * m == 0 returns at once; x may be NULL when n == 0.  ws: at least tpq_topk_workspace_bytes(m, n, k, dtype) bytes (0 bytes, ws may be NULL, when
 * every row is selected by one CTA or one warp); TPQ_ERR_WORKSPACE when it is smaller. */
enum { TPQ_DTYPE_F32 = 0, TPQ_DTYPE_F16 = 1 };
size_t tpq_topk_workspace_bytes(int64_t m, int64_t n, int k, int dtype);
int tpq_topk(const void* x, int64_t m, int64_t n, int dtype, int k,
             float* values, int64_t* indices, void* ws, size_t ws_bytes, void* stream);

/* ------------------------------------------------------------------ re-rank (IVFPQRIndex.search, second pass)
 * candidates [nq, k1] i64: the first pass's addresses (-1 = none), k <= k1 <= 1024.  storage [(M + Mr)/4, capacity, 4]
 * u8 as tpq_index.storage with code_size = M + Mr: bytes 0..M-1 of an item are its first-level code, M..M+Mr-1 its
 * re-rank code.  pq_codebook [M, d/M, 256] (read only when use_residual; may be NULL otherwise), pq_rerank_codebook
 * [Mr, d/Mr, 256].  Per candidate, exactly in fp32:
 *   y_e = y2_e + y1_e (use_residual) or y2_e, y1 / y2 the first-level / re-rank codebook entries of its codes;
 *   EUCLIDEAN acc = fmaf(-dif, dif, acc), dif = x_e - y_e, e ascending from +0 (tpq_max_sim's arithmetic);
 *   COSINE    acc = fmaf(x_e, y_e, acc) on x / (||x|| + 1e-9) (as tpq_normalize_columns), y not normalised;
 * i.e. the value equals tpq_max_sim(x_q, decoded candidate).  -> values [nq, k] f32 descending (-inf padded), ids
 * [nq, k] i64 (address2id[address], -1 padded), address [nq, k] i64 (nullable, -1 padded); order score descending,
 * then address ascending.  Arguments are checked before any launch; nq == 0 returns at once.  ws: at least
 * tpq_rerank_workspace_bytes(d, nq, k) bytes. */
size_t tpq_rerank_workspace_bytes(int d, int nq, int k);
int tpq_rerank(const float* x_dn, int d, int nq, const int64_t* candidates, int k1,
               const uint8_t* storage, int64_t capacity, int M, int Mr,
               const float* pq_codebook, const float* pq_rerank_codebook, int use_residual, int metric,
               int k, const int64_t* address2id, float* values, int64_t* ids, int64_t* address,
               void* ws, size_t ws_bytes, void* stream);

/* ------------------------------------------------------------------ exact refine (RefineFlatIndex.search, second pass)
 * candidates [nq, k1] i64: addresses into vectors (-1 = none; any address outside [0, n) is dropped too), k <= k1 <=
 * 1024; a candidate listed twice is scored twice.  vectors [n, d] f32 row-major, n < 2^32.  Per candidate y, exactly in
 * fp32:
 *   EUCLIDEAN acc = fmaf(-dif, dif, acc), dif = x_e - y_e, e ascending from +0, exactly d terms (tpq_max_sim's arithmetic);
 *   COSINE    acc = fmaf(x_e, y_e, acc) on x / (||x|| + 1e-9) (as tpq_normalize_columns), y as stored (the caller
 *             stores normalised vectors);
 * i.e. the value equals tpq_max_sim(x_q, y), the arithmetic of tpq_rerank.  -> values [nq, k] f32 descending (-inf
 * padded), ids [nq, k] i64 (address2id[address], -1 padded), address [nq, k] i64 (nullable, -1 padded); order score
 * descending, then address ascending.  Arguments are checked before any launch (k and k1, metric, sizes, workspace,
 * pointers; vectors may be NULL when n == 0); nq == 0 returns at once.  ws: at least
 * tpq_refine_flat_workspace_bytes(d, nq, k) bytes. */
size_t tpq_refine_flat_workspace_bytes(int d, int nq, int k);
int tpq_refine_flat(const float* x_dn, int d, int nq, const int64_t* candidates, int k1,
                    const float* vectors, int64_t n, int metric, int k, const int64_t* address2id,
                    float* values, int64_t* ids, int64_t* address, void* ws, size_t ws_bytes, void* stream);

/* ------------------------------------------------------------------ k-means / codec neighbours of the path
 * tpq_max_sim: MultiKMeans assignment, MaxSimCuda(dim=2, mode "tn") (kernels/MaxSimCuda.py:184-238,
 *   kernels/cuda/max_sim.cu:182-309; caller clustering/MultiKMeans.py:314-333):
 *   data [l, d, n], centroids [l, d, k] -> maxsims [l, n] f32, labels [l, n] i64.
 *   metric EUCLIDEAN: sum_e -(x-c)^2 (direct form, max_sim.cu:78-98); COSINE: sum_e x*c ("inner");
 *   MANHATTAN: sum_e -|x-c| (max_sim.cu:100-120, exact kernel only).
 *   Ties: lowest centroid index (the reference's cross-tile label write is racy, max_sim.cu:173-178).
 * tpq_compute_centroids: ComputeCentroidsCuda (kernels/ComputeCentroidsCuda.py:43-81, kernels/cuda/compute_centroids.cu:9-86):
 *   data [l, d, n], labels [l, n] i64 -> centroids [l, d, k] = member mean, 0 for an empty cluster; every member sum is
 *   taken in point order (bit-reproducible).  The workspace size is 0 (ws may be NULL).
 * tpq_pq_decode: PQDecodeCuda (kernels/PQDecodeCuda.py:38-65, kernels/cuda/pq_decode.cu:7-53):
 *   codebook [M, dsub, 256], code [M, n] u8 -> out [M*dsub, n] f32. */
/* exact == 1: fp32 SIMT kernel, the reference's arithmetic bit for bit.  exact == 0 or 2: TF32 wgmma kernel where
 * the shape allows (euclidean, d % 8 == 0, d <= 64, k <= 256, n % 4 == 0), else the exact kernel: labels may differ
 * from the exact ones only between centroids closer than TF32 rounding.  maxsims: exact == 2 -> recomputed exactly
 * in fp32 for the chosen centroid; exact == 0 -> 2*score - |x|^2 from the TF32 score (~1e-3 relative). */
int tpq_max_sim(const float* data, const float* centroids, int l, int d, int64_t n, int k, int metric,
                int exact, float* maxsims, int64_t* labels, void* stream);
/* tpq_kmeans_assign: the assignment step of KMeans / MultiKMeans (clustering/KMeans.py, MultiKMeans.py) for every k and
 *   d: data [l, d, n], centroids [l, d, k] -> maxsims [l, n] f32, labels [l, n] i64, metric as tpq_max_sim (MANHATTAN
 *   included).  Dispatch, first match:
 *     - euclidean, d % 8 == 0, d <= 64, 8 <= k <= 256, k % 4 == 0, n % 4 == 0, n >= 128, 16-byte-aligned data and
 *       centroids: the TF32 wgmma kernel of tpq_max_sim (all centroids resident in shared memory);
 *     - euclidean or cosine, d % 8 == 0, 8 <= d <= 256, 8 <= k <= 2^20, n % 4 == 0, 16-byte-aligned data and
 *       centroids: the TF32 wgmma kernel that streams the centroids (needs the workspace);
 *     - otherwise (manhattan included) the exact fp32 kernel of tpq_max_sim(exact == 1), bit for bit.
 *   On the TF32 kernels labels may differ from the exact ones only between centroids closer than TF32 rounding; ties of
 *   the TF32 score go to the lowest index.  Cosine scores are inner products: normalise data and centroids first.
 *   maxsims: exact_values != 0 -> recomputed exactly in fp32 for the chosen centroid, in the exact kernel's order
 *   (bit-identical to it wherever the labels agree; like tpq_max_sim's exact == 2); exact_values == 0 -> derived from
 *   the TF32 score, 2*score - |x|^2 (euclidean) or score (cosine), ~1e-3 relative (like exact == 0).  The exact kernel
 *   always writes exact values.
 *   ws: at least tpq_kmeans_assign_workspace_bytes(l, d, k) bytes, 16-byte aligned (0 bytes, ws may be NULL, when
 *   d or k is outside the streaming kernel's range); TPQ_ERR_WORKSPACE when the streaming kernel needs more. */
size_t tpq_kmeans_assign_workspace_bytes(int l, int d, int k);
int tpq_kmeans_assign(const float* data, const float* centroids, int l, int d, int64_t n, int k, int metric,
                      int exact_values, float* maxsims, int64_t* labels, void* ws, size_t ws_bytes, void* stream);
size_t tpq_compute_centroids_workspace_bytes(int l, int k);
int tpq_compute_centroids(const float* data, const int64_t* labels, int l, int d, int64_t n, int k,
                          float* centroids, void* ws, size_t ws_bytes, void* stream);
int tpq_pq_decode(const float* codebook, const uint8_t* code, int M, int dsub, int64_t n, float* out, void* stream);

/* ------------------------------------------------------------------ build side: placement of new items
 * IVFPQIndex.add -> CellContainer.add (container/CellContainer.py:313-367).
 * tpq_get_ioa: index of appearance of every label among equal labels, input order (kernels/cuda/get_ioa.cu:8-47);
 *   counts [n_cells] (nullable) = items per cell (what `cells.unique(return_counts=True)` feeds `_cell_size[...] +=`).
 * tpq_empty_prefix: prefix[a] = empty slots in [0, a), a = 0..capacity (only needed when the container has holes).
 * tpq_get_write_address: the ioa-th empty slot of the item's cell (kernels/cuda/get_write_address_v2.cu:9-41);
 *   empty_prefix == NULL asserts "no holes": the empties of a cell are [start + size, start + capacity).  -1 = no room.
 * tpq_store_codes: set_data_by_address (CellContainer.py:213-239) + address2id / is_empty / cell_size updates
 *   (:354-360; cell_size becomes max(old, slot + 1)).  codes [code_size, n] u8 (index->code_size, 0 = n_subvectors;
 *   else a multiple of 4 >= n_subvectors, checked before the launch).  If codes_scan / block_valid (the scan layout of
 *   `index`, non-const here) are given they are updated in place with the first n_subvectors code bytes, so the layout
 *   stays valid after the add.
 * tpq_expand_move's M is the number of code bytes per item (code_size), i.e. storage holds M/4 word planes.
 * tpq_expand_move: CellContainer.expand (:249-311) for many cells at once: every old slot a moves to a + shift[cell(a)];
 *   the caller pre-fills the new buffers (storage 0, address2id -1, is_empty 1) and updates the per-cell tables. */
size_t tpq_ioa_workspace_bytes(int64_t n, int n_cells);
int tpq_get_ioa(const int64_t* cells, int64_t n, int n_cells, int64_t* ioa, int64_t* counts,
                void* ws, size_t ws_bytes, void* stream);
size_t tpq_empty_prefix_workspace_bytes(int64_t capacity);
int tpq_empty_prefix(const uint8_t* is_empty, int64_t capacity, uint32_t* prefix /* [capacity + 1] */,
                     void* ws, size_t ws_bytes, void* stream);
int tpq_get_write_address(const int64_t* cells, const int64_t* ioa, int64_t n,
                          const int64_t* cell_start, const int64_t* cell_size, const int64_t* cell_capacity,
                          int n_cells, const uint32_t* empty_prefix, int64_t* write_adr, void* stream);
int tpq_store_codes(const uint8_t* codes, const int64_t* cells, const int64_t* write_adr, const int64_t* ids,
                    int64_t n, tpq_index* index, uint8_t* storage, int64_t* address2id, uint8_t* is_empty,
                    int64_t* cell_size, uint8_t* codes_scan, uint32_t* block_valid, void* stream);
int tpq_expand_move(const uint8_t* old_storage, const int64_t* old_address2id, const uint8_t* old_is_empty,
                    const int64_t* old_cell_start, const int64_t* shift, int n_cells, int M,
                    int64_t old_capacity, int64_t new_capacity,
                    uint8_t* storage, int64_t* address2id, uint8_t* is_empty, void* stream);

/* ------------------------------------------------------------------ measurement hook (bench.py roofline leg)
 * When enabled, every scan-kernel launch is bracketed by CUDA events on its own stream;
 * tpq_profile_scan_ms waits for them and returns the summed duration and launch count since
 * the last call.  Process-wide, not thread-safe; leave disabled in production. */
int tpq_profile_enable(int on);
int tpq_profile_scan_ms(float* total_ms, int* n_launches);

/* ------------------------------------------------------------------ fused scan + exchange (multi-GPU)
 * The scan of tpq_ivfpq_search(_cells) with its output fused into the cross-shard exchange: every CTA stores its sorted
 * top-k keys straight into slot `my_slot` of each rank's gather buffer peer_keys[p] ([n_slots, nq, k] u64 in peer-mapped
 * memory, e.g. torch symmetric memory) over NVLink, instead of a local buffer that a collective would copy afterwards.
 * The caller then synchronises the ranks (symmetric-memory barrier) and runs tpq_merge_topk on its own buffer.
 * cells == NULL: the coarse probe runs inside (x as given to search); else x / cells / base_sims / n_probe_list as for
 * tpq_ivfpq_search_cells.  TPQ_ERR_UNSUPPORTED when the batch is small enough to be sliced (use the gathered path). */
int tpq_ivfpq_scan_push(const tpq_index* index, const float* x_dn, const int64_t* cells, const float* base_sims,
                        const int64_t* n_probe_list, int nq, int n_probe, int k, int smart, float temperature,
                        uint64_t* const* peer_keys, int n_peers, int my_slot,
                        void* ws, size_t ws_bytes, void* stream);

/* ------------------------------------------------------------------ cross-shard merge
 * keys_in [n_parts, nq, k] (the all-gather's layout; each part sorted descending, 0 = empty slot) -> top-k per query,
 * decoded: values (-inf pad), address (-1 pad), ids = address2id[address] (BaseContainer.py:58-65). */
int tpq_merge_topk(const uint64_t* keys_in, int nq, int n_parts, int k,
                   const int64_t* address2id, int64_t capacity,
                   float* values, int64_t* ids, int64_t* address, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TPQ_B200_H */
