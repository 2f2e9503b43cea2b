// Build side of the container: where do new items go, and put them there -- in BOTH layouts.
//
// Replaces, for IVFPQIndex.add -> CellContainer.add (torchpq/container/CellContainer.py:313-367):
//   get_ioa            kernels/cuda/get_ioa.cu:8-47            index of appearance of every label among equal labels
//   get_write_address  kernels/cuda/get_write_address_v2.cu:9-41   the ioa-th empty slot of the item's cell
//   set_data_by_address + bookkeeping   CellContainer.py:213-239, 354-360
//   expand             CellContainer.py:249-311
// The reference's get_ioa is O(n * n_unique / 256) (every CTA walks the whole label array) and its write-address kernel
// walks the cell slot by slot per ITEM; here: a chunked stable counting sort (one shared-memory bitonic sort per 4096
// labels + a per-cell scan over chunks), a binary search in a prefix sum of `is_empty` (only when the container has
// holes), and one scatter kernel that writes the reference layout AND the scan layout (so `add` does not invalidate it).
#include "scan_layout.cuh"

namespace tpq {

constexpr int PL_CH = 4096;          // labels per chunk (one CTA)

// ----------------------------------------------------------------------------- index of appearance
// Per chunk: sort (label << 32 | position) in shared memory; the rank of an item among equal labels of its chunk is its
// sorted position minus the first position of its label (stable: ties are ordered by position).  Run lengths go to
// hist[chunk][label] (dense, zeroed by the caller), local ranks to lrank[i].
__global__ void __launch_bounds__(512)
ioa_local_kernel(const int64_t* __restrict__ cells, int64_t n, int n_cells, uint16_t* __restrict__ lrank,
                 int32_t* __restrict__ hist) {
  __shared__ uint64_t key[PL_CH];
  const int64_t base = (int64_t)blockIdx.x * PL_CH;
  const int np = (int)min((int64_t)PL_CH, n - base);
  for (int i = threadIdx.x; i < PL_CH; i += blockDim.x) {
    uint64_t kk = ~0ull;                                              // padding sorts last
    if (i < np) {
      const int64_t c = cells[base + i];
      if (c >= 0 && c < n_cells) kk = ((uint64_t)c << 32) | (uint32_t)i;   // out-of-range labels are left out (ioa 0, not counted)
    }
    key[i] = kk;
  }
  __syncthreads();
  for (int k = 2; k <= PL_CH; k <<= 1) {                              // ascending bitonic sort
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int t = threadIdx.x; t < PL_CH / 2; t += blockDim.x) {
        const int lo = ((t & ~(j - 1)) << 1) | (t & (j - 1)), hi = lo + j;
        const bool asc = (lo & k) == 0;
        const uint64_t x = key[lo], y = key[hi];
        if ((x > y) == asc) { key[lo] = y; key[hi] = x; }
      }
      __syncthreads();
    }
  }
  for (int i = threadIdx.x; i < np; i += blockDim.x) {
    const uint64_t kk = key[i];
    if (kk == ~0ull) continue;
    const uint32_t lab = (uint32_t)(kk >> 32);
    int lo = 0, hi = i;                                               // first position whose label is `lab`
    while (lo < hi) { const int mid = (lo + hi) >> 1; if ((uint32_t)(key[mid] >> 32) < lab) lo = mid + 1; else hi = mid; }
    lrank[base + (uint32_t)kk] = (uint16_t)(i - lo);
    if (i == lo) {                                                    // run start: its length is this chunk's count of `lab`
      int a = i, b = np;
      while (a < b) { const int mid = (a + b) >> 1; if ((uint32_t)(key[mid] >> 32) <= lab) a = mid + 1; else b = mid; }
      hist[(size_t)blockIdx.x * n_cells + lab] = a - i;
    }
  }
}

// hist[chunk][c] <- number of items of cell c in chunks before `chunk` (exclusive scan down the chunks); counts[c] = total.
__global__ void ioa_scan_kernel(int32_t* __restrict__ hist, int n_chunks, int n_cells, int64_t* __restrict__ counts) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_cells) return;
  int run = 0;
  for (int ch = 0; ch < n_chunks; ++ch) {
    const size_t o = (size_t)ch * n_cells + c;
    const int v = hist[o];
    hist[o] = run;
    run += v;
  }
  if (counts) counts[c] = run;
}

__global__ void ioa_finish_kernel(const int64_t* __restrict__ cells, const uint16_t* __restrict__ lrank,
                                  const int32_t* __restrict__ hist, int64_t n, int n_cells, int64_t* __restrict__ ioa) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int64_t c = cells[i];
  if (c < 0 || c >= n_cells) { ioa[i] = 0; return; }
  ioa[i] = (int64_t)hist[(size_t)(i / PL_CH) * n_cells + c] + lrank[i];
}

// ----------------------------------------------------------------------------- empties before every slot
// prefix[a] = number of empty slots in [0, a); prefix[capacity] = total.  Three passes over 1 B per slot.
constexpr int EP_T = 256, EP_PER = 16, EP_TILE = EP_T * EP_PER;
__global__ void __launch_bounds__(EP_T)
empty_tile_sums_kernel(const uint8_t* __restrict__ is_empty, int64_t cap, uint32_t* __restrict__ tile_sums) {
  __shared__ uint32_t ws[EP_T / 32];
  const int64_t base = (int64_t)blockIdx.x * EP_TILE;
  uint32_t s = 0;
  for (int u = 0; u < EP_PER; ++u) {
    const int64_t a = base + (int64_t)u * EP_T + threadIdx.x;
    if (a < cap) s += is_empty[a] != 0;
  }
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) { uint32_t t = 0; for (int w = 0; w < EP_T / 32; ++w) t += ws[w]; tile_sums[blockIdx.x] = t; }
}
__global__ void __launch_bounds__(1024)
scan_u32_inplace_kernel(uint32_t* __restrict__ v, int n) {               // exclusive scan, one CTA
  __shared__ uint32_t wsum[32];
  __shared__ uint32_t carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int i0 = 0; i0 < n; i0 += 1024) {
    const int i = i0 + threadIdx.x;
    const uint32_t x = i < n ? v[i] : 0u;
    const uint32_t incl = cta_inclusive_scan(x, wsum, carry);
    if (i < n) v[i] = incl - x;
  }
}
__global__ void __launch_bounds__(EP_T)
empty_prefix_kernel(const uint8_t* __restrict__ is_empty, int64_t cap, const uint32_t* __restrict__ tile_base,
                    uint32_t* __restrict__ prefix) {
  __shared__ uint32_t wsum[EP_T / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t a0 = (int64_t)blockIdx.x * EP_TILE + (int64_t)threadIdx.x * EP_PER;   // EP_PER consecutive slots per thread
  uint32_t f[EP_PER], s = 0;
  #pragma unroll
  for (int u = 0; u < EP_PER; ++u) { f[u] = (a0 + u < cap) ? (is_empty[a0 + u] != 0) : 0u; s += f[u]; }
  const uint32_t incl = warp_inclusive_scan(s, lane);
  if (lane == 31) wsum[warp] = incl;
  __syncthreads();
  uint32_t before = tile_base[blockIdx.x] + incl - s;
  for (int w = 0; w < warp; ++w) before += wsum[w];
  #pragma unroll
  for (int u = 0; u < EP_PER; ++u) { if (a0 + u <= cap) prefix[a0 + u] = before; before += f[u]; }
}

// ----------------------------------------------------------------------------- write addresses
// The ioa-th empty slot at or after cell_start[c] (get_write_address_v2.cu:9-41; its `divSize` is the cell's capacity).
// No holes (prefix == nullptr): the empties of a cell are exactly [start + size, start + capacity).
__global__ void write_address_kernel(const int64_t* __restrict__ cells, const int64_t* __restrict__ ioa, int64_t n,
                                     const int64_t* __restrict__ cell_start, const int64_t* __restrict__ cell_size,
                                     const int64_t* __restrict__ cell_capacity, int n_cells,
                                     const uint32_t* __restrict__ prefix, int64_t* __restrict__ write_adr) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int64_t c = cells[i];
  if (c < 0 || c >= n_cells) { write_adr[i] = -1; return; }
  const int64_t s = cell_start[c], r = ioa[i];
  if (!prefix) { write_adr[i] = (cell_size[c] + r < cell_capacity[c]) ? s + cell_size[c] + r : -1; return; }
  const uint32_t want = prefix[s] + (uint32_t)r;                       // global rank of the empty slot we are after
  int64_t lo = s, hi = s + cell_capacity[c];                            // smallest a in [lo, hi) with prefix[a + 1] > want
  if (prefix[hi] <= want) { write_adr[i] = -1; return; }               // the cell has fewer than r + 1 empty slots
  while (lo < hi) { const int64_t mid = (lo + hi) >> 1; if (prefix[mid + 1] > want) hi = mid; else lo = mid + 1; }
  write_adr[i] = lo;
}

// ----------------------------------------------------------------------------- store
// One thread per (item, 4-code word): storage[g][adr] = codes[4g..4g+3][i] (CellContainer.py:213-239); word 0's thread
// also does the bookkeeping of CellContainer.add's tail (:354-360).  _cell_size is kept as the cell's high-water mark
// (atomicMax of slot + 1): without holes that IS old size + count.  If a scan layout is given it receives the same codes,
// lane-rotated (scan_layout.cuh), and the block's valid bit.  A code wider than the scanned one (code_size > M, the
// re-rank code of IVFPQRIndex) has more word planes; only the first M/4 are scanned and reach the scan layout.
__global__ void store_codes_kernel(const uint8_t* __restrict__ codes, const int64_t* __restrict__ cells,
                                   const int64_t* __restrict__ write_adr, const int64_t* __restrict__ ids, int64_t n, int M,
                                   int64_t cap, uint32_t* __restrict__ storage, int64_t* __restrict__ address2id,
                                   uint8_t* __restrict__ is_empty, long long* __restrict__ cell_size,
                                   const int64_t* __restrict__ cell_start,
                                   uint8_t* __restrict__ codes_scan, uint32_t* __restrict__ block_valid,
                                   const int32_t* __restrict__ cell_block_start, int MP, int shard_rank, int shard_world) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int g = blockIdx.y;
  if (i >= n) return;
  const int64_t a = write_adr[i];
  if (a < 0 || a >= cap) return;
  uint32_t w = 0;
  #pragma unroll
  for (int b = 0; b < 4; ++b) w |= (uint32_t)codes[(size_t)(4 * g + b) * n + i] << (8 * b);
  storage[(size_t)g * cap + a] = w;
  const int64_t c = cells[i];
  const int64_t pos = a - cell_start[c];
  if (g == 0) {
    address2id[a] = ids[i];
    is_empty[a] = 0;
    atomicMax(cell_size + c, (long long)(pos + 1));
  }
  if (codes_scan && g < M / 4 && shard_owns(c, shard_rank, shard_world)) {
    const int64_t B = (int64_t)cell_block_start[c] + (pos >> 5);
    const int lane = (int)(pos & 31);
    #pragma unroll
    for (int b = 0; b < 4; ++b) {
      const int t = rot_byte(4 * g + b, lane);
      codes_scan[scan_chunk_offset(B, MP, t >> 4, lane) + (t & 15)] = (uint8_t)(w >> (8 * b));
    }
    if (g == 0) atomicOr(block_valid + B, 1u << lane);
  }
}

// ----------------------------------------------------------------------------- expand
// CellContainer.expand (CellContainer.py:249-311) for any set of cells in one pass: new_start[c] = old_start[c] + the
// growth of all earlier cells; every old slot moves to old address + shift of its cell.  New buffers are pre-filled by the
// caller (storage 0, address2id -1, is_empty 1).
__global__ void expand_move_kernel(const uint32_t* __restrict__ old_storage, const int64_t* __restrict__ old_a2i,
                                   const uint8_t* __restrict__ old_empty, const int64_t* __restrict__ old_start,
                                   const int64_t* __restrict__ shift, int n_cells, int64_t old_cap, int64_t new_cap, int planes,
                                   uint32_t* __restrict__ storage, int64_t* __restrict__ a2i, uint8_t* __restrict__ empty) {
  const int64_t a = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= old_cap) return;
  int lo = 0, hi = n_cells;                                            // last cell with old_start <= a
  while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (old_start[mid] <= a) lo = mid; else hi = mid; }
  const int64_t b = a + shift[lo];
  if (b < 0 || b >= new_cap) return;
  a2i[b] = old_a2i[a];
  empty[b] = old_empty[a];
  for (int g = 0; g < planes; ++g) storage[(size_t)g * new_cap + b] = old_storage[(size_t)g * old_cap + a];
}

}  // namespace tpq

using namespace tpq;

static inline int64_t n_chunks_of(int64_t n) { return (n + PL_CH - 1) / PL_CH; }

extern "C" size_t tpq_ioa_workspace_bytes(int64_t n, int n_cells) {
  if (n <= 0 || n_cells <= 0) return 0;
  return align_up((size_t)n_chunks_of(n) * n_cells * 4, 256) + align_up((size_t)n * 2, 256);
}

extern "C" int tpq_get_ioa(const int64_t* cells, int64_t n, int n_cells, int64_t* ioa, int64_t* counts,
                           void* ws, size_t ws_bytes, void* stream) {
  TPQ_REQUIRE(n >= 0 && n_cells > 0, "tpq_get_ioa: bad sizes");
  cudaStream_t st = (cudaStream_t)stream;
  if (n == 0) { if (counts) TPQ_CUDA(cudaMemsetAsync(counts, 0, (size_t)n_cells * 8, st)); return TPQ_OK; }
  TPQ_REQUIRE(cells && ioa, "tpq_get_ioa: null pointer");
  if (!ws || ws_bytes < tpq_ioa_workspace_bytes(n, n_cells)) { set_error("tpq_get_ioa: workspace too small"); return TPQ_ERR_WORKSPACE; }
  const int64_t nch = n_chunks_of(n);
  TPQ_REQUIRE(nch <= 0x7fffffff, "tpq_get_ioa: too many items for one call");
  uint8_t* w = reinterpret_cast<uint8_t*>(ws);
  int32_t* hist = reinterpret_cast<int32_t*>(w);            w += align_up((size_t)nch * n_cells * 4, 256);
  uint16_t* lrank = reinterpret_cast<uint16_t*>(w);
  TPQ_CUDA(cudaMemsetAsync(hist, 0, (size_t)nch * n_cells * 4, st));
  ioa_local_kernel<<<(unsigned)nch, 512, 0, st>>>(cells, n, n_cells, lrank, hist);
  TPQ_LAUNCH_CHECK("ioa_local_kernel");
  ioa_scan_kernel<<<(n_cells + 255) / 256, 256, 0, st>>>(hist, (int)nch, n_cells, counts);
  TPQ_LAUNCH_CHECK("ioa_scan_kernel");
  ioa_finish_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(cells, lrank, hist, n, n_cells, ioa);
  TPQ_LAUNCH_CHECK("ioa_finish_kernel");
  return TPQ_OK;
}

extern "C" size_t tpq_empty_prefix_workspace_bytes(int64_t capacity) {
  return align_up((size_t)((capacity + EP_TILE) / EP_TILE + 1) * 4, 256);
}

extern "C" int tpq_empty_prefix(const uint8_t* is_empty, int64_t capacity, uint32_t* prefix, void* ws, size_t ws_bytes, void* stream) {
  TPQ_REQUIRE(is_empty && prefix && capacity >= 0 && capacity < 0xFFFFFFFFll, "tpq_empty_prefix: bad argument");
  if (!ws || ws_bytes < tpq_empty_prefix_workspace_bytes(capacity)) { set_error("tpq_empty_prefix: workspace too small"); return TPQ_ERR_WORKSPACE; }
  cudaStream_t st = (cudaStream_t)stream;
  const int tiles = (int)((capacity + EP_TILE) / EP_TILE);              // covers slot `capacity` itself (the total)
  uint32_t* tsum = reinterpret_cast<uint32_t*>(ws);
  empty_tile_sums_kernel<<<tiles, EP_T, 0, st>>>(is_empty, capacity, tsum);
  TPQ_LAUNCH_CHECK("empty_tile_sums_kernel");
  scan_u32_inplace_kernel<<<1, 1024, 0, st>>>(tsum, tiles);
  TPQ_LAUNCH_CHECK("scan_u32_inplace_kernel");
  empty_prefix_kernel<<<tiles, EP_T, 0, st>>>(is_empty, capacity, tsum, prefix);
  TPQ_LAUNCH_CHECK("empty_prefix_kernel");
  return TPQ_OK;
}

extern "C" int tpq_get_write_address(const int64_t* cells, const int64_t* ioa, int64_t n,
                                     const int64_t* cell_start, const int64_t* cell_size, const int64_t* cell_capacity,
                                     int n_cells, const uint32_t* empty_prefix, int64_t* write_adr, void* stream) {
  TPQ_REQUIRE(n >= 0 && n_cells > 0, "tpq_get_write_address: bad sizes");
  if (n == 0) return TPQ_OK;
  TPQ_REQUIRE(cells && ioa && cell_start && cell_size && cell_capacity && write_adr, "tpq_get_write_address: null pointer");
  write_address_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(cells, ioa, n, cell_start, cell_size,
                                                                                     cell_capacity, n_cells, empty_prefix, write_adr);
  TPQ_LAUNCH_CHECK("write_address_kernel");
  return TPQ_OK;
}

extern "C" int tpq_store_codes(const uint8_t* codes, const int64_t* cells, const int64_t* write_adr, const int64_t* ids,
                               int64_t n, tpq_index* ix, uint8_t* storage, int64_t* address2id, uint8_t* is_empty,
                               int64_t* cell_size, uint8_t* codes_scan, uint32_t* block_valid, void* stream) {
  TPQ_REQUIRE(ix && n >= 0, "tpq_store_codes: bad argument");
  if (n == 0) return TPQ_OK;
  TPQ_REQUIRE(codes && cells && write_adr && ids && storage && address2id && is_empty && cell_size && ix->cell_start,
              "tpq_store_codes: null pointer");
  const int M = ix->n_subvectors;
  const int code_size = ix->code_size ? ix->code_size : M;
  TPQ_REQUIRE(M > 0 && M % 4 == 0, "n_subvectors must be a positive multiple of 4, got %d", M);
  TPQ_REQUIRE(code_size >= M && code_size % 4 == 0, "code_size=%d must be 0 or a multiple of 4 that is >= n_subvectors=%d",
              ix->code_size, M);
  TPQ_REQUIRE(!codes_scan || (block_valid && ix->cell_block_start && ix->m_pad == scan_m_pad(M)), "tpq_store_codes: incomplete scan layout");
  dim3 grid((unsigned)((n + 255) / 256), code_size / 4);
  store_codes_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(
      codes, cells, write_adr, ids, n, M, ix->capacity, reinterpret_cast<uint32_t*>(storage), address2id, is_empty,
      reinterpret_cast<long long*>(cell_size), ix->cell_start, codes_scan, block_valid, ix->cell_block_start, ix->m_pad,
      ix->shard_rank, ix->shard_world < 1 ? 1 : ix->shard_world);
  TPQ_LAUNCH_CHECK("store_codes_kernel");
  return TPQ_OK;
}

extern "C" int tpq_expand_move(const uint8_t* old_storage, const int64_t* old_address2id, const uint8_t* old_is_empty,
                               const int64_t* old_cell_start, const int64_t* shift, int n_cells, int M,
                               int64_t old_capacity, int64_t new_capacity,
                               uint8_t* storage, int64_t* address2id, uint8_t* is_empty, void* stream) {
  TPQ_REQUIRE(old_storage && old_address2id && old_is_empty && old_cell_start && shift && storage && address2id && is_empty,
              "tpq_expand_move: null pointer");
  TPQ_REQUIRE(n_cells > 0 && M > 0 && M % 4 == 0 && old_capacity >= 0 && new_capacity >= old_capacity, "tpq_expand_move: bad sizes");
  if (old_capacity == 0) return TPQ_OK;
  expand_move_kernel<<<(unsigned)((old_capacity + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const uint32_t*>(old_storage), old_address2id, old_is_empty, old_cell_start, shift, n_cells,
      old_capacity, new_capacity, M / 4, reinterpret_cast<uint32_t*>(storage), address2id, is_empty);
  TPQ_LAUNCH_CHECK("expand_move_kernel");
  return TPQ_OK;
}
