// Builds the scan layout (format: scan_layout.cuh) and the scan-side codebooks from the reference's buffers.
#include "lut.cuh"

namespace tpq {

// cell_block_start[c] = sum over owned c' < c of ceil(cell_size[c'] / 32)
__global__ void __launch_bounds__(1024)
relayout_plan_kernel(const int64_t* __restrict__ cell_size, int C, int rank, int world,
                     int32_t* __restrict__ cell_block_start) {
  __shared__ int warp_sums[32];
  __shared__ int carry_s;
  if (threadIdx.x == 0) { carry_s = 0; cell_block_start[0] = 0; }
  __syncthreads();
  for (int c0 = 0; c0 < C; c0 += 1024) {
    const int c = c0 + threadIdx.x;
    const int incl = cta_inclusive_scan(c < C && shard_owns(c, rank, world) ? (int)scan_blocks(cell_size[c]) : 0,
                                        warp_sums, carry_s);
    if (c < C) cell_block_start[c + 1] = incl;
  }
}

// one warp per output block
__global__ void __launch_bounds__(256)
relayout_codes_kernel(const uint32_t* __restrict__ storage,   // [M/4, cap] words
                      const uint8_t* __restrict__ is_empty, const int64_t* __restrict__ cell_start,
                      const int64_t* __restrict__ cell_size, const int32_t* __restrict__ cell_block_start,
                      int C, int M, int MP, int64_t cap, int64_t n_blocks,
                      uint8_t* __restrict__ codes_scan, uint32_t* __restrict__ block_valid) {
  extern __shared__ __align__(16) uint8_t smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const int row = MP + 4;                                   // padded record stride (bytes)
  uint8_t* rec = smem + (size_t)warp * 32 * row;
  for (int64_t B = (int64_t)blockIdx.x * nw + warp; B < n_blocks; B += (int64_t)gridDim.x * nw) {
    // cell of this block: last c with cell_block_start[c] <= B
    int lo = 0, hi = C;                                     // invariant: start[lo] <= B < start[hi]
    while (hi - lo > 1) { int mid = (lo + hi) >> 1; if (cell_block_start[mid] <= B) lo = mid; else hi = mid; }
    // cells with zero blocks share a start value with their successor; move to the one that owns B
    const int c = lo;
    const int64_t pos = (B - cell_block_start[c]) * 32 + lane;
    const int64_t a = cell_start[c] + pos;
    const bool inrange = pos < cell_size[c] && a < cap;
    const bool live = inrange && is_empty[a] == 0;
    for (int g = 0; g < MP / 4; ++g) {
      uint32_t w = (inrange && g < M / 4) ? storage[(size_t)g * cap + a] : 0u;
      *reinterpret_cast<uint32_t*>(rec + lane * row + g * 4) = w;
    }
    __syncwarp();
    for (int j = 0; j < MP / 16; ++j) {
      uint32_t o[4];
      #pragma unroll
      for (int wd = 0; wd < 4; ++wd) {
        uint32_t v = 0;
        #pragma unroll
        for (int bb = 0; bb < 4; ++bb) {
          const int m = rot_subq(j * 16 + wd * 4 + bb, lane);
          v |= ((m < M) ? (uint32_t)rec[lane * row + m] : 0u) << (8 * bb);
        }
        o[wd] = v;
      }
      *reinterpret_cast<uint4*>(codes_scan + scan_chunk_offset(B, MP, j, lane)) = make_uint4(o[0], o[1], o[2], o[3]);
    }
    unsigned mask = __ballot_sync(0xffffffffu, live);
    if (lane == 0) block_valid[B] = mask;
    __syncwarp();
  }
}

// pq_codebook [M, dsub, 256] -> pq_codebook_t [256, MP, dsub], pq_norm_t [256, MP]
__global__ void relayout_codebook_kernel(const float* __restrict__ cb, int M, int MP, int dsub, int metric,
                                         float* __restrict__ cbt, float* __restrict__ nrm) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;          // c * MP + m
  if (idx >= 256 * MP) return;
  int c = idx / MP, m = idx % MP;
  float b2 = 0.f;
  for (int i = 0; i < dsub; ++i) {
    float v = (m < M) ? cb[((size_t)m * dsub + i) * 256 + c] : 0.f;
    cbt[(size_t)idx * dsub + i] = v;
    b2 = __fadd_rn(b2, __fmul_rn(v, v));
  }
  nrm[idx] = (metric == TPQ_METRIC_EUCLIDEAN) ? b2 : 0.f;
}

}  // namespace tpq

using namespace tpq;

extern "C" size_t tpq_part2_scan_bytes(int M, int n_cells) {
  return (size_t)n_cells * lut_bytes(scan_m_pad(M));
}

extern "C" int tpq_relayout_part2(const float* vq_codebook, const float* pq_codebook, int d, int M, int n_cells,
                                  float* part2_scan, void* stream) {
  TPQ_REQUIRE(vq_codebook && pq_codebook && part2_scan, "tpq_relayout_part2: null pointer");
  TPQ_REQUIRE(d > 0 && M > 0 && d % M == 0 && n_cells > 0, "tpq_relayout_part2: bad sizes");
  // part2_scan[c] = the residual LUT's cell half (lut.cuh), the cells of vq_codebook [d, n_cells] as the rows.  The
  // kernel writes m_pad rows; a partly used last group's other rows stay +0.
  if (scan_m_pad(M) % 64)
    TPQ_CUDA(cudaMemsetAsync(part2_scan, 0, tpq_part2_scan_bytes(M, n_cells), (cudaStream_t)stream));
  return launch_lut(vq_codebook, n_cells, 0, n_cells, pq_codebook, d, M, kLutPart2, kLutScan, part2_scan,
                    (cudaStream_t)stream);
}

extern "C" int tpq_relayout_plan(const int64_t* cell_size, int n_cells, int shard_rank, int shard_world,
                                 int32_t* cell_block_start, void* stream) {
  TPQ_REQUIRE(cell_size && cell_block_start && n_cells > 0, "tpq_relayout_plan: bad argument");
  TPQ_REQUIRE(shard_world >= 1 && shard_rank >= 0 && shard_rank < shard_world, "bad shard %d/%d", shard_rank, shard_world);
  relayout_plan_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(cell_size, n_cells, shard_rank, shard_world, cell_block_start);
  TPQ_LAUNCH_CHECK("relayout_plan_kernel");
  return TPQ_OK;
}

extern "C" size_t tpq_codes_scan_bytes(int M, int64_t n_blocks) {
  return (size_t)n_blocks * scan_block_bytes(scan_m_pad(M));
}

extern "C" int tpq_relayout_codes(const tpq_index* ix, uint8_t* codes_scan, uint32_t* block_valid, void* stream) {
  TPQ_REQUIRE(ix && codes_scan && block_valid, "tpq_relayout_codes: null pointer");
  TPQ_REQUIRE(ix->storage && ix->is_empty && ix->cell_start && ix->cell_size && ix->cell_block_start,
              "tpq_relayout_codes: index is missing reference buffers or the block plan");
  const int M = ix->n_subvectors;
  TPQ_REQUIRE(M > 0 && M % 4 == 0, "n_subvectors must be a positive multiple of 4, got %d", M);
  const int MP = scan_m_pad(M);
  TPQ_REQUIRE(ix->m_pad == MP, "index.m_pad=%d, expected %d", ix->m_pad, MP);
  TPQ_REQUIRE(ix->capacity <= 0xFFFFFFFFll, "capacity %lld exceeds the 32-bit address range", (long long)ix->capacity);
  if (ix->n_blocks == 0) return TPQ_OK;
  const int nw = 8;
  size_t smem = (size_t)nw * 32 * (MP + 4);
  TPQ_CUDA(cudaFuncSetAttribute(relayout_codes_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int64_t grid = (ix->n_blocks + nw - 1) / nw;
  const int64_t cap = (int64_t)device_sm_count() * 64;
  if (grid > cap) grid = cap;
  relayout_codes_kernel<<<(int)grid, nw * 32, smem, (cudaStream_t)stream>>>(
      reinterpret_cast<const uint32_t*>(ix->storage), ix->is_empty, ix->cell_start, ix->cell_size,
      ix->cell_block_start, ix->n_cells, M, MP, ix->capacity, ix->n_blocks, codes_scan, block_valid);
  TPQ_LAUNCH_CHECK("relayout_codes_kernel");
  return TPQ_OK;
}

extern "C" int tpq_relayout_codebook(const float* pq_codebook, int d, int M, int metric,
                                     float* pq_codebook_t, float* pq_norm_t, void* stream) {
  TPQ_REQUIRE(pq_codebook && pq_codebook_t && pq_norm_t, "tpq_relayout_codebook: null pointer");
  TPQ_REQUIRE(d > 0 && M > 0 && d % M == 0, "d_vector=%d must be a multiple of n_subvectors=%d", d, M);
  TPQ_REQUIRE(metric == TPQ_METRIC_EUCLIDEAN || metric == TPQ_METRIC_COSINE, "tpq_relayout_codebook: unsupported metric %d", metric);
  const int MP = scan_m_pad(M);
  int n = 256 * MP;
  relayout_codebook_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(pq_codebook, M, MP, d / M, metric,
                                                                              pq_codebook_t, pq_norm_t);
  TPQ_LAUNCH_CHECK("relayout_codebook_kernel");
  return TPQ_OK;
}
