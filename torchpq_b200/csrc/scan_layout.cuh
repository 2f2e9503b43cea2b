// Scan ("shadow") layout of the index and the rule by which a scan visits probe entries: relayout.cu, place.cu, scan.cu.
//
// The reference keeps codes as _storage[M/4, capacity, 4] (container/CellContainer.py:46-53,
// 213-239): 4-byte granules strided by 4*capacity bytes -- fine for its 4-byte loads
// (ivfpq_topk.cu:650-660), useless for 128-bit ones.  The scan layout groups every cell's
// slots [cell_start, cell_start+cell_capacity) into blocks of 32 vectors; a block is
// m_pad/16 chunks of 512 bytes, chunk j holding 16 bytes for each of the 32 lanes, so one
// warp-wide LDG.128 per chunk is a single fully coalesced 512-byte request.
//
// Lane l owns vector l of the block.  Its m_pad record bytes are LANE-ROTATED: record byte
// t (half-group h = t/32, rotation r = t%32) holds the code of sub-quantizer
//     m(l, t) = 32*h + ((l + r) & 31)
// so that at any step the 32 lanes of a warp look up 32 different sub-quantizers, i.e. 32
// different shared-memory banks of the [code][sub-quantizer] LUT (scan.cu) -- every LDS is
// conflict-free whatever the codes are.  Padding sub-quantizers (m >= M) get code 0.
//
// A LUT in scan layout is lut[g][code][s] (g = m / 64, s = m % 64, fp32): one 64 KB group of 256 x 64 floats per 64
// sub-quantizers, in the scan kernels' shared memory and in the tables written to global memory.
#pragma once
#include "common.cuh"

namespace tpq {

__host__ __device__ constexpr int scan_m_pad(int M) { return (M + 31) / 32 * 32; }
__host__ __device__ constexpr size_t scan_block_bytes(int MP) { return (size_t)MP * 32; }
// the 16 bytes of lane `lane` in chunk j of block B
__host__ __device__ __forceinline__ size_t scan_chunk_offset(int64_t B, int MP, int j, int lane) {
  return (size_t)B * scan_block_bytes(MP) + ((size_t)j * 32 + lane) * 16;
}
// record byte t of lane `lane` holds sub-quantizer rot_subq(t, lane); sub-quantizer m is in record byte rot_byte(m, lane)
__host__ __device__ constexpr int rot_subq(int t, int lane) { return (t & ~31) + ((lane + t) & 31); }
__host__ __device__ constexpr int rot_byte(int m, int lane) { return (m & ~31) | ((m - lane) & 31); }
// the lane's LUT slot offsets for the scan kernels: byte b of off[i] = 4 * slot of record byte 4 i + b in its half-group
__device__ __forceinline__ void lane_slot_offsets(uint32_t (&off)[8], int lane) {
  #pragma unroll
  for (int i = 0; i < 8; ++i) {
    uint32_t v = 0;
    #pragma unroll
    for (int b = 0; b < 4; ++b) v |= (uint32_t)(rot_subq(4 * i + b, lane) * 4) << (8 * b);
    off[i] = v;
  }
}

constexpr int kLutGroup = 256 * 64;                                               // floats of one 64-sub-quantizer group
__host__ __device__ constexpr int lut_groups(int MP) { return (MP + 63) / 64; }
__host__ __device__ constexpr int lut_bytes(int MP) { return lut_groups(MP) * kLutGroup * 4; }
__host__ __device__ constexpr int lut_index(int m, int code) { return (m >> 6) * kLutGroup + code * 64 + (m & 63); }
// byte offset of code 0 of half-group h (sub-quantizers 32 h .. 32 h + 31) of group g
__host__ __device__ constexpr int lut_half_group_offset(int g, int h) { return (g * kLutGroup + h * 32) * 4; }

// cell c is laid out on shard (rank, world); another shard's cells get zero blocks
template <class I>
__host__ __device__ constexpr bool shard_owns(I c, int rank, int world) { return c % world == rank; }

// The visiting rule of the query-major kernel (ivfpq_topk.cu:837-870), which the cell-major path must reproduce pair for
// pair to stay exact.  A query scans its first P probe entries: the plain kernel enters the first cell unconditionally,
// the residual one loops `for cCell < nProbe` (:1080) and may scan none.
template <bool RES>
__device__ __forceinline__ int probe_count(int64_t n_probe_list_q, int n_probe) {
  const int P = (int)n_probe_list_q;
  return RES ? max(0, min(P, n_probe)) : max(1, min(P, n_probe));
}

// Which of a query's first P entries are visited, for every probe-list scan (IVFPQ's scan layout and IVFFlat's flat
// store alike): entry j is skipped when its cell is outside [0, n_cells) (caller-supplied lists are not trusted) or when
// its cell_start equals that of entry j - 1 (a cell listed twice in a row is scanned once; twice apart, twice).  A visited
// entry scans its cell's live extent [s, s + cell_size), nothing for an empty cell.  s: the cell's start, -1 outside.
__device__ __forceinline__ bool probe_visits(const int64_t* cq, int j, int n_cells, const int64_t* cell_start, int64_t& s) {
  const int64_t c = cq[j];
  const bool ok = c >= 0 && c < n_cells;
  s = ok ? cell_start[c] : -1;
  bool skip = !ok;
  if (ok && j > 0) {
    const int64_t cp = cq[j - 1];
    skip = cp >= 0 && cp < n_cells && s == cell_start[cp];
  }
  return !skip;
}

__host__ __device__ constexpr int64_t scan_blocks(int64_t n) { return n > 0 ? (n + 31) >> 5 : 0; }
// Blocks a scan reads of a cell whose layout holds blocks [b0, b1): the layout has a block for every slot of the cell's
// capacity (none for another shard's cell), the live extent is cell_size.
__device__ __forceinline__ int cell_blocks(int b0, int b1, int64_t size) { return (int)min((int64_t)(b1 - b0), scan_blocks(size)); }

struct ProbeEntry {
  int64_t cell;                 // 0 (and nb 0) when outside [0, n_cells): caller-supplied probe lists are not trusted
  int blk0;                     // first block of the cell (0 for none)
  uint32_t addr0;               // address of its first slot
  int nb;                       // blocks to scan: 0 for none, an empty or another shard's cell, or the previous entry's
};                              // cell_start (a cell listed twice apart is scanned twice)
__device__ __forceinline__ ProbeEntry probe_entry(const int64_t* cq, int j, int n_cells, const int64_t* cell_start,
                                                  const int64_t* cell_size, const int32_t* cell_block_start) {
  ProbeEntry e;
  const int64_t c = cq[j];
  const bool ok = c >= 0 && c < n_cells;
  int64_t s;
  const bool visit = probe_visits(cq, j, n_cells, cell_start, s);
  e.cell = ok ? c : 0;
  e.blk0 = ok ? cell_block_start[c] : 0;
  e.addr0 = (uint32_t)s;
  e.nb = visit ? cell_blocks(e.blk0, cell_block_start[c + 1], cell_size[c]) : 0;
  return e;
}

}  // namespace tpq
