// Range search's match buffers: the CTA's, shared by flat_range_kernel (flat.cu) and ivfflat_range_kernel (ivfflat.cu),
// and the warp's, of ivfpq_range_kernel (scan.cu).
//
// A range kernel keeps no per-query lists: after each 128-column tile's epilogue every thread holds its scores in
// registers, and the ones above the threshold are appended to one buffer of the CTA in shared memory as (row of the
// query tile, make_key(score, address)).  When the buffer cannot take another whole tile, and at the end, the CTA
// reserves its place in the caller's match arrays with one global atomic and copies the buffer out, coalesced.  The
// global counter always reaches the exact total; entries at or past `cap` are counted and not written.
//
// The IVFPQ scan's CTA serves one query, and its warps take 32-vector blocks from a dynamic cursor, each at its own
// pace: there a warp stages its own matches (keys only: the query is the CTA's) and flushes them itself, by the same
// rule, when its buffer cannot take another block and when it runs out of blocks.  No CTA barrier is involved.
#pragma once
#include "common.cuh"

namespace tpq {

constexpr int kRangeBuf = 9216;       // entries: one 64 x 128 tile's every score, plus 1024

struct RangeBuf {
  uint64_t key[kRangeBuf];
  unsigned long long base;            // the flush's first global entry
  int cnt;                            // staged entries
  uint8_t row[kRangeBuf];             // row of the CTA's query tile (QT <= 64)
};

#ifdef __CUDACC__
// The thread's matches among its micro-tile: bit i * 8 + j of `pass` marks o[i][j], whose tile row is row(i) and whose
// address is addr(j).  One shared atomic per warp reserves the warp's run; a thread writes its matches in a row.
template <int MI, class Row, class Addr>
__device__ __forceinline__ void range_append(RangeBuf& b, uint32_t pass, const float (&o)[MI][8], Row row, Addr addr,
                                             int lane) {
  const int mine = __popc(pass);
  const int incl = warp_inclusive_scan(mine, lane);
  int at = 0;
  if (lane == 31 && incl) at = atomicAdd(&b.cnt, incl);
  at = __shfl_sync(0xffffffffu, at, 31) + incl - mine;
  if (!pass) return;
  #pragma unroll
  for (int i = 0; i < MI; ++i)
    #pragma unroll
    for (int j = 0; j < 8; ++j)
      if (pass & (1u << (i * 8 + j))) {
        b.key[at] = make_key(o[i][j], addr(j));
        b.row[at] = (uint8_t)row(i);
        ++at;
      }
}

// Called by every thread after a barrier that follows the last append.  query(row) maps a tile row to the query it
// belongs to.  Ends with the buffer empty; the next append must follow a barrier (GemmTile::run's first).
template <class Query>
__device__ __forceinline__ void range_flush(RangeBuf& b, unsigned long long* __restrict__ total, int64_t cap,
                                            uint64_t* __restrict__ keys_out, int32_t* __restrict__ q_out,
                                            Query query) {
  const int n = b.cnt;
  if (n == 0) return;                                  // uniform: every thread read it after the same barrier
  if (threadIdx.x == 0) b.base = atomicAdd(total, (unsigned long long)n);
  __syncthreads();
  const unsigned long long base = b.base;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const unsigned long long g = base + i;
    if (g < (unsigned long long)cap) {
      keys_out[g] = b.key[i];
      q_out[g] = query(b.row[i]);
    }
  }
  __syncthreads();                                     // every thread has read n and the buffer
  if (threadIdx.x == 0) b.cnt = 0;
}
#endif  // __CUDACC__

constexpr int kRangeWarpBuf = 96;     // keys a warp stages: it flushes when fewer than a block's 32 places are left

// Where a warp's matches go: a kernel parameter (__grid_constant__, so the warps read it in place, not from registers).
struct RangeOut {
  float t;                            // the threshold: a score matches when score > t
  uint64_t* keys; int32_t* query; int64_t cap; unsigned long long* total;
};

// One warp's match buffer: buf [kRangeWarpBuf] keys in shared memory, its count in a (warp-uniform) register.
struct RangeWarpBuf {
  uint64_t* buf;
  int cnt;
  int32_t q;                          // the query every match of the warp belongs to
  const RangeOut* out;
#ifdef __CUDACC__
  // the lanes with `pass` append their keys (every lane calls); flush when another block might not fit
  __device__ __forceinline__ void push(bool pass, uint64_t key, int lane) {
    cnt += warp_append(buf, cnt, pass, key, lane);
    if (cnt > kRangeWarpBuf - 32) flush(lane);
  }
  // Lane 0 reserves the run with one global atomic; the lanes copy it out, coalesced.  Ends with the buffer empty.
  __device__ __forceinline__ void flush(int lane) {
    if (cnt == 0) return;                              // warp-uniform
    __syncwarp();                                      // every lane's appended key is visible to the warp
    unsigned long long base = 0;
    if (lane == 0) base = atomicAdd(out->total, (unsigned long long)cnt);
    base = __shfl_sync(0xffffffffu, base, 0);
    for (int i = lane; i < cnt; i += 32) {
      const unsigned long long g = base + i;
      if (g < (unsigned long long)out->cap) { out->keys[g] = buf[i]; out->query[g] = q; }
    }
    __syncwarp();                                      // every lane has read the buffer before it is refilled
    cnt = 0;
  }
#endif
};

}  // namespace tpq
