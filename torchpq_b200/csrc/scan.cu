// The hot path: fused IVF list scan + top-k over the scan layout (relayout.cu).
//
// Replaces the reference's ivfpq_topk kernel (torchpq/kernels/cuda/ivfpq_topk.cu:822-971,
// >90 % of search time there) together with the LUT hand-off, the [nq,n_probe] gathers
// (IVFPQIndex.py:420-421) and get_id_by_address (container/BaseContainer.py:58-65).
//
// Per (query, slice) CTA:
//   * the query's LUT sits in shared memory TRANSPOSED, lut[g][code][s] (scan_layout.cuh), and because the codes are
//     lane-rotated, lane l at step t reads slot s = 32*(h&1) + ((l + t) & 31): 32 lanes -> 32 distinct banks.
//   * one PRMT builds the whole address: byte 1 = the code byte, byte 0 = the lane's
//     precomputed slot offset, bytes 2..3 = sign-replicated zero; the half-group and
//     group offsets are LDS immediates.  Inner loop = PRMT + LDS + FADD per code byte.
//   * the LUT itself is built by the CTA, in place, from the L2-resident transposed codebook (build_lut, lut.cuh; d/M
//     in {1,2,4,8}); otherwise it is staged through HBM by lut_kernel (lut.cu).
//   * each warp streams whole 32-vector blocks with coalesced 128-bit loads in units of 64
//     sub-quantizers, software pipelined one unit ahead (ping-pong register sets).
//   * top-k (CtaTopK, common.cuh): one compare against the CTA-wide running k-th best + one ballot per
//     block; survivors are staged per warp and merged into the CTA's single sorted list under a lock;
//     the threshold is bootstrapped, and the buffers are drained, by CTA-wide sorts.  The selector lays out its own
//     shared memory (threshold, lock, list, staging buffers): the kernel reserves CtaTopK::bytes and passes the address.
//   * RES variant: residual IVFPQ (per-cell LUT = query half + precomputed cell half).
// Sub-quantizer sums are fp32 in four interleaved partial sums (exact for integer LUTs;
// ~1e-7 relative otherwise -- the reference's m-ascending order lives in scan_ref.cu).
// Experiment knobs (TPQ_SCAN_CFG, TPQ_BOOT_R, TPQ_LUT_MODE, TPQ_CELL_CFG, TPQ_CELL_ABLATE) and per-phase cycle counters
// exist only in the -DTPQ_DEBUG_KNOBS build (make dbg -> libtpq_b200_dbg.so, used by scripts/); the product library reads no environment.
#include <stdlib.h>
#include <string.h>
#include <type_traits>
#include "lut.cuh"
#include "range.cuh"
#include "tc_common.cuh"

namespace tpq {

// ----------------------------------------------------------------------------- scan kernel
__device__ __forceinline__ uint32_t prmt(uint32_t a, uint32_t b, uint32_t sel) {
  uint32_t d;
  asm("prmt.b32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(sel));
  return d;
}
// LUT entry for code byte J of `w`, slot offset byte J of `off`; imm = group/half-group byte offset.
template <int J>
__device__ __forceinline__ float lut_at(const uint8_t* lut, uint32_t w, uint32_t off, int imm) {
  constexpr uint32_t sel = (4u + J) | (uint32_t(J) << 4) | ((8u | (4u + J)) << 8) | ((8u | (4u + J)) << 12);
  return *reinterpret_cast<const float*>(lut + prmt(w, off, sel) + imm);
}
__device__ __forceinline__ uint4 ldg_stream(const uint4* p) {
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
  return v;
}

// A block (32 vectors x MP code bytes) is consumed in UNITS of up to 64 sub-quantizers (4 chunks = 16 words per
// lane), so the register footprint and the software pipeline are the same for every M: while unit u is being
// looked up, unit u+1 (the next 64 sub-quantizers of the block, or the first unit of the warp's next block) is in flight.
template <int MP>
struct Units {
  static constexpr int NSB = lut_groups(MP);          // unit u is looked up in LUT group u
  __host__ __device__ static constexpr int words(int sb) { return (sb == NSB - 1 && (MP % 64) != 0) ? 8 : 16; }
};

template <int MP, int SB>
__device__ __forceinline__ void load_unit(uint32_t (&w)[16], const uint8_t* __restrict__ codes, int64_t B, int lane) {
  // chunks 4 SB .. 4 SB + 3 of block B; lane's 16 bytes of chunk c are uint4 32 c + lane (scan_chunk_offset)
  const uint4* p = reinterpret_cast<const uint4*>(codes + (size_t)B * scan_block_bytes(MP)) + SB * 128 + lane;
  #pragma unroll
  for (int j = 0; j < Units<MP>::words(SB) / 4; ++j) {
    const uint4 v = ldg_stream(p + j * 32);
    w[4 * j + 0] = v.x; w[4 * j + 1] = v.y; w[4 * j + 2] = v.z; w[4 * j + 3] = v.w;
  }
}

template <int MP, int SB>
__device__ __forceinline__ void adc_unit(const uint32_t (&w)[16], const uint32_t (&off)[8], const uint8_t* lut, float (&acc)[4]) {
  #pragma unroll
  for (int i = 0; i < Units<MP>::words(SB); ++i) {
    const int imm = lut_half_group_offset(SB, i >> 3);
    acc[0] += lut_at<0>(lut, w[i], off[i & 7], imm);
    acc[1] += lut_at<1>(lut, w[i], off[i & 7], imm);
    acc[2] += lut_at<2>(lut, w[i], off[i & 7], imm);
    acc[3] += lut_at<3>(lut, w[i], off[i & 7], imm);
  }
}

// This lane's score of a block: the four partial sums of adc_unit are added in this association, on top of `base`.
__device__ __forceinline__ float block_score(const float (&acc)[4], float base) {
  return base + ((acc[0] + acc[1]) + (acc[2] + acc[3]));
}
// This lane's key of a block, its address addr0 + lane.  Every key and every range match of the scan kernels is formed
// from block_score, which is what makes the cell-major path's results, and range search's scores, the query-major
// kernel's bit for bit.
__device__ __forceinline__ uint64_t block_key(const float (&acc)[4], float base, uint32_t addr0, int lane) {
  return make_key(block_score(acc, base), addr0 + lane);
}

// Per-warp scan state.  regs[2][16] is the ping-pong pair of unit buffers; every index into it is a
// compile-time constant after unrolling (PAR / SB are template parameters), so it lives in registers.
// RANGE: the blocks' scores go to the warp's range buffer `rs` (every live score above its threshold) instead of the
// CTA's top-k `tk`.
template <int MP, int NW, bool RANGE = false>
struct Scanner {
  static constexpr int NSB = Units<MP>::NSB;
  const uint8_t* codes; const uint32_t* valid; const uint8_t* lut;
  const int32_t* seg_prefix; const int32_t* seg_blk0; const uint32_t* seg_addr0;
  int* next;                                            // CTA-wide cursor: next block (of the concatenated probe list) to hand out
  int lane;
  uint32_t off[8];
  uint32_t regs[2][16];
  CtaTopK tk;
  uint64_t thr;
  RangeWarpBuf rs;
  float base;                                          // residual IVFPQ: coarse similarity of the current cell (else 0)
  int seg, seg_lo, seg_hi, seg_b0; uint32_t seg_a0;     // current probe segment, cached in registers
  int64_t B_cur, B_nxt; uint32_t a0_cur, a0_nxt, valid_cur, valid_nxt;

  __device__ __forceinline__ void locate(int b, int64_t& B, uint32_t& addr0) {
    if (b >= seg_hi) {
      do { ++seg; seg_lo = seg_hi; seg_hi = seg_prefix[seg + 1]; } while (b >= seg_hi);
      seg_b0 = seg_blk0[seg]; seg_a0 = seg_addr0[seg];
    }
    const int rel = b - seg_lo;
    B = (int64_t)seg_b0 + rel;
    addr0 = seg_a0 + (uint32_t)rel * 32u;
  }
  template <int PAR, int SB>
  __device__ __forceinline__ void step(float (&acc)[4], bool has_next) {
    constexpr int BUF = (PAR + SB) & 1;
    if constexpr (SB + 1 < NSB) {
      load_unit<MP, SB + 1>(regs[BUF ^ 1], codes, B_cur, lane);
    } else {
      if (has_next) { load_unit<MP, 0>(regs[BUF ^ 1], codes, B_nxt, lane); valid_nxt = __ldg(valid + B_nxt); }
    }
    adc_unit<MP, SB>(regs[BUF], off, lut, acc);
    if constexpr (SB + 1 < NSB) step<PAR, SB + 1>(acc, has_next);
  }
  // consume the block at the cursor (its unit 0 is already in regs[PAR]); prefetch the next block's unit 0
  template <int PAR>
  __device__ __forceinline__ void process_block(bool has_next) {
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    step<PAR, 0>(acc, has_next);
    if constexpr (RANGE) {
      const float s = block_score(acc, base);              // fp32 compare: +0 > -0 is false, a NaN never matches
      const bool live = (valid_cur >> lane) & 1u;
      rs.push(live && s > rs.out->t, make_key(s, a0_cur + lane), lane);
    } else {
      const uint64_t key = block_key(acc, base, a0_cur, lane);
      const bool live = (valid_cur >> lane) & 1u;
      if (PAR == 0) thr = tk.threshold();                // running k-th best of the CTA
      tk.push(live && key > thr, key, lane);
    }
    B_cur = B_nxt; a0_cur = a0_nxt; valid_cur = valid_nxt;
  }
  template <int SB>
  __device__ __forceinline__ void simple_units(float (&acc)[4], int64_t B) {
    load_unit<MP, SB>(regs[0], codes, B, lane);
    adc_unit<MP, SB>(regs[0], off, lut, acc);
    if constexpr (SB + 1 < NSB) simple_units<SB + 1>(acc, B);
  }
  // score one block without pipelining and return this lane's key (0 if the slot is not live)
  __device__ __forceinline__ uint64_t key_of_block(int b) {
    int64_t B; uint32_t a0;
    locate(b, B, a0);
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    simple_units<0>(acc, B);
    const uint32_t v = __ldg(valid + B);
    return ((v >> lane) & 1u) ? block_key(acc, base, a0, lane) : 0ull;
  }
  // Blocks are handed out dynamically: `next` is a CTA-wide counter in shared memory.  (A static stripe b = warp,
  // warp + NW, ... left the CTA waiting for its slowest warp -- the warp schedulers favour the oldest warps, so the
  // youngest ones finished noticeably later than warp 0, most with 16 warps and one CTA per SM.)  The index of the
  // block after next is fetched before the current block is consumed, so the atomic's latency is off the critical path.
  __device__ __forceinline__ int grab() {
    int b = 0;
    if (lane == 0) b = atomicAdd(next, 1);
    return __shfl_sync(0xffffffffu, b, 0);
  }
  __device__ __forceinline__ void run(int b_end) {
    int b = grab();
    if (b >= b_end) return;
    locate(b, B_cur, a0_cur);
    load_unit<MP, 0>(regs[0], codes, B_cur, lane);
    valid_cur = __ldg(valid + B_cur);
    for (;;) {
      b = grab();
      bool more = b < b_end;
      if (more) locate(b, B_nxt, a0_nxt);
      process_block<0>(more);
      if (!more) break;
      if constexpr (NSB % 2 == 1) {                       // odd unit count: the buffers swap roles every block
        b = grab();
        more = b < b_end;
        if (more) locate(b, B_nxt, a0_nxt);
        process_block<1>(more);
        if (!more) break;
      }
    }
  }
};

struct ScanSmem { size_t lut, part1, seg_blk0, seg_addr0, seg_cell, seg_prefix, next, topk, total; };
static ScanSmem scan_smem(int MP, int n_probe, int nw, int kp, bool residual = false, bool part1_in_smem = false) {
  ScanSmem s; size_t off = 0;
  s.lut = off;        off += lut_bytes(MP);
  s.part1 = off;      off += (residual && part1_in_smem) ? lut_bytes(MP) : 0;   // query half of the residual LUT
  s.seg_cell = off;   off += residual ? (size_t)n_probe * 4 : 0;
  s.seg_blk0 = off;   off += (size_t)n_probe * 4;
  s.seg_addr0 = off;  off += (size_t)n_probe * 4;
  s.seg_prefix = off; off += (size_t)(n_probe + 1) * 4;
  s.next = off;       off += 4;                                       // the block cursor (Scanner::next)
  off = align_up(off, 8);
  s.topk = off;       off += CtaTopK::bytes(nw, kp);
  s.total = off;
  return s;
}

struct ScanArgs {
  const uint8_t* codes; const uint32_t* valid; const int32_t* cell_block_start; const int64_t* cell_start;
  const int64_t* cell_size;
  const float* lut_scan;          // [nq_chunk][MG][256][64] (staged-LUT variant, DSUB == 0)
  const float* x;                 // [d, nq] queries (in-CTA LUT variant)
  const float* cbt;               // pq_codebook_t [256, MP, dsub]
  const float* part2_scan;        // residual: [C][MG][256][64] per-cell half of the LUT
  const float* base_sims;         // residual: [nq, n_probe] coarse similarities
  int M, metric;
  const int64_t* cells;           // [nq, n_probe]
  const int64_t* n_probe_list;    // [nq]
  uint64_t* keys_out;             // [nq, S, k]
  uint64_t* peer_keys[8];         // fused exchange: every rank's gather buffer [world, nq, k] (NVLink peer memory)
  int n_peers, peer_slot;         // n_peers == 0: keys go to keys_out
  int nq, q_base, n_probe, k, kp, S;
  int boot_r;                     // blocks per warp in the bootstrap (1 or 2)
  int n_cells;                    // probe entries outside [0, n_cells) are treated as empty segments
  const int* only_cnt;            // non-null: scan only the chunk's queries qi with only_cnt[qi] > only_cap (cell-major overflow)
  int only_cap;
#ifdef TPQ_DEBUG_KNOBS
  unsigned long long* phase;      // [16]; [0..4] summed clock64 deltas: prologue, bootstrap, scan, drain; [4] = CTAs
  int boot_mode;                  // 1 = merge-tree bootstrap (A/B against the quick start)
#endif
};

// The CTA's sorted top-k keys leave the SM here.  Fused exchange (n_peers > 0, dist.py): instead of a local buffer that an
// NCCL all-gather would then copy, the CTA stores its k keys straight into slot `peer_slot` of EVERY rank's gather buffer
// over NVLink (coalesced 8-byte stores, k * 8 B per peer), so the transfer overlaps the scans still running; a
// symmetric-memory barrier and the merge kernel follow.
template <int NW>
__device__ __forceinline__ void write_keys(const ScanArgs& A, const uint64_t* list, int q, int slice, int tid) {
  if (A.n_peers > 0) {
    const size_t o = ((size_t)A.peer_slot * A.nq + q) * A.k;
    for (int p = 0; p < A.n_peers; ++p) {
      uint64_t* out = A.peer_keys[p] + o;
      for (int i = tid; i < A.k; i += NW * 32) out[i] = list[i];
    }
    return;
  }
  uint64_t* out = A.keys_out + ((size_t)q * A.S + slice) * A.k;
  for (int i = tid; i < A.k; i += NW * 32) out[i] = list[i];
}

// The start of a query-major CTA, before its first barrier: warp 0 lays out the query's probe segments (their dependent
// global loads overlap the other warps' LUT work; visiting rule: probe_entry, scan_layout.cuh) while the CTA stages or
// builds the LUT (CU: build_lut's unroll).  Returns P, the probe entries the query visits.
template <int MP, int NW, int DSUB, bool RES, int CU = (DSUB >= 8 ? 2 : 8)>
__device__ __forceinline__ int scan_prologue(const ScanArgs& A, const ScanSmem& L, uint8_t* smem, int qi, int q, int tid,
                                             int lane, int warp) {
  constexpr int MG = lut_groups(MP);
  uint8_t* lut = smem;                                       // L.lut == 0 by construction
  int32_t*  seg_blk0   = reinterpret_cast<int32_t*>(smem + L.seg_blk0);
  uint32_t* seg_addr0  = reinterpret_cast<uint32_t*>(smem + L.seg_addr0);
  int32_t*  seg_prefix = reinterpret_cast<int32_t*>(smem + L.seg_prefix);
  const int P = probe_count<RES>(A.n_probe_list[q], A.n_probe);
  int32_t* seg_cell = reinterpret_cast<int32_t*>(smem + L.seg_cell);
  if (warp == 0) {
    int carry = 0;
    if (lane == 0) seg_prefix[0] = 0;
    const int64_t* cq = A.cells + (size_t)q * A.n_probe;
    for (int j0 = 0; j0 < P; j0 += 32) {
      const int j = j0 + lane;
      int nb = 0;
      if (j < P) {
        const ProbeEntry e = probe_entry(cq, j, A.n_cells, A.cell_start, A.cell_size, A.cell_block_start);
        nb = e.nb;
        seg_blk0[j] = e.blk0;
        seg_addr0[j] = e.addr0;
        if constexpr (RES) seg_cell[j] = (int32_t)e.cell;
      }
      const int incl = warp_inclusive_scan(nb, lane);
      if (j < P) seg_prefix[j + 1] = carry + incl;
      carry += __shfl_sync(0xffffffffu, incl, 31);
    }
  }
  if constexpr (DSUB == 0 && RES) {
    // residual with a staged query half: part1 stays in global memory (L2) and is added to part2 cell by cell
  } else if constexpr (DSUB == 0) {
    // --- stage LUT (MG * 64 KB, coalesced 16-byte copies)
    const float4* src = reinterpret_cast<const float4*>(A.lut_scan + (size_t)qi * MG * kLutGroup);
    float4* dst = reinterpret_cast<float4*>(lut);
    #pragma unroll 4
    for (int i = tid; i < MG * kLutGroup / 4; i += NW * 32) dst[i] = __ldg(src + i);
  } else {
    // --- build the LUT in place (or, RES, the query half of the residual LUT)
    build_lut<MP, NW, DSUB, RES, CU>(reinterpret_cast<float*>(RES ? smem + L.part1 : lut), A.x, A.cbt, A.M, A.nq, q,
                                     A.metric, lane, warp);
  }
  return P;
}

// Residual IVFPQ's scan of blocks [b_begin, b_end): the CTA walks the visited cells in lock step, re-forms the LUT as
// part1 + part2 of the cell, seeds every score with the cell's coarse similarity, and runs the Scanner over the cell's
// blocks.  Called by every thread after the prologue's barrier.
template <int MP, int NW, int DSUB, class Sc>
__device__ __forceinline__ void residual_walk(Sc& sc, const ScanArgs& A, const ScanSmem& L, uint8_t* smem, int P,
                                              int b_begin, int b_end, int q, int qi, int tid) {
  constexpr int MG = lut_groups(MP);
  const int32_t* seg_prefix = reinterpret_cast<const int32_t*>(smem + L.seg_prefix);
  const int32_t* seg_cell = reinterpret_cast<const int32_t*>(smem + L.seg_cell);
  // query half of the LUT: the shared-memory table built by the prologue (DSUB > 0), or the staged copy in global memory
  const float4* p1 = DSUB > 0 ? reinterpret_cast<const float4*>(smem + L.part1)
                              : reinterpret_cast<const float4*>(A.lut_scan + (size_t)qi * MG * kLutGroup);
  float4* dst = reinterpret_cast<float4*>(smem);
  for (int j = 0; j < P; ++j) {
    const int b0 = max(seg_prefix[j], b_begin), b1 = min(seg_prefix[j + 1], b_end);
    if (b1 <= b0) continue;                                          // skipped entry, empty cell, another shard's or slice's blocks
    __syncthreads();                                                 // every warp is done with the previous cell's LUT
    if (tid == 0) *sc.next = b0;
    const float4* p2 = reinterpret_cast<const float4*>(A.part2_scan + (size_t)seg_cell[j] * MG * kLutGroup);
    #pragma unroll 4
    for (int i = tid; i < MG * kLutGroup / 4; i += NW * 32) {                 // store_precomputed_to_smem: part1 + part2 (:609-628)
      const float4 a = DSUB > 0 ? p1[i] : __ldg(p1 + i), b = __ldg(p2 + i);
      dst[i] = make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
    }
    __syncthreads();
    sc.base = A.base_sims[(size_t)q * A.n_probe + j];
    sc.run(b1);
  }
}

// DSUB > 0: the CTA builds its query's LUT itself (build_lut, lut.cuh) from the (L2-resident) transposed codebook -- no
// LUT round trip through HBM, no LUT workspace.  DSUB == 0: the LUT was staged by lut_kernel (lut.cu) and is copied in.
// RES: residual IVFPQ (ivfpq_topk_residual_precomputed, ivfpq_topk.cu:1039-1207).  The LUT of a (query, cell) pair
// is part1[query] + part2[cell]: the query half is built once into a second shared-memory table, and the CTA
// walks the probed cells in lock step, re-forming the LUT (one float4 add per 16 bytes) before each cell; the
// cell's coarse similarity seeds every score.
template <int MP, int NW, int MINB, int DSUB, bool RES>
__global__ void __launch_bounds__(NW * 32, MINB)
ivfpq_scan_kernel(ScanArgs A, ScanSmem L) {
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* lut = smem;                                       // L.lut == 0 by construction
  int32_t*  seg_blk0   = reinterpret_cast<int32_t*>(smem + L.seg_blk0);
  uint32_t* seg_addr0  = reinterpret_cast<uint32_t*>(smem + L.seg_addr0);
  int32_t*  seg_prefix = reinterpret_cast<int32_t*>(smem + L.seg_prefix);

  const int qi = blockIdx.x / A.S, slice = blockIdx.x % A.S;  // query within this chunk
  const int q = A.q_base + qi;
  if (A.only_cnt && A.only_cnt[qi] <= A.only_cap) return;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
#ifdef TPQ_DEBUG_KNOBS
  long long t_ph = clock64();
#endif

  const int P = scan_prologue<MP, NW, DSUB, RES>(A, L, smem, qi, q, tid, lane, warp);
#ifdef TPQ_DEBUG_KNOBS
  auto phase_mark = [&](int i) {
    if (A.phase && tid == 0) { const long long t = clock64(); atomicAdd(A.phase + i, (unsigned long long)(t - t_ph)); t_ph = t; }
  };
#define TPQ_PHASE(i) phase_mark(i)
#else
#define TPQ_PHASE(i) ((void)0)
#endif
  Scanner<MP, NW> sc;
  sc.codes = A.codes; sc.valid = A.valid; sc.lut = lut;
  sc.seg_prefix = seg_prefix; sc.seg_blk0 = seg_blk0; sc.seg_addr0 = seg_addr0; sc.lane = lane;
  sc.next = reinterpret_cast<int*>(smem + L.next);
  sc.tk.init(smem + L.topk, NW, warp, A.kp, A.k);
  lane_slot_offsets(sc.off, lane);
  __syncthreads();
  TPQ_PHASE(0);

  const int total = seg_prefix[P];
  const int b_begin = (int)(((int64_t)total * slice) / A.S);
  const int b_end = (int)(((int64_t)total * (slice + 1)) / A.S);
  sc.thr = 0; sc.base = 0.f;
  sc.seg = 0; sc.seg_lo = 0; sc.seg_hi = seg_prefix[1]; sc.seg_b0 = seg_blk0[0]; sc.seg_a0 = seg_addr0[0];
  CtaTopK& tk = sc.tk;
  if constexpr (RES) {
    residual_walk<MP, NW, DSUB>(sc, A, L, smem, P, b_begin, b_end, q, qi, tid);
    tk.cta_drain(lane, warp);
    write_keys<NW>(A, tk.list, q, slice, tid);
    return;
  }
  // bootstrap: the first R blocks of every warp, sorted in registers per warp, give the threshold a lower bound after
  // one barrier (cta_quickstart) without R * NW lock-serialised flushes.  The merge tree (cta_bootstrap) exists only in
  // the debug build, where it is the default.
  const int R = A.boot_r;
  if (tid == 0) *sc.next = b_begin + R * NW;                    // the bootstrap's barriers publish it
  {
    #pragma unroll 1
    for (int r = 0; r < R; ++r) {
      const int b = b_begin + warp + r * NW;
      tk.buf[r * 32 + lane] = (b < b_end) ? sc.key_of_block(b) : 0ull;
    }
    tk.cnt = R * 32;
#ifdef TPQ_DEBUG_KNOBS
    if (A.boot_mode == 1) tk.cta_bootstrap(NW, R, lane, warp); else
#endif
    tk.cta_quickstart(NW, R, lane, warp);
  }
  TPQ_PHASE(1);
  sc.run(b_end);
  TPQ_PHASE(2);
  tk.cta_drain(lane, warp);                                // leftovers of all warps: register sorts + merge tree, no lock
  TPQ_PHASE(3);
#ifdef TPQ_DEBUG_KNOBS
  if (A.phase && tid == 0) atomicAdd(A.phase + 4, 1ull);
#endif
  write_keys<NW>(A, tk.list, q, slice, tid);
}
#undef TPQ_PHASE

// The range search's query-major kernel: ivfpq_scan_kernel's CTA per (query, slice), its prologue, residual walk and
// Scanner, with every live score above R.t kept instead of a top-k.  Each warp stages its matches in its own
// kRangeWarpBuf keys (range.cuh), in the shared memory the top-k of a k = 1 search takes (scan_smem's topk), and
// flushes them itself.
template <int MP, int NW, int MINB, int DSUB, bool RES>
__global__ void __launch_bounds__(NW * 32, MINB)
ivfpq_range_kernel(ScanArgs A, ScanSmem L, const __grid_constant__ RangeOut R) {
  extern __shared__ __align__(1024) uint8_t smem[];
  static_assert((size_t)NW * kRangeWarpBuf * 8 <= CtaTopK::bytes(NW, 32), "a warp's range buffer lies in the k = 1 top-k's place");
  const int qi = blockIdx.x / A.S, slice = blockIdx.x % A.S;
  const int q = A.q_base + qi;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  int32_t* seg_blk0 = reinterpret_cast<int32_t*>(smem + L.seg_blk0);
  uint32_t* seg_addr0 = reinterpret_cast<uint32_t*>(smem + L.seg_addr0);
  int32_t* seg_prefix = reinterpret_cast<int32_t*>(smem + L.seg_prefix);
  // the LUT build of ivfpq_scan_kernel<192, 16, 1, 4, false> spills; here its codebook loop is unrolled 4 times, not 8
  constexpr int CU = (MP == 192 && DSUB == 4) ? 4 : (DSUB >= 8 ? 2 : 8);
  const int P = scan_prologue<MP, NW, DSUB, RES, CU>(A, L, smem, qi, q, tid, lane, warp);
  Scanner<MP, NW, true> sc;
  sc.codes = A.codes; sc.valid = A.valid; sc.lut = smem;
  sc.seg_prefix = seg_prefix; sc.seg_blk0 = seg_blk0; sc.seg_addr0 = seg_addr0; sc.lane = lane;
  sc.next = reinterpret_cast<int*>(smem + L.next);
  sc.rs = RangeWarpBuf{reinterpret_cast<uint64_t*>(smem + L.topk) + (size_t)warp * kRangeWarpBuf, 0, q, &R};
  lane_slot_offsets(sc.off, lane);
  __syncthreads();
  const int total = seg_prefix[P];
  const int b_begin = (int)(((int64_t)total * slice) / A.S);
  const int b_end = (int)(((int64_t)total * (slice + 1)) / A.S);
  sc.base = 0.f;
  sc.seg = 0; sc.seg_lo = 0; sc.seg_hi = seg_prefix[1]; sc.seg_b0 = seg_blk0[0]; sc.seg_a0 = seg_addr0[0];
  if constexpr (RES) {
    residual_walk<MP, NW, DSUB>(sc, A, L, smem, P, b_begin, b_end, q, qi, tid);
  } else {
    if (tid == 0) *sc.next = b_begin;
    __syncthreads();
    sc.run(b_end);
  }
  sc.rs.flush(lane);                                       // what is left when the warp runs out of blocks
}


// ----------------------------------------------------------------------------- merge + decode
// keys_in: n_parts sorted lists of k keys per query -> top-k, decoded.
// One warp per query.  (Cross-slice merge for small batches and cross-shard merge after the
// all-gather; with n_parts == 1 it is just the decode + get_id_by_address, BaseContainer.py:58-65.)
__global__ void __launch_bounds__(128)
merge_topk_kernel(const uint64_t* __restrict__ keys_in, int nq, int n_parts, int k, int kp,
                  int64_t part_stride, int64_t query_stride,
                  const int64_t* __restrict__ address2id, int64_t capacity,
                  float* __restrict__ values, int64_t* __restrict__ ids, int64_t* __restrict__ address,
                  uint64_t* __restrict__ keys_out) {
  extern __shared__ __align__(16) uint8_t smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int q = blockIdx.x * (blockDim.x >> 5) + warp;
  if (q >= nq) return;
  uint64_t* A = reinterpret_cast<uint64_t*>(smem) + (size_t)warp * 2 * kp;
  uint64_t* Bf = A + kp;
  const uint64_t* src = keys_in + (size_t)q * query_stride;
  for (int i = lane; i < kp; i += 32) A[i] = i < k ? src[i] : 0ull;
  __syncwarp();
  for (int p = 1; p < n_parts; ++p) {
    const uint64_t* sp = src + (size_t)p * part_stride;
    for (int i = lane; i < kp; i += 32) Bf[i] = i < k ? sp[i] : 0ull;
    __syncwarp();
    warp_merge_desc(A, kp, Bf, kp, lane);
  }
  for (int i = lane; i < k; i += 32) {
    const uint64_t key = A[i];
    const size_t o = (size_t)q * k + i;
    const int64_t a = key ? (int64_t)key_addr(key) : -1;
    if (values) values[o] = key ? key_score(key) : -INFINITY;
    if (address) address[o] = a;
    if (ids) ids[o] = (a >= 0 && a < capacity) ? address2id[a] : -1;
    if (keys_out) keys_out[o] = key;
  }
}

static int launch_merge(const uint64_t* keys_in, int nq, int n_parts, int k, int64_t part_stride, int64_t query_stride,
                        const int64_t* address2id, int64_t capacity, float* values, int64_t* ids, int64_t* address,
                        uint64_t* keys_out, cudaStream_t st) {
  const int kp = list_capacity(k);
  const int wpb = 4;
  size_t smem = (size_t)wpb * 2 * kp * 8;
  TPQ_CUDA(cudaFuncSetAttribute(merge_topk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  merge_topk_kernel<<<(nq + wpb - 1) / wpb, wpb * 32, smem, st>>>(keys_in, nq, n_parts, k, kp, part_stride, query_stride,
                                                                 address2id, capacity, values, ids, address, keys_out);
  TPQ_LAUNCH_CHECK("merge_topk_kernel");
  return TPQ_OK;
}

// ----------------------------------------------------------------------------- cell-major scan (M <= 64, large cells)
// The query-major kernel reads a probed cell's codes once per (query, cell) pair: at 2441 vectors per cell that is
// 156 KB per pair against a 64 KB LUT.  The cell-major path turns the loop around: a CTA holds a chunk of one cell's
// code blocks in registers and the LUTs of the queries probing that cell stream past it, so a pair costs one LUT read.
//   pass 1  the query-major kernel on each query's first probe entry -> its sorted top-k; key k-1 bounds the query
//           (0 when that cell has fewer than k live vectors);
//   pass 2  ivfpq_cell_scan_kernel over entries 1 .. P-1: every key above the bound is appended to the query's survivors;
//   select  per query, the top k of the pass-1 list and the survivors (cell_select_kernel).
// Exact: a candidate that is neither in the pass-1 list nor a survivor is <= the bound, and the pass-1 list already
// holds k keys >= the bound.  Both kernels form their keys in block_key, so results are bit-identical.
constexpr int kCellSlots = 3;         // LUT ring depth (64 KB each)
constexpr int kCellNW = 12;           // warps of a cell-scan CTA
constexpr int kCellR = 7;             // code blocks per warp held in registers (168 registers): a chunk is up to 84 blocks = 2688 vectors
constexpr int kCellWin = 256;         // pairs of an item whose (query, bound) records sit in shared memory at a time
// Dynamic shared memory of a cell-scan CTA: the ring, 256 B of barriers and slot state, the warps' survivor stages, then
// the record window (kCellWin bounds, kCellWin queries, kCellWin survivor counts, kCellWin reserved bases).
constexpr size_t cell_win_offset(int nw, int r) { return (size_t)kCellSlots * lut_bytes(64) + 256 + (size_t)nw * r * 32 * 8; }
constexpr size_t cell_smem_bytes(int nw, int r) { return cell_win_offset(nw, r) + (size_t)kCellWin * 20; }
// Survivor log of a cell-scan CTA: one bucket per pair of the window, each as large as a chunk's keys can be.
constexpr size_t cell_log_keys(int nw, int r) { return (size_t)kCellWin * nw * r * 32; }

// Shared-memory accesses of the record window, by 32-bit shared address.  The window is kept apart from the pointers the
// compiler derives from the kernel's shared base, and the pair body keeps reading its bound from the slot's fixed word
// (its only indexed access is the atomic on its survivor count, through these opaque addresses): indexed reads of the window in the pair body made ptxas move that base from a uniform register into a
// vector register and add it to every lookup's address (4.2 instead of 3.3 instructions per lookup, sass_census.py).
__device__ __forceinline__ uint32_t lds_u32(uint32_t a) { uint32_t v; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a) : "memory"); return v; }
__device__ __forceinline__ uint64_t lds_u64(uint32_t a) { uint64_t v; asm volatile("ld.shared.u64 %0, [%1];" : "=l"(v) : "r"(a) : "memory"); return v; }
__device__ __forceinline__ void sts_u32(uint32_t a, uint32_t v) { asm volatile("st.shared.u32 [%0], %1;" :: "r"(a), "r"(v) : "memory"); }
__device__ __forceinline__ void sts_u64(uint32_t a, uint64_t v) { asm volatile("st.shared.u64 [%0], %1;" :: "r"(a), "l"(v) : "memory"); }
__device__ __forceinline__ uint32_t atoms_add_u32(uint32_t a, uint32_t v) {
  uint32_t old;
  asm volatile("atom.shared.add.u32 %0, [%1], %2;" : "=r"(old) : "r"(a), "r"(v) : "memory");
  return old;
}
constexpr int kCellBuckets = 128;     // work classes of the largest-first item order (4 per octave)

struct CellItem { int32_t cell, b_lo, b_hi, pad; };   // blocks [b_lo, b_hi) of the cell (relative to its first block)

struct CellArgs {
  const uint8_t* codes; const uint32_t* valid; const int32_t* cell_block_start; const int64_t* cell_start;
  const float* lut_scan;          // [n][256][64] LUTs of this chunk's queries (cell_lut_kernel)
  const int32_t* cell_off;        // [C] first pair of each cell in pair_q
  const int32_t* cell_cnt;        // [C] pairs per cell
  const int32_t* pair_q;          // chunk-local query of each pair, grouped by cell
  const CellItem* items; const int* n_items; int* cursor;
  const uint64_t* keys;           // [nq][k] pass-1 lists; key k-1 is the query's bound
  uint64_t* surv; int* surv_cnt;  // [n][cap] survivors, [n] their count (> cap: overflow), by chunk-local query
  uint64_t* log;                  // [gridDim.x][kCellWin][NW * R * 32]: each CTA's survivors of a window, by pair
  int q_base, k, cap;
#ifdef TPQ_DEBUG_KNOBS
  unsigned long long* phase;      // the phase buffer's [8..15]: warp-cycles summed over all warps in item prologue (barrier,
                                  // code loads, first LUT wait), mbar_wait, scoring, release + issue, pair tail (shared
                                  // reservation + log copy), window flush; [14] = warps, [15] = their cycles from kernel
                                  // entry to exit
  int ablate;                     // WRONG RESULTS, to bound a gain: bit 0 = no refills (every pair of an item reuses the
                                  // first kCellSlots LUTs), bit 1 = no survivors (thr = ~0)
#endif
};

// thread per (query, entry): count the visited pairs of entries 1 .. P-1 per cell; slot = the pair's rank in its cell
__global__ void cell_pairs_count_kernel(const int64_t* __restrict__ cells, const int64_t* __restrict__ npl, int q_base, int n,
                                        int n_probe, int n_cells, const int64_t* __restrict__ cell_start,
                                        const int64_t* __restrict__ cell_size, const int32_t* __restrict__ cbs,
                                        int* __restrict__ cell_cnt, int* __restrict__ slot, int64_t* __restrict__ ones) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (int64_t)n * n_probe) return;
  const int qi = (int)(t / n_probe), j = (int)(t % n_probe);
  const int q = q_base + qi;
  if (j == 0) ones[q] = 1;                                     // pass 1 scans entry 0 only
  int pos = -1;
  if (j >= 1 && j < probe_count<false>(npl[q], n_probe)) {
    const ProbeEntry e = probe_entry(cells + (size_t)q * n_probe, j, n_cells, cell_start, cell_size, cbs);
    if (e.nb > 0) pos = atomicAdd(cell_cnt + e.cell, 1);
  }
  slot[t] = pos;
}

__global__ void cell_pairs_scatter_kernel(const int64_t* __restrict__ cells, int q_base, int n, int n_probe,
                                          const int* __restrict__ slot, const int* __restrict__ cell_off,
                                          int* __restrict__ pair_q) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (int64_t)n * n_probe) return;
  const int s = slot[t];
  if (s < 0) return;
  const int qi = (int)(t / n_probe);
  pair_q[cell_off[cells[(size_t)(q_base + qi) * n_probe + t % n_probe]] + s] = qi;
}

// One CTA: cell_off = exclusive prefix of cell_cnt; work items = chunks of at most `chunk` blocks of every cell with
// pairs, ordered by work (pairs x blocks) descending in classes of 4 per octave, the chunks of one cell adjacent.
__global__ void __launch_bounds__(1024) cell_plan_kernel(const int* __restrict__ cell_cnt, const int32_t* __restrict__ cbs,
                                                         const int64_t* __restrict__ cell_size, int n_cells,
                                                         int chunk, int* __restrict__ cell_off,
                                                         CellItem* __restrict__ items, int* __restrict__ n_items) {
  __shared__ int hist[kCellBuckets], base[kCellBuckets], warp_sum[32], carry;
  const int tid = threadIdx.x;
  for (int i = tid; i < kCellBuckets; i += 1024) hist[i] = 0;
  if (tid == 0) carry = 0;
  __syncthreads();
  auto chunks_of = [&](int c, int& nb, int& bucket) {
    nb = cell_blocks(cbs[c], cbs[c + 1], cell_size[c]);
    const int np = cell_cnt[c];
    if (np == 0 || nb == 0) { nb = 0; return 0; }
    const int nch = (nb + chunk - 1) / chunk;
    const uint32_t w = (uint32_t)np * (uint32_t)((nb + nch - 1) / nch);
    const int lg = 31 - __clz(w);
    const int sub = lg >= 2 ? (int)((w >> (lg - 2)) & 3u) : (int)((w << (2 - lg)) & 3u);
    bucket = kCellBuckets - 1 - min(kCellBuckets - 1, 4 * lg + sub);   // larger work -> smaller bucket index
    return nch;
  };
  for (int c0 = 0; c0 < n_cells; c0 += 1024) {
    const int c = c0 + tid;
    const int v = c < n_cells ? cell_cnt[c] : 0;
    const int incl = cta_inclusive_scan(v, warp_sum, carry);
    if (c < n_cells) {
      cell_off[c] = incl - v;
      int nb, b;
      const int nch = chunks_of(c, nb, b);
      if (nch) atomicAdd(&hist[b], nch);
    }
  }
  __syncthreads();
  if (tid == 0) {
    int s = 0;
    for (int b = 0; b < kCellBuckets; ++b) { base[b] = s; s += hist[b]; }
    *n_items = s;
  }
  __syncthreads();
  for (int c = tid; c < n_cells; c += 1024) {
    int nb, b;
    const int nch = chunks_of(c, nb, b);
    if (!nch) continue;
    const int pos = atomicAdd(&base[b], nch);
    for (int j = 0; j < nch; ++j)
      items[pos + j] = CellItem{c, (int)((int64_t)nb * j / nch), (int)((int64_t)nb * (j + 1) / nch), 0};
  }
}

// Persistent: a CTA takes items (cell, chunk) from a global cursor.  Warp w holds blocks w, w + NW, ... of the chunk
// (R at most) in registers.  The LUTs of the pairs of the cell arrive by TMA into a ring of kCellSlots 64 KB slots; the
// last warp to finish with a slot refills it, so no warp waits for another except through the ring.  Per block the
// scoring is the query-major kernel's adc_unit, so a key is the same bit for bit.  Each lookup is PRMT + LDS + FADD, as
// in the query-major kernel: the pair body is compiled once per ring slot, so the slot's offset is an LDS immediate
// and the shared-window base a uniform register (scripts/sass_census.py counts it).
// Survivors leave in two steps.  A warp appends its keys of pair i to bucket i of the CTA's log at an offset from a
// shared-memory count, with stores that return nothing.  After the window's last pair, the CTA reserves each pair's
// place in its query's survivor list with one global atomic per pair, all issued together, and copies the buckets there.
template <int NW, int R>
__global__ void __launch_bounds__(NW * 32, 1)
ivfpq_cell_scan_kernel(CellArgs A) {
  constexpr int MP = 64;
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* ring = smem;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + kCellSlots * lut_bytes(64));
  uint64_t* slot_thr = full + kCellSlots;
  int* rel = reinterpret_cast<int*>(slot_thr + kCellSlots);   // warps done with the slot's current LUT
  int* item_sh = rel + kCellSlots;                             // [2]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  uint64_t* stage = reinterpret_cast<uint64_t*>(smem + kCellSlots * lut_bytes(64) + 256) + (size_t)warp * R * 32;
  uint32_t win_thr = smem_u32(smem + cell_win_offset(NW, R));
  asm volatile("" : "+r"(win_thr));                            // from here on just a number to the compiler (see lds_u32)
  const uint32_t win_q = win_thr + kCellWin * 8;
  const uint32_t win_cnt = win_q + kCellWin * 4;               // survivors of each pair of the window, in its log bucket
  const uint32_t win_base = win_cnt + kCellWin * 4;            // their place in the query's survivor list
  constexpr int kBucket = NW * R * 32;                         // a chunk's keys: a bucket never overflows
  static_assert(kCellWin <= NW * 32, "one thread per record of the window");
  if (tid == 0) {
    for (int s = 0; s < kCellSlots; ++s) { mbar_init(&full[s], 1); rel[s] = 0; }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (tid < kCellWin) sts_u32(win_cnt + 4 * tid, 0u);         // the item loop's first barrier publishes it
#ifdef TPQ_DEBUG_KNOBS
  // per-warp cycle account, kept in shared memory behind the stages (the kernel has no registers to spare)
  unsigned long long* acct = reinterpret_cast<unsigned long long*>(smem + cell_smem_bytes(NW, R)) + warp * 8;
  const bool no_refill = A.ablate & 1, no_surv = A.ablate & 2;
  const uint32_t t_in = (uint32_t)clock();
  uint32_t t_ph = t_in;
  if (A.phase && lane < 8) acct[lane] = 0;
  __syncwarp();
  auto cell_mark = [&](int ph) {
    if (A.phase) { const uint32_t t = (uint32_t)clock(); if (lane == 0) acct[ph] += t - t_ph; t_ph = t; }
  };
#define TPQ_CELL_PHASE(ph) cell_mark(ph)
#else
  constexpr bool no_refill = false, no_surv = false;
#define TPQ_CELL_PHASE(ph) ((void)0)
#endif
  uint32_t off[8];
  lane_slot_offsets(off, lane);
  // one thread: LUT of pair i of the window into slot s (every warp has released the slot), its bound into the slot's
  // word.
  // It reads shared memory only: the thread that refills a slot is the last to leave it, and every warp waits for
  // what it waits for here.
  auto issue = [&](int i, int s) {
    const int qi = (int)lds_u32(win_q + 4 * i);
    slot_thr[s] = lds_u64(win_thr + 8 * i);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // the warps' reads of the slot precede the TMA write
    mbar_expect_tx(&full[s], lut_bytes(64));
    bulk_load(ring + s * lut_bytes(64), A.lut_scan + (size_t)qi * kLutGroup, lut_bytes(64), &full[s]);
  };
  uint32_t parity = 0;                                         // bit s: phase parity of slot s's next fill
  const int n_items = *A.n_items;
  for (int it = 0;; ++it) {
    if (tid == 0) item_sh[it & 1] = atomicAdd(A.cursor, 1);
    __syncthreads();                                           // also: every warp is done with the previous item
    const int item = item_sh[it & 1];
    if (item >= n_items) break;
    const CellItem ci = A.items[item];
    const int np = A.cell_cnt[ci.cell];
    const int32_t* pq = A.pair_q + A.cell_off[ci.cell];
    // Pair i of every item uses slot i % kCellSlots: the ring is drained at the barrier above, so it can restart at
    // slot 0, and each pair body below is compiled for its slot (the slot's offset is an LDS immediate).
    const int b0 = A.cell_block_start[ci.cell];
    const uint32_t a0 = (uint32_t)A.cell_start[ci.cell];
    // blocks of this warp (may be <= 0); broadcast from lane 0 so that the compiler knows it is warp-uniform and the
    // `r < nr` branches need no divergence handling around the ballots
    const int nr = __shfl_sync(0xffffffffu, (ci.b_hi - ci.b_lo - warp + NW - 1) / NW, 0);
    uint32_t w[R][16], vmask[R];
    #pragma unroll
    for (int r = 0; r < R; ++r) {
      if (r < nr) {
        const int64_t B = (int64_t)b0 + ci.b_lo + warp + r * NW;
        load_unit<MP, 0>(w[r], A.codes, B, lane);
        vmask[r] = __ldg(A.valid + B);
      }
    }
    auto pair = [&](auto slot, int i, int np) {                // pair i of the window's np, in ring slot `slot`
      constexpr int s = decltype(slot)::value;
      if (!no_refill || i < kCellSlots) {                      // no refills: the slot was armed once, at the item's start
        mbar_wait(&full[s], (parity >> s) & 1u);
        parity ^= 1u << s;
      }
      TPQ_CELL_PHASE(i == 0 ? 0 : 1);
      const uint64_t thr = no_surv ? ~0ull : slot_thr[s];
      const uint8_t* lut = ring + s * lut_bytes(64);
      int n = 0;
      #pragma unroll
      for (int r = 0; r < R; ++r) {
        if (r < nr) {
          float acc[4] = {0.f, 0.f, 0.f, 0.f};
          adc_unit<MP, 0>(w[r], off, lut, acc);
          // base -0.f: x + -0.f is x, so no add is issued.  The query-major kernel adds +0.f here, which is the same
          // score: a sum of partial sums that start from +0.f is never -0.f.
          const uint64_t key = block_key(acc, -0.f, a0 + (uint32_t)(ci.b_lo + warp + r * NW) * 32u, lane);
          n += warp_append(stage, n, ((vmask[r] >> lane) & 1u) && key > thr, key, lane);
        }
      }
      __syncwarp();
      TPQ_CELL_PHASE(2);
      if (lane == 0) {                                         // release the slot; the last warp refills it
        int old;
        asm volatile("atom.acq_rel.cta.shared::cta.add.u32 %0, [%1], 1;" : "=r"(old) : "r"(smem_u32(&rel[s])) : "memory");
        if (old == NW - 1) {
          rel[s] = 0;
          if (!no_refill && i + kCellSlots < np) issue(i + kCellSlots, s);
        }
      }
      TPQ_CELL_PHASE(3);
      if (n) {                                                 // into bucket i of the log; the window's flush reserves
        // the first 32 staged keys are read before the count is, so the two shared-memory round trips overlap
        const uint64_t k0 = lane < n ? stage[lane] : 0ull;
        uint32_t o = 0;
        if (lane == 0) o = atoms_add_u32(win_cnt + 4 * i, (uint32_t)n);
        o = __shfl_sync(0xffffffffu, o, 0);
        uint64_t* dst = A.log + ((size_t)blockIdx.x * kCellWin + i) * kBucket + o;
        if (lane < n) dst[lane] = k0;
        for (int j = lane + 32; j < n; j += 32) dst[j] = stage[j];
        __syncwarp();
      }
      TPQ_CELL_PHASE(4);
    };
    // After the window's last pair: one global atomic per pair with survivors reserves the pair's place in its query's
    // list, and the warps copy each bucket there unless its query has overflowed (surv_cnt ends at the same sum
    // whatever the order, so the same queries overflow).  The counts are zeroed for the next window.
    auto flush = [&](int nwin) {
      __syncthreads();                                         // every count final, every log store visible to the CTA
      if (tid < nwin) {
        const uint32_t c = lds_u32(win_cnt + 4 * tid);
        if (c) {
          const int b = atomicAdd(A.surv_cnt + lds_u32(win_q + 4 * tid), (int)c);
          if (b + (int)c <= A.cap) sts_u32(win_base + 4 * tid, (uint32_t)b);
          else sts_u32(win_cnt + 4 * tid, 0u);                 // overflowed: nothing to copy
        }
      }
      __syncthreads();
      // Warp w copies buckets w, w + NW, ...: the first 64 keys of U buckets are loaded before any is stored, so a warp
      // waits for U buckets' reads at once (at C3 a bucket holds about 60 keys).  The first bucket is broadcast from
      // lane 0, as nr is: a loop the compiler cannot prove warp-uniform leaves the next window's pair bodies possibly
      // diverged, and ptxas then adds the shared base to every lookup (4.2 instead of 3.35 instructions per lookup,
      // sass_census.py).
      constexpr int U = 2;
      for (int t0 = __shfl_sync(0xffffffffu, warp, 0); t0 < nwin; t0 += U * NW) {
        uint32_t c[U];
        uint64_t v[U][2];
        #pragma unroll
        for (int u = 0; u < U; ++u) {
          const int t = t0 + u * NW;
          c[u] = t < nwin ? lds_u32(win_cnt + 4 * t) : 0u;
          const uint64_t* src = A.log + ((size_t)blockIdx.x * kCellWin + t) * kBucket;
          v[u][0] = lane < c[u] ? src[lane] : 0ull;
          v[u][1] = lane + 32 < c[u] ? src[lane + 32] : 0ull;
        }
        #pragma unroll
        for (int u = 0; u < U; ++u) {
          const int t = t0 + u * NW;
          if (c[u] == 0) continue;
          const uint64_t* src = A.log + ((size_t)blockIdx.x * kCellWin + t) * kBucket;
          uint64_t* dst = A.surv + (size_t)lds_u32(win_q + 4 * t) * A.cap + lds_u32(win_base + 4 * t);
          if (lane < c[u]) dst[lane] = v[u][0];
          if (lane + 32 < c[u]) dst[lane + 32] = v[u][1];
          for (uint32_t j = lane + 64; j < c[u]; j += 32) dst[j] = src[j];
          __syncwarp();
          if (lane == 0) sts_u32(win_cnt + 4 * t, 0u);
        }
      }
      TPQ_CELL_PHASE(5);
    };
    static_assert(kCellSlots == 3, "one pair body per ring slot");
    for (int p0 = 0; p0 < np; p0 += kCellWin) {
      // the window's records: each pair's query and its bound, key k-1 of the query's pass-1 list
      const int nwin = min(np - p0, kCellWin);
      if (p0) __syncthreads();                                 // every warp is done with the previous window and the ring
      if (tid < nwin) {
        const int qi = pq[p0 + tid];
        sts_u32(win_q + 4 * tid, (uint32_t)qi);
        sts_u64(win_thr + 8 * tid, A.keys[(size_t)(A.q_base + qi) * A.k + A.k - 1]);
      }
      __syncthreads();
      if (tid == 0)
        for (int i = 0; i < min(nwin, kCellSlots); ++i) issue(i, i);
      for (int i = 0; i < nwin; i += kCellSlots) {
        pair(std::integral_constant<int, 0>(), i, nwin);
        if (i + 1 < nwin) pair(std::integral_constant<int, 1>(), i + 1, nwin);
        if (i + 2 < nwin) pair(std::integral_constant<int, 2>(), i + 2, nwin);
      }
      if (!no_surv) flush(nwin);                               // no survivors: every count is 0
    }
  }
#ifdef TPQ_DEBUG_KNOBS
  cell_mark(0);                                                // the wait at the last barrier
  if (A.phase && lane == 0) {
    for (int ph = 0; ph < 6; ++ph) atomicAdd(A.phase + ph, acct[ph]);
    atomicAdd(A.phase + 6, 1ull);
    atomicAdd(A.phase + 7, (unsigned long long)((uint32_t)clock() - t_in));
  }
#endif
#undef TPQ_CELL_PHASE
}

// CTA per query: its LUT in scan layout into global memory, as the query-major kernel builds it in shared memory
template <int DSUB>
__global__ void __launch_bounds__(256) cell_lut_kernel(const float* __restrict__ x, const float* __restrict__ cbt, int M,
                                                       int nq, int q_base, int metric, float* __restrict__ lut) {
  build_lut<64, 8, DSUB, false>(lut + (size_t)blockIdx.x * kLutGroup, x, cbt, M, nq, q_base + blockIdx.x, metric,
                                threadIdx.x & 31, threadIdx.x >> 5);
}

// warp per query: keys[q] <- top k of keys[q] (the pass-1 list) and the survivors; overflowed queries are left to the
// query-major re-run
__global__ void __launch_bounds__(128) cell_select_kernel(uint64_t* __restrict__ keys, const uint64_t* __restrict__ surv,
                                                          const int* __restrict__ surv_cnt, int q_base, int n, int k,
                                                          int kp, int cap) {
  extern __shared__ __align__(16) uint8_t smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int qi = blockIdx.x * 4 + warp;
  if (qi >= n) return;
  const int q = q_base + qi;
  const int ns = surv_cnt[qi];
  if (ns == 0 || ns > cap) return;
  uint64_t* list = reinterpret_cast<uint64_t*>(smem) + (size_t)warp * (kp + kTopkBuf);
  WarpTopK tk;
  tk.init(list, list + kp, kp, k, lane);
  uint64_t* kq = keys + (size_t)q * k;
  for (int i = lane; i < k; i += 32) list[i] = kq[i];
  __syncwarp();
  const uint64_t* sq = surv + (size_t)qi * cap;
  for (int i0 = 0; i0 < ns; i0 += 32) {
    const uint64_t key = i0 + lane < ns ? sq[i0 + lane] : 0ull;
    tk.push(key > tk.kth(), key, lane);
  }
  tk.flush(lane);
  __syncwarp();
  for (int i = lane; i < k; i += 32) kq[i] = list[i];
}

// ----------------------------------------------------------------------------- host orchestration
constexpr int kQueryChunk = 16384;    // queries per scan launch (bounds the LUT workspace: 64 KB * MG each)

// optional CUDA-event timing of the scan launches (bench.py's roofline leg); off by default
constexpr int kProfMax = 1024;
static bool g_prof_on = false;
static int g_prof_n = 0;
static cudaEvent_t g_prof_start[kProfMax], g_prof_stop[kProfMax];
static bool g_prof_created = false;

#ifdef TPQ_DEBUG_KNOBS
static unsigned long long* g_phase = nullptr;     // device buffer of 16 counters, set by tpq_debug_set_phase_buffer
#endif

constexpr int kCellMinLive = 1536;    // live vectors per cell, on average, from which the cell-major scan pays
// survivors kept per query; a query with more is scanned again by the query-major kernel
static int cell_cap(int k) { return k * 8 > 8192 ? k * 8 : 8192; }

struct SearchWs {
  size_t coarse, probe_sims, cells, npl, xnorm, lut, keys;
  size_t cell_cnt, cell_off, slot, pair_q, items, ones, surv, surv_cnt, cell_log;   // cell-major scan only
  size_t total;
};

// What a search of nq queries runs.  plan_scan is the only place that decides it; the workspace size, the launches and
// the three search entry points all read the plan.
struct ScanPlan {
  int S, chunk;                   // CTAs (slices) per query; queries per scan launch
  bool range;                     // range search: ivfpq_range_kernel, no keys workspace, never cell-major
  bool cell_major;               // the cell-major stage (ivfpq_cell_scan_kernel) instead of one query-major launch
  int dsub;                       // LUT source: d/M = 1, 2, 4 or 8 when built in the kernel (on the cell-major path:
                                  // by cell_lut_kernel), 0 = staged through global memory by lut_kernel
  bool residual, part1_in_smem;   // residual IVFPQ; its query half of the LUT in a second shared-memory table
  int MP, NW, MINB;               // the query-major kernel: ivfpq_scan_kernel<MP, NW, MINB, qm_dsub(), residual>
  int boot_r;                     // blocks per warp in the kernel's bootstrap
  int cell_nw, cell_r;            // the cell-major kernel: ivfpq_cell_scan_kernel<cell_nw, cell_r>
  int cell_ctas;                  // its persistent CTAs, one per SM; each has a survivor log in the workspace
#ifdef TPQ_DEBUG_KNOBS
  int boot_mode; unsigned long long* phase;
  int cell_ablate;
#endif
  ScanSmem L;                     // the query-major kernel's shared memory
  SearchWs ws;
  int rc; char err[160];          // rc != TPQ_OK: the configuration cannot run, and why
  // the query-major kernel's DSUB: on the cell-major path it reads the LUTs cell_lut_kernel left in the workspace
  int qm_dsub() const { return cell_major ? 0 : dsub; }
};

static SearchWs search_ws(const tpq_index* ix, int nq, int n_probe, int k, const ScanPlan& P) {
  SearchWs w; size_t off = 0;
  const bool cm = P.cell_major;
  w.coarse = off;     off += align_up(tpq_coarse_workspace_bytes(ix->d_vector, nq, ix->n_cells), 256);
  w.probe_sims = off; off += align_up((size_t)nq * n_probe * 4, 256);
  w.cells = off;      off += align_up((size_t)nq * n_probe * 8, 256);
  w.npl = off;        off += align_up((size_t)nq * 8, 256);
  w.xnorm = off;      off += align_up((size_t)nq * ix->d_vector * 4, 256);
  w.lut = off;        off += P.qm_dsub() ? 0 : align_up((size_t)P.chunk * lut_bytes(ix->m_pad), 256);
  w.keys = off;       off += P.range ? 0 : align_up((size_t)nq * P.S * k * 8, 256);
  const size_t C = cm ? (size_t)ix->n_cells : 0, pairs = cm ? (size_t)P.chunk * n_probe : 0;
  const size_t n_items = cm ? C + (size_t)ix->n_blocks / (P.cell_nw * P.cell_r) + 1 : 0;
  w.cell_cnt = off;   off += align_up((C + 2) * 4, 256);                  // pairs per cell, then the item count and cursor
  w.cell_off = off;   off += align_up(C * 4, 256);
  w.slot = off;       off += align_up(pairs * 4, 256);
  w.pair_q = off;     off += align_up(pairs * 4, 256);
  w.items = off;      off += align_up(n_items * sizeof(CellItem), 256);
  w.ones = off;       off += align_up(cm ? (size_t)nq * 8 : 0, 256);
  w.surv = off;       off += align_up(cm ? (size_t)P.chunk * cell_cap(k) * 8 : 0, 256);
  w.surv_cnt = off;   off += align_up(cm ? (size_t)P.chunk * 4 : 0, 256);
  // 5.5 MB per CTA at 12 x 7 (726 MB at 132 SMs): sized by the SM count, not by the batch
  w.cell_log = off;   off += align_up(cm ? (size_t)P.cell_ctas * cell_log_keys(P.cell_nw, P.cell_r) * 8 : 0, 256);
  w.total = off;
  return w;
}

// push: the fused-push path (tpq_ivfpq_scan_push), which keeps the query-major kernel.  range: range search
// (tpq_ivfpq_range_search, k = 1), the query-major kernel's slicing, chunking and configuration with
// ivfpq_range_kernel in its place; its shared memory is that of a k = 1 search.
static ScanPlan plan_scan(const tpq_index* ix, int nq, int n_probe, int k, bool push, bool range = false) {
  ScanPlan P{};
  P.range = range;
  const int dsub = ix->d_vector / ix->n_subvectors;
  const int want = device_sm_count() * 4;       // enough CTAs for ~2 waves of 2 CTAs/SM when the batch is small
  P.S = nq >= want ? 1 : ((want + nq - 1) / nq > 64 ? 64 : (want + nq - 1) / nq);
  P.chunk = nq < kQueryChunk ? nq : kQueryChunk;
  P.residual = ix->residual != 0;
  P.MP = ix->m_pad;
  P.boot_r = 2;
  P.cell_nw = kCellNW; P.cell_r = kCellR;
  P.cell_ctas = device_sm_count();
  // LUT source: built inside the scan CTA when d/M is 1, 2, 4 or 8 (the codebook slice a CTA reads from L2, M*dsub KB,
  // is then small next to the codes it goes on to stream: C4, d/M = 8, reads 0.98 MB of codebook per 7.5 MB of codes
  // and saves the 2 x 128 KB LUT round trip through HBM plus one launch); staged through HBM by lut_kernel
  // otherwise.  Residual IVFPQ keeps TWO tables when the query half is built in the CTA: that fits for M <= 64 and pays
  // for d/M <= 4.
  P.dsub = (dsub == 1 || dsub == 2 || dsub == 4 || dsub == 8) ? dsub : 0;
  if (P.residual && (P.MP > 64 || dsub == 8)) P.dsub = 0;
  if (P.residual || P.MP > 64) {
    // residual: one 16-warp CTA per SM; M > 64: the LUT is >= 128 KB, so one CTA per SM with twice the warps
    P.NW = 16; P.MINB = 1;
  } else if (P.MP == 64) {
    // Long probe lists: 2 CTAs/SM with a deep prefetch (127 registers).  Short ones (small cells, or one shard of a
    // cell-sharded index): per-CTA prologue/epilogue weighs more, so 3 lighter CTAs/SM overlap them better.
    const double blocks_per_cta = (double)ix->n_blocks / ix->n_cells * n_probe / P.S;
    P.NW = 8; P.MINB = blocks_per_cta >= 2000.0 ? 2 : 3;
  } else {
    P.NW = 8; P.MINB = 2;
  }
#ifdef TPQ_DEBUG_KNOBS
  // experiment knobs (scripts/sweep_scan.py), read once per search
  const char* lm = getenv("TPQ_LUT_MODE");            // "staged": every LUT through lut_kernel
  if (lm && !strcmp(lm, "staged")) P.dsub = 0;
  const char* rm = getenv("TPQ_RES_MODE");            // residual, "staged*": the query half through lut_kernel,
  if (P.residual && rm && !strncmp(rm, "staged", 6)) {  // "staged2|3": with 8-warp CTAs, 2|3 per SM, at M <= 64
    P.dsub = 0;
    if (P.MP == 64 && !strcmp(rm, "staged3")) { P.NW = 8; P.MINB = 3; }
    if (P.MP == 64 && !strcmp(rm, "staged2")) { P.NW = 8; P.MINB = 2; }
  }
  const char* cfg = getenv("TPQ_SCAN_CFG");           // "<warps>x<min CTAs/SM>" of the plain query-major kernel at M <= 64
  if (cfg && !P.residual && P.MP == 64) {
    if (!strcmp(cfg, "8x2"))  { P.NW = 8;  P.MINB = 2; }
    if (!strcmp(cfg, "8x3"))  { P.NW = 8;  P.MINB = 3; }
    if (!strcmp(cfg, "16x1")) { P.NW = 16; P.MINB = 1; }
    if (!strcmp(cfg, "4x4"))  { P.NW = 4;  P.MINB = 4; }
  }
  const char* br = getenv("TPQ_BOOT_R");
  if (br && atoi(br) == 1) P.boot_r = 1;
  const char* bm = getenv("TPQ_BOOT_MODE");
  P.boot_mode = bm ? atoi(bm) : 1;
  P.phase = g_phase;
  const char* cc = getenv("TPQ_CELL_CFG");            // "<warps>x<blocks per warp>" of the cell-major kernel
  if (cc && !strcmp(cc, "14x6")) { P.cell_nw = 14; P.cell_r = 6; }
  if (cc && !strcmp(cc, "16x5")) { P.cell_nw = 16; P.cell_r = 5; }
  const char* ca = getenv("TPQ_CELL_ABLATE");         // bit 0: no refills, bit 1: no survivors (CellArgs::ablate)
  P.cell_ablate = ca ? atoi(ca) & 3 : 0;
#endif
  // Cell-major scan when a pair's LUT (64 KB) is clearly smaller than the codes of the cell it meets: the plain index at
  // M <= 64, with an in-kernel LUT build, whose cells hold more than kCellMinLive live vectors (codes) on average, on an
  // unsliced batch.  Unsharded only: on a cell shard, a query's entry 0 is usually another shard's cell, which gives
  // pass 1 no vectors and the bound 0, so every owned candidate would survive and overflow.
  P.cell_major = !push && !range && !P.residual && P.MP == 64 && P.dsub && P.S == 1 && ix->shard_world == 1 && ix->n_blocks > 0 &&
                 ix->mean_cell_live >= kCellMinLive;
  if (P.cell_major) { P.NW = 8; P.MINB = 2; }        // pass 1 and the overflow re-run: 120 registers, 0 spill bytes
  P.part1_in_smem = P.residual && P.dsub > 0;
  P.L = scan_smem(P.MP, n_probe, P.NW, list_capacity(k), P.residual, P.part1_in_smem);
  P.ws = search_ws(ix, nq, n_probe, k, P);
  if (P.residual && ix->metric != TPQ_METRIC_EUCLIDEAN) {
    P.rc = TPQ_ERR_UNSUPPORTED;
    snprintf(P.err, sizeof P.err, "residual IVFPQ is defined for the euclidean metric");
  } else if (P.MP > 192) {
    P.rc = TPQ_ERR_UNSUPPORTED;
    if (P.residual)
      snprintf(P.err, sizeof P.err, "residual IVFPQ: n_subvectors=%d (padded %d) > 192 is not supported", ix->n_subvectors, P.MP);
    else
      snprintf(P.err, sizeof P.err, "n_subvectors=%d (padded %d) > 192 is not supported by the scan-layout path", ix->n_subvectors, P.MP);
  } else if (P.L.total > kSmemLimit) {
    P.rc = TPQ_ERR_UNSUPPORTED;
    snprintf(P.err, sizeof P.err, "scan: M=%d n_probe=%d k=%d needs %zu B of shared memory (> 227 KB)", ix->n_subvectors, n_probe, k, P.L.total);
  }
  return P;
}

// The plan's query-major kernel.  The instantiations named here are all that exist; plan_scan picks among them.
using ScanKernel = void (*)(ScanArgs, ScanSmem);
template <int DSUB>
static ScanKernel scan_kernel_d(const ScanPlan& P) {
  if (P.residual) {
    if constexpr (DSUB == 1 || DSUB == 2 || DSUB == 4)
      return P.MP == 32 ? ivfpq_scan_kernel<32, 16, 1, DSUB, true> : ivfpq_scan_kernel<64, 16, 1, DSUB, true>;
#ifdef TPQ_DEBUG_KNOBS
    if (P.MP == 64 && P.NW == 8) return P.MINB == 3 ? ivfpq_scan_kernel<64, 8, 3, 0, true> : ivfpq_scan_kernel<64, 8, 2, 0, true>;
#endif
    switch (P.MP) {
      case 32:  return ivfpq_scan_kernel<32, 16, 1, 0, true>;
      case 64:  return ivfpq_scan_kernel<64, 16, 1, 0, true>;
      case 96:  return ivfpq_scan_kernel<96, 16, 1, 0, true>;
      case 128: return ivfpq_scan_kernel<128, 16, 1, 0, true>;
      case 160: return ivfpq_scan_kernel<160, 16, 1, 0, true>;
      case 192: return ivfpq_scan_kernel<192, 16, 1, 0, true>;
    }
    return nullptr;
  }
#ifdef TPQ_DEBUG_KNOBS
  if (P.MP == 64 && P.NW == 16) return ivfpq_scan_kernel<64, 16, 1, DSUB, false>;
  if (P.MP == 64 && P.NW == 4)  return ivfpq_scan_kernel<64, 4, 4, DSUB, false>;
#endif
  switch (P.MP) {
    case 32:  return ivfpq_scan_kernel<32, 8, 2, DSUB, false>;
    case 64:  return P.MINB == 2 ? ivfpq_scan_kernel<64, 8, 2, DSUB, false> : ivfpq_scan_kernel<64, 8, 3, DSUB, false>;
    case 96:  return ivfpq_scan_kernel<96, 16, 1, DSUB, false>;
    case 128: return ivfpq_scan_kernel<128, 16, 1, DSUB, false>;
    case 160: return ivfpq_scan_kernel<160, 16, 1, DSUB, false>;
    case 192: return ivfpq_scan_kernel<192, 16, 1, DSUB, false>;
  }
  return nullptr;
}
static ScanKernel scan_kernel(const ScanPlan& P) {
  switch (P.qm_dsub()) {
    case 1:  return scan_kernel_d<1>(P);
    case 2:  return scan_kernel_d<2>(P);
    case 4:  return scan_kernel_d<4>(P);
    case 8:  return scan_kernel_d<8>(P);
    default: return scan_kernel_d<0>(P);
  }
}
// The plan's range kernel, scan_kernel's counterpart: one ivfpq_range_kernel for every configuration the product plan
// picks, and only those (the debug build's other configurations have none: nullptr).
using RangeKernel = void (*)(ScanArgs, ScanSmem, RangeOut);
template <int DSUB>
static RangeKernel range_kernel_d(const ScanPlan& P) {
  if (P.residual) {
    if (P.NW != 16) return nullptr;
    if constexpr (DSUB == 1 || DSUB == 2 || DSUB == 4)
      return P.MP == 32 ? ivfpq_range_kernel<32, 16, 1, DSUB, true> : ivfpq_range_kernel<64, 16, 1, DSUB, true>;
    switch (P.MP) {
      case 32:  return ivfpq_range_kernel<32, 16, 1, 0, true>;
      case 64:  return ivfpq_range_kernel<64, 16, 1, 0, true>;
      case 96:  return ivfpq_range_kernel<96, 16, 1, 0, true>;
      case 128: return ivfpq_range_kernel<128, 16, 1, 0, true>;
      case 160: return ivfpq_range_kernel<160, 16, 1, 0, true>;
      case 192: return ivfpq_range_kernel<192, 16, 1, 0, true>;
    }
    return nullptr;
  }
  if (P.MP <= 64 && P.NW != 8) return nullptr;
  switch (P.MP) {
    case 32:  return ivfpq_range_kernel<32, 8, 2, DSUB, false>;
    case 64:  return P.MINB == 2 ? ivfpq_range_kernel<64, 8, 2, DSUB, false> : ivfpq_range_kernel<64, 8, 3, DSUB, false>;
    case 96:  return ivfpq_range_kernel<96, 16, 1, DSUB, false>;
    case 128: return ivfpq_range_kernel<128, 16, 1, DSUB, false>;
    case 160: return ivfpq_range_kernel<160, 16, 1, DSUB, false>;
    case 192: return ivfpq_range_kernel<192, 16, 1, DSUB, false>;
  }
  return nullptr;
}
static RangeKernel range_kernel(const ScanPlan& P) {
  switch (P.dsub) {                                          // a range plan is never cell-major: qm_dsub() == dsub
    case 1:  return range_kernel_d<1>(P);
    case 2:  return range_kernel_d<2>(P);
    case 4:  return range_kernel_d<4>(P);
    case 8:  return range_kernel_d<8>(P);
    default: return range_kernel_d<0>(P);
  }
}
using CellLutKernel = decltype(&cell_lut_kernel<1>);
static CellLutKernel cell_lut(int dsub) {                    // the cell-major path builds its LUTs in-kernel only
  switch (dsub) {
    case 1:  return cell_lut_kernel<1>;
    case 2:  return cell_lut_kernel<2>;
    case 4:  return cell_lut_kernel<4>;
    default: return cell_lut_kernel<8>;
  }
}

// One scan of a batch: its queries and probe lists, and the search workspace w.  base_sims: the coarse similarities
// (read by residual IVFPQ); n_peers > 0: the fused exchange into every peer's gather buffer, else the keys go to the
// workspace's keys [nq][S][k].
struct ScanJob {
  const tpq_index* ix; const float* x; const int64_t* cells; const int64_t* npl; const float* base_sims;
  int nq, n_probe, k;
  uint8_t* w; cudaStream_t st; uint64_t* const* peer_keys; int n_peers, peer_slot;
};

// the arguments of every query-major launch for the chunk at q0
static ScanArgs scan_args(const ScanPlan& P, const ScanJob& J, int q0) {
  const tpq_index* ix = J.ix;
  ScanArgs A{};
  A.x = J.x; A.cbt = ix->pq_codebook_t; A.M = ix->n_subvectors; A.metric = ix->metric; A.part2_scan = ix->part2_scan;
  A.codes = ix->codes_scan; A.valid = ix->block_valid; A.cell_block_start = ix->cell_block_start;
  A.cell_start = ix->cell_start; A.cell_size = ix->cell_size; A.n_cells = ix->n_cells; A.boot_r = P.boot_r;
  A.lut_scan = reinterpret_cast<const float*>(J.w + P.ws.lut); A.cells = J.cells; A.n_probe_list = J.npl;
  A.base_sims = J.base_sims; A.keys_out = reinterpret_cast<uint64_t*>(J.w + P.ws.keys);
  A.nq = J.nq; A.q_base = q0; A.n_probe = J.n_probe; A.k = J.k; A.kp = list_capacity(J.k); A.S = P.S;
  A.n_peers = J.n_peers; A.peer_slot = J.peer_slot;
  for (int p = 0; p < J.n_peers; ++p) A.peer_keys[p] = J.peer_keys[p];
#ifdef TPQ_DEBUG_KNOBS
  A.phase = P.phase; A.boot_mode = P.boot_mode;
#endif
  return A;
}

// The cell-major scan of the n queries at q0 (see ivfpq_cell_scan_kernel); leaves their keys [n][k].  qmajor and A:
// the plan's query-major kernel and its arguments for the chunk, for pass 1 and the overflow re-run.
static int cell_stage(const ScanPlan& P, const ScanJob& J, ScanKernel qmajor, ScanArgs A, int q0, int n) {
  const tpq_index* ix = J.ix;
  const SearchWs& W = P.ws;
  uint8_t* w = J.w;
  const int kp = list_capacity(J.k), cap = cell_cap(J.k), C = ix->n_cells;
  cudaStream_t st = J.st;
  float* lut_ws = reinterpret_cast<float*>(w + W.lut);
  uint64_t* keys = reinterpret_cast<uint64_t*>(w + W.keys);
  int* cell_cnt = reinterpret_cast<int*>(w + W.cell_cnt);
  int* n_items = cell_cnt + C;
  int *cell_off = reinterpret_cast<int*>(w + W.cell_off), *slot = reinterpret_cast<int*>(w + W.slot);
  int* pair_q = reinterpret_cast<int*>(w + W.pair_q);
  CellItem* items = reinterpret_cast<CellItem*>(w + W.items);
  int64_t* ones = reinterpret_cast<int64_t*>(w + W.ones);
  uint64_t* surv = reinterpret_cast<uint64_t*>(w + W.surv);
  int* surv_cnt = reinterpret_cast<int*>(w + W.surv_cnt);

  auto cscan = ivfpq_cell_scan_kernel<kCellNW, kCellR>;
  size_t cs_smem = cell_smem_bytes(P.cell_nw, P.cell_r);
#ifdef TPQ_DEBUG_KNOBS
  if (P.cell_nw == 14) cscan = ivfpq_cell_scan_kernel<14, 6>;
  if (P.cell_nw == 16) cscan = ivfpq_cell_scan_kernel<16, 5>;
  cs_smem += (size_t)P.cell_nw * 64;                                      // the warps' cycle accounts
#endif
  TPQ_CUDA(cudaFuncSetAttribute(cscan, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cs_smem));
  const size_t sel_smem = (size_t)4 * (kp + kTopkBuf) * 8;
  TPQ_CUDA(cudaFuncSetAttribute(cell_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sel_smem));
  TPQ_CUDA(cudaMemsetAsync(cell_cnt, 0, (size_t)(C + 2) * 4, st));
  TPQ_CUDA(cudaMemsetAsync(surv_cnt, 0, (size_t)n * 4, st));
  cell_lut(P.dsub)<<<n, 256, 0, st>>>(J.x, ix->pq_codebook_t, ix->n_subvectors, J.nq, q0, ix->metric, lut_ws);
  TPQ_LAUNCH_CHECK("cell_lut_kernel");
  const int64_t nt = (int64_t)n * J.n_probe;
  const int pgrid = (int)((nt + 255) / 256);
  cell_pairs_count_kernel<<<pgrid, 256, 0, st>>>(J.cells, J.npl, q0, n, J.n_probe, C, ix->cell_start, ix->cell_size,
                                                 ix->cell_block_start, cell_cnt, slot, ones);
  TPQ_LAUNCH_CHECK("cell_pairs_count_kernel");
  A.n_probe_list = ones;
  qmajor<<<n, P.NW * 32, P.L.total, st>>>(A, P.L);                        // pass 1: entry 0 of every query
  TPQ_LAUNCH_CHECK("ivfpq_scan_kernel");
  cell_plan_kernel<<<1, 1024, 0, st>>>(cell_cnt, ix->cell_block_start, ix->cell_size, C, P.cell_nw * P.cell_r, cell_off,
                                       items, n_items);
  TPQ_LAUNCH_CHECK("cell_plan_kernel");
  cell_pairs_scatter_kernel<<<pgrid, 256, 0, st>>>(J.cells, q0, n, J.n_probe, slot, cell_off, pair_q);
  TPQ_LAUNCH_CHECK("cell_pairs_scatter_kernel");
  CellArgs CA;
  CA.codes = ix->codes_scan; CA.valid = ix->block_valid; CA.cell_block_start = ix->cell_block_start;
  CA.cell_start = ix->cell_start; CA.lut_scan = lut_ws; CA.cell_off = cell_off; CA.cell_cnt = cell_cnt; CA.pair_q = pair_q;
  CA.items = items; CA.n_items = n_items; CA.cursor = n_items + 1; CA.keys = keys; CA.surv = surv; CA.surv_cnt = surv_cnt;
  CA.log = reinterpret_cast<uint64_t*>(w + W.cell_log);
  CA.q_base = q0; CA.k = J.k; CA.cap = cap;
#ifdef TPQ_DEBUG_KNOBS
  CA.phase = P.phase ? P.phase + 8 : nullptr; CA.ablate = P.cell_ablate;
#endif
  cscan<<<P.cell_ctas, P.cell_nw * 32, cs_smem, st>>>(CA);
  TPQ_LAUNCH_CHECK("ivfpq_cell_scan_kernel");
  cell_select_kernel<<<(n + 3) / 4, 128, sel_smem, st>>>(keys, surv, surv_cnt, q0, n, J.k, kp, cap);
  TPQ_LAUNCH_CHECK("cell_select_kernel");
  A.n_probe_list = J.npl; A.only_cnt = surv_cnt; A.only_cap = cap;
  qmajor<<<n, P.NW * 32, P.L.total, st>>>(A, P.L);                        // queries whose survivors overflowed
  TPQ_LAUNCH_CHECK("ivfpq_scan_kernel");
  return TPQ_OK;
}

// Every scan launch of a batch, per chunk of P.chunk queries: the cell-major stage, or the staged LUT (when there is
// one) and the query-major kernel -- on a range plan the range kernel, whose matches go to R.  The profiling events
// bracket the scan stage of each chunk: the whole cell-major stage, or the query-major (or range) kernel.
static int launch(const ScanPlan& P, const ScanJob& J, const RangeOut* R = nullptr) {
  const tpq_index* ix = J.ix;
  const ScanKernel kern = P.range ? nullptr : scan_kernel(P);
  const RangeKernel rkern = P.range ? range_kernel(P) : nullptr;
  if (P.range) TPQ_CUDA(cudaFuncSetAttribute(rkern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)P.L.total));
  else TPQ_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)P.L.total));
  for (int q0 = 0; q0 < J.nq; q0 += P.chunk) {
    const int n = (J.nq - q0) < P.chunk ? (J.nq - q0) : P.chunk;
    if (!P.cell_major && P.dsub == 0) {
      if (int rc = launch_lut(J.x, J.nq, q0, n, ix->pq_codebook, ix->d_vector, ix->n_subvectors,
                              P.residual ? kLutPart1 : ix->metric, kLutScan, reinterpret_cast<float*>(J.w + P.ws.lut), J.st))
        return rc;
    }
    const ScanArgs A = scan_args(P, J, q0);
    const bool prof = g_prof_on && g_prof_n < kProfMax;
    if (prof) cudaEventRecord(g_prof_start[g_prof_n], J.st);
    if (P.range) {
      rkern<<<n * P.S, P.NW * 32, P.L.total, J.st>>>(A, P.L, *R);
      TPQ_LAUNCH_CHECK("ivfpq_range_kernel");
    } else if (P.cell_major) {
      if (int rc = cell_stage(P, J, kern, A, q0, n)) return rc;
    } else {
      kern<<<n * P.S, P.NW * 32, P.L.total, J.st>>>(A, P.L);
      TPQ_LAUNCH_CHECK("ivfpq_scan_kernel");
    }
    if (prof) cudaEventRecord(g_prof_stop[g_prof_n++], J.st);
  }
  return TPQ_OK;
}

static int check_index(const tpq_index* ix, int k) {
  TPQ_REQUIRE(ix, "null index");
  TPQ_REQUIRE(ix->d_vector > 0 && ix->n_subvectors > 0 && ix->d_vector % ix->n_subvectors == 0,
              "d_vector=%d must be a multiple of n_subvectors=%d", ix->d_vector, ix->n_subvectors);
  TPQ_REQUIRE(ix->n_subvectors % 4 == 0, "n_subvectors=%d must be a multiple of 4", ix->n_subvectors);
  TPQ_REQUIRE(ix->metric == TPQ_METRIC_EUCLIDEAN || ix->metric == TPQ_METRIC_COSINE,
              "unsupported distance (reference supports euclidean and cosine only)");
  TPQ_REQUIRE(ix->vq_codebook && ix->pq_codebook && ix->cell_start && ix->cell_size && ix->address2id, "index is missing reference buffers");
  TPQ_REQUIRE(ix->codes_scan || ix->n_blocks == 0, "index has no scan layout (call tpq_relayout_codes first)");
  TPQ_REQUIRE(ix->block_valid || ix->n_blocks == 0, "index has no scan layout (block_valid)");
  TPQ_REQUIRE(ix->cell_block_start && ix->pq_codebook_t && ix->pq_norm_t, "index has no scan layout (plan / codebook)");
  TPQ_REQUIRE(ix->m_pad == scan_m_pad(ix->n_subvectors), "index.m_pad is inconsistent");
  TPQ_REQUIRE(ix->capacity >= 0 && ix->capacity <= 0xFFFFFFFFll, "capacity exceeds the 32-bit address range");
  TPQ_REQUIRE(0 < k && k <= 1024, "k must be in (0, 1024], got %d", k);        // IVFPQIndex.py:473
  return TPQ_OK;
}

// The coarse stage inside the search workspace: cosine queries are normalised (IVFPQIndex.py:474-475), then every query
// gets its probe list, the lists' similarities and lengths.
struct Probes { const float* x; const float* sims; const int64_t* cells; const int64_t* npl; };
static int coarse_stage(const tpq_index* ix, const float* x_dn, int nq, int n_probe, int smart, float temperature,
                        uint8_t* w, const SearchWs& W, cudaStream_t stream, Probes& p) {
  p.x = x_dn;
  if (ix->metric == TPQ_METRIC_COSINE) {
    float* xn = reinterpret_cast<float*>(w + W.xnorm);
    if (int rc = tpq_normalize_columns(x_dn, ix->d_vector, nq, xn, stream)) return rc;
    p.x = xn;
  }
  float* sims = reinterpret_cast<float*>(w + W.probe_sims);
  int64_t *cells = reinterpret_cast<int64_t*>(w + W.cells), *npl = reinterpret_cast<int64_t*>(w + W.npl);
  if (int rc = tpq_coarse_probe(p.x, ix->vq_codebook, ix->d_vector, nq, ix->n_cells, n_probe, smart, temperature,
                                sims, cells, npl, w + W.coarse, W.probe_sims - W.coarse, stream)) return rc;
  p.sims = sims; p.cells = cells; p.npl = npl;
  return TPQ_OK;
}

// Where a search's keys go: merged across slices and decoded into values / ids / address / keys (each may be null), or,
// with n_peers > 0, pushed by the scan straight into every peer's gather buffer.
struct SearchOut {
  float* values; int64_t* ids; int64_t* address; uint64_t* keys;
  uint64_t* const* peer_keys; int n_peers, peer_slot;
};

// The search behind the three entry points, after their argument checks: plan, check the workspace, run the coarse
// stage unless the probe lists are given (p.cells), scan, then merge or push.
static int search(const tpq_index* ix, Probes p, int nq, int n_probe, int k, int smart, float temperature,
                  const SearchOut& o, void* ws, size_t ws_bytes, cudaStream_t st) {
  const bool push = o.n_peers > 0;
  const ScanPlan P = plan_scan(ix, nq, n_probe, k, push);
  if (push && P.S != 1) { set_error("tpq_ivfpq_scan_push: batch of %d queries is sliced; use the gathered exchange", nq); return TPQ_ERR_UNSUPPORTED; }
  if (push && nq > kQueryChunk) { set_error("tpq_ivfpq_scan_push: at most %d queries per call", kQueryChunk); return TPQ_ERR_UNSUPPORTED; }
  if (!ws || ws_bytes < P.ws.total) { set_error("workspace too small (%zu < %zu)", ws_bytes, P.ws.total); return TPQ_ERR_WORKSPACE; }
  if (!p.cells) TPQ_REQUIRE(n_probe <= ix->n_cells, "n_probe=%d must be in [1, n_cells=%d]", n_probe, ix->n_cells);
  for (int i = 0; i < o.n_peers; ++i) TPQ_REQUIRE(o.peer_keys[i], "null peer buffer");
  if (ix->residual && (!ix->part2_scan || (p.cells && !p.sims))) { set_error("residual search needs part2_scan and base_sims"); return TPQ_ERR_BAD_ARG; }
  if (P.rc) { set_error("%s", P.err); return P.rc; }
  uint8_t* w = reinterpret_cast<uint8_t*>(ws);
  if (!p.cells)
    if (int rc = coarse_stage(ix, p.x, nq, n_probe, smart, temperature, w, P.ws, st, p)) return rc;
  if (int rc = launch(P, ScanJob{ix, p.x, p.cells, p.npl, p.sims, nq, n_probe, k, w, st, o.peer_keys, o.n_peers, o.peer_slot}))
    return rc;
  if (push) return TPQ_OK;
  return launch_merge(reinterpret_cast<uint64_t*>(w + P.ws.keys), nq, P.S, k, k, (int64_t)P.S * k, ix->address2id,
                      ix->capacity, o.values, o.ids, o.address, o.keys, st);
}

}  // namespace tpq

using namespace tpq;

#ifdef TPQ_DEBUG_KNOBS
extern "C" int tpq_debug_set_phase_buffer(unsigned long long* dev_buf16) { g_phase = dev_buf16; return TPQ_OK; }
#endif

extern "C" int tpq_profile_enable(int on) {
  if (on && !g_prof_created) {
    for (int i = 0; i < kProfMax; ++i) { TPQ_CUDA(cudaEventCreate(&g_prof_start[i])); TPQ_CUDA(cudaEventCreate(&g_prof_stop[i])); }
    g_prof_created = true;
  }
  g_prof_on = on != 0;
  g_prof_n = 0;
  return TPQ_OK;
}

extern "C" int tpq_profile_scan_ms(float* total_ms, int* n_launches) {
  TPQ_REQUIRE(total_ms && n_launches, "null pointer");
  float tot = 0.f;
  for (int i = 0; i < g_prof_n; ++i) {
    TPQ_CUDA(cudaEventSynchronize(g_prof_stop[i]));
    float ms = 0.f;
    TPQ_CUDA(cudaEventElapsedTime(&ms, g_prof_start[i], g_prof_stop[i]));
    tot += ms;
  }
  *total_ms = tot; *n_launches = g_prof_n;
  g_prof_n = 0;
  return TPQ_OK;
}

extern "C" size_t tpq_search_workspace_bytes(const tpq_index* ix, int nq, int n_probe, int k) {
  if (!ix || nq <= 0 || n_probe <= 0 || k <= 0) return 0;
  return plan_scan(ix, nq, n_probe, k, /*push=*/false).ws.total;
}

extern "C" int tpq_ivfpq_search_cells(const tpq_index* ix, const float* x_dn, const int64_t* cells, const float* base_sims,
                                      const int64_t* n_probe_list, int nq, int n_probe, int k,
                                      float* values, int64_t* ids, int64_t* address, uint64_t* keys_out,
                                      void* ws, size_t ws_bytes, void* stream) {
  if (int rc = check_index(ix, k)) return rc;
  TPQ_REQUIRE(nq >= 0 && n_probe >= 1, "bad n_query=%d / n_probe=%d", nq, n_probe);
  TPQ_REQUIRE(x_dn && cells && n_probe_list, "null pointer argument");
  if (nq == 0) return TPQ_OK;
  return search(ix, Probes{x_dn, base_sims, cells, n_probe_list}, nq, n_probe, k, 0, 0.f,
                SearchOut{values, ids, address, keys_out, nullptr, 0, 0}, ws, ws_bytes, (cudaStream_t)stream);
}

extern "C" int tpq_ivfpq_search(const tpq_index* ix, const float* x_dn, int nq, int n_probe, int k,
                                int smart, float temperature,
                                float* values, int64_t* ids, int64_t* address, uint64_t* keys_out,
                                void* ws, size_t ws_bytes, void* stream) {
  if (int rc = check_index(ix, k)) return rc;
  TPQ_REQUIRE(nq >= 0 && x_dn, "bad query batch");
  TPQ_REQUIRE(n_probe >= 1 && n_probe <= ix->n_cells, "n_probe=%d must be in [1, n_cells=%d]", n_probe, ix->n_cells);
  if (nq == 0) return TPQ_OK;
  return search(ix, Probes{x_dn, nullptr, nullptr, nullptr}, nq, n_probe, k, smart, temperature,
                SearchOut{values, ids, address, keys_out, nullptr, 0, 0}, ws, ws_bytes, (cudaStream_t)stream);
}

// cells == nullptr: the whole coarse stage runs here (replicated probe)
extern "C" int tpq_ivfpq_scan_push(const tpq_index* ix, const float* x_dn, const int64_t* cells, const float* base_sims,
                                   const int64_t* n_probe_list, int nq, int n_probe, int k, int smart, float temperature,
                                   uint64_t* const* peer_keys, int n_peers, int my_slot,
                                   void* ws, size_t ws_bytes, void* stream) {
  if (int rc = check_index(ix, k)) return rc;
  TPQ_REQUIRE(nq >= 0 && n_probe >= 1 && x_dn, "bad query batch");
  TPQ_REQUIRE(peer_keys && n_peers >= 1 && n_peers <= 8 && my_slot >= 0, "tpq_ivfpq_scan_push: bad peer list");
  TPQ_REQUIRE((cells == nullptr) == (n_probe_list == nullptr), "cells and n_probe_list go together");
  if (nq == 0) return TPQ_OK;
  return search(ix, Probes{x_dn, base_sims, cells, n_probe_list}, nq, n_probe, k, smart, temperature,
                SearchOut{nullptr, nullptr, nullptr, nullptr, peer_keys, n_peers, my_slot}, ws, ws_bytes,
                (cudaStream_t)stream);
}

// ----------------------------------------------------------------------------- range search
extern "C" size_t tpq_ivfpq_range_workspace_bytes(const tpq_index* ix, int nq, int n_probe) {
  if (!ix || nq <= 0 || n_probe <= 0) return 0;
  return plan_scan(ix, nq, n_probe, 1, /*push=*/false, /*range=*/true).ws.total;
}

// cells == nullptr: the coarse stage of tpq_ivfpq_search runs here; else the probe lists of tpq_ivfpq_search_cells
extern "C" int tpq_ivfpq_range_search(const tpq_index* ix, const float* x_dn, const int64_t* cells, const float* base_sims,
                                      const int64_t* n_probe_list, int nq, int n_probe, int smart, float temperature,
                                      float threshold, uint64_t* match_keys, int32_t* match_query, int64_t cap,
                                      uint64_t* total, void* ws, size_t ws_bytes, void* stream) {
  if (int rc = check_index(ix, 1)) return rc;
  TPQ_REQUIRE(nq >= 0 && x_dn, "tpq_ivfpq_range_search: bad query batch");
  TPQ_REQUIRE((cells == nullptr) == (n_probe_list == nullptr), "tpq_ivfpq_range_search: cells and n_probe_list go together");
  TPQ_REQUIRE(n_probe >= 1 && (cells || n_probe <= ix->n_cells), "n_probe=%d must be in [1, n_cells=%d]", n_probe, ix->n_cells);
  if (!cells && n_probe > 1024) { set_error("n_probe=%d > 1024 is not supported", n_probe); return TPQ_ERR_UNSUPPORTED; }
  TPQ_REQUIRE(threshold == threshold, "tpq_ivfpq_range_search: the threshold is NaN");
  TPQ_REQUIRE(cap >= 0, "tpq_ivfpq_range_search: cap=%lld is negative", (long long)cap);
  TPQ_REQUIRE(total && (cap == 0 || (match_keys && match_query)), "tpq_ivfpq_range_search: null total or match buffer");
  if (ix->residual && (!ix->part2_scan || (cells && !base_sims))) {
    set_error("tpq_ivfpq_range_search: residual search needs part2_scan and base_sims");
    return TPQ_ERR_BAD_ARG;
  }
  if (nq == 0) return TPQ_OK;
  const ScanPlan P = plan_scan(ix, nq, n_probe, 1, /*push=*/false, /*range=*/true);
  if (P.rc) { set_error("%s", P.err); return P.rc; }
  if (!range_kernel(P)) { set_error("tpq_ivfpq_range_search: no range kernel for this scan configuration"); return TPQ_ERR_UNSUPPORTED; }
  if (!ws || ws_bytes < P.ws.total) {
    set_error("tpq_ivfpq_range_search: workspace too small (%zu < %zu)", ws_bytes, P.ws.total);
    return TPQ_ERR_WORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  TPQ_CUDA(cudaMemsetAsync(total, 0, sizeof(uint64_t), st));
  if (ix->n_blocks == 0) return TPQ_OK;                     // nothing to score
  uint8_t* w = reinterpret_cast<uint8_t*>(ws);
  Probes p{x_dn, base_sims, cells, n_probe_list};
  if (!cells)
    if (int rc = coarse_stage(ix, x_dn, nq, n_probe, smart, temperature, w, P.ws, st, p)) return rc;
  const RangeOut R{threshold, match_keys, match_query, cap, reinterpret_cast<unsigned long long*>(total)};
  return launch(P, ScanJob{ix, p.x, p.cells, p.npl, p.sims, nq, n_probe, 1, w, st, nullptr, 0, 0}, &R);
}

extern "C" int tpq_merge_topk(const uint64_t* keys_in, int nq, int n_parts, int k,
                              const int64_t* address2id, int64_t capacity,
                              float* values, int64_t* ids, int64_t* address, void* stream) {
  TPQ_REQUIRE(keys_in && nq >= 0 && n_parts >= 1 && 0 < k && k <= 1024, "tpq_merge_topk: bad argument");
  TPQ_REQUIRE(!ids || address2id, "tpq_merge_topk: ids requested without address2id");
  if (nq == 0) return TPQ_OK;
  // keys_in is [n_parts, nq, k] (the all-gather's natural layout): part stride nq*k, query stride k
  return launch_merge(keys_in, nq, n_parts, k, (int64_t)nq * k, k, address2id, capacity, values, ids, address, nullptr,
                      (cudaStream_t)stream);
}
