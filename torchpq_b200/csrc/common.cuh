// Shared device/host helpers for the tpq_b200 kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include "../../include/tpq_b200.h"

namespace tpq {

// ----------------------------------------------------------------------------- errors
void set_error(const char* fmt, ...);
int  cuda_fail(cudaError_t e, const char* what);
// streaming multiprocessors of the current device (grid sizing)
int  device_sm_count();

#define TPQ_REQUIRE(cond, ...)                                   \
  do { if (!(cond)) { ::tpq::set_error(__VA_ARGS__); return TPQ_ERR_BAD_ARG; } } while (0)
#define TPQ_CUDA(call)                                           \
  do { cudaError_t e__ = (call); if (e__ != cudaSuccess) return ::tpq::cuda_fail(e__, #call); } while (0)
#define TPQ_LAUNCH_CHECK(name)                                   \
  do { cudaError_t e__ = cudaGetLastError(); if (e__ != cudaSuccess) return ::tpq::cuda_fail(e__, name); } while (0)

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }
static inline int next_pow2(int x) { int p = 1; while (p < x) p <<= 1; return p; }
// slots of a sorted top-k list in shared memory: k rounded up to a power of two, at least one warp's worth
static inline int list_capacity(int k) { return next_pow2(k < 32 ? 32 : k); }
// dynamic shared memory one CTA may use on sm_90
constexpr size_t kSmemLimit = 227 * 1024;

// ----------------------------------------------------------------------------- candidate keys
// A candidate is one 64-bit key: high word = order-preserving image of the fp32 score,
// low word = ~address.  Larger key == better candidate under the total order
// (score descending, address ascending).  Key 0 is "empty" (below every real key).
__host__ __device__ __forceinline__ uint32_t score_to_ord(float f) {
#ifdef __CUDA_ARCH__
  uint32_t b = __float_as_uint(f);
#else
  uint32_t b; memcpy(&b, &f, 4);
#endif
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__host__ __device__ __forceinline__ float ord_to_score(uint32_t o) {
  uint32_t b = (o & 0x80000000u) ? (o ^ 0x80000000u) : ~o;
#ifdef __CUDA_ARCH__
  return __uint_as_float(b);
#else
  float f; memcpy(&f, &b, 4); return f;
#endif
}
__device__ __forceinline__ uint64_t make_key(float score, uint32_t addr) {
  return ((uint64_t)score_to_ord(score) << 32) | (uint64_t)(0xFFFFFFFFu - addr);
}
__device__ __forceinline__ float    key_score(uint64_t k) { return ord_to_score((uint32_t)(k >> 32)); }
__device__ __forceinline__ uint32_t key_addr(uint64_t k)  { return 0xFFFFFFFFu - (uint32_t)k; }

#ifdef __CUDACC__
// Inclusive prefix sum over the lanes of a full warp: returns the sum of v over lanes 0 .. lane.
template <class T>
__device__ __forceinline__ T warp_inclusive_scan(T v, int lane) {
  #pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const T t = __shfl_up_sync(0xffffffffu, v, o); if (lane >= o) v += t; }
  return v;
}

// One 1024-value tile of a CTA-wide inclusive prefix sum (blockDim.x == 1024, called by every thread): returns carry +
// the sum of v over threads 0 .. threadIdx.x, and advances carry (shared memory) by the tile's total.  wsum: [32] shared.
template <class T>
__device__ __forceinline__ T cta_inclusive_scan(T v, T* wsum, T& carry) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const T incl = warp_inclusive_scan(v, lane);
  if (lane == 31) wsum[warp] = incl;
  __syncthreads();
  if (warp == 0) wsum[lane] = warp_inclusive_scan(wsum[lane], lane);   // inclusive over warps
  __syncthreads();
  const T r = carry + (warp ? wsum[warp - 1] : T(0)) + incl;
  __syncthreads();
  if (threadIdx.x == 1023) carry = r;
  __syncthreads();
  return r;
}

// ----------------------------------------------------------------------------- bitonic networks in registers
// A warp holds a sequence of 32*R keys as x[r] = element r*32 + lane.  Compare-exchanges at distance >= 32 are
// register-to-register inside a thread; smaller distances are one SHFL.64 per key -- a quarter of the shared-memory
// traffic of the same stage done through LDS/STS pairs, and free of bank conflicts (the strided 64-bit accesses of the
// small-distance stages were the bulk of the scan kernel's bank conflicts in round 1).
__device__ __forceinline__ uint64_t shfl_xor64(uint64_t v, int m) {
  return (uint64_t)__shfl_xor_sync(0xffffffffu, (unsigned long long)v, m);
}
__device__ __forceinline__ uint64_t key_max(uint64_t a, uint64_t b) { return a > b ? a : b; }
__device__ __forceinline__ uint64_t key_min(uint64_t a, uint64_t b) { return a < b ? a : b; }

// The stage loops are deliberately NOT unrolled: a flush is rare next to the scan loop it interrupts, and the fully
// unrolled networks (1250 SHFLs, 12 k instructions once inlined at every push site) evicted the hot loop from the
// instruction cache, which made them slower than the rolled form on an L2-resident shard.

__device__ __forceinline__ void key_cswap(uint64_t& a, uint64_t& b, bool desc) {     // desc: a <- max, b <- min
  const uint64_t hi = key_max(a, b), lo = key_min(a, b);
  a = desc ? hi : lo; b = desc ? lo : hi;
}

// bitonic sequence -> sorted (descending, or ascending when ASC); R = 1, 2 or 4
template <int R, bool ASC = false>
__device__ __forceinline__ void reg_merge(uint64_t (&x)[R], int lane) {
  static_assert(R == 1 || R == 2 || R == 4, "a warp run is 32, 64 or 128 keys");
  if (R == 4) { key_cswap(x[0], x[R / 2], !ASC); key_cswap(x[R / 4], x[R - 1], !ASC); }     // distance 64
  if (R >= 2) {                                                                            // distance 32
    #pragma unroll
    for (int r = 0; r < R; r += 2) key_cswap(x[r], x[r + (R >= 2)], !ASC);
  }
  #pragma unroll 1
  for (int j = 16; j > 0; j >>= 1) {
    const bool up = (lane & j) != 0;
    #pragma unroll
    for (int r = 0; r < R; ++r) {
      const uint64_t y = shfl_xor64(x[r], j);
      x[r] = (up != ASC) ? key_min(x[r], y) : key_max(x[r], y);
    }
  }
}

// arbitrary sequence -> sorted (descending, or ascending when ASC); R = 1, 2 or 4
template <int R, bool ASC = false>
__device__ __forceinline__ void reg_sort(uint64_t (&x)[R], int lane) {
  static_assert(R == 1 || R == 2 || R == 4, "a warp run is 32, 64 or 128 keys");
  #pragma unroll 1
  for (int k = 2; k <= 32 * R; k <<= 1) {
    int j = k >> 1;
    // distances >= 32 are register-to-register; element index = r*32 + lane, direction bit = index & k
    if (R == 4 && k == 128) { key_cswap(x[0], x[R / 2], !ASC); key_cswap(x[R / 4], x[R - 1], !ASC); j = 32; }
    if (R >= 2 && j == 32) {
      #pragma unroll
      for (int r = 0; r < R; r += 2) key_cswap(x[r], x[r + (R >= 2)], (((r * 32) & k) == 0) != ASC);
      j = 16;
    }
    #pragma unroll 1
    for (; j > 0; j >>= 1) {
      const bool up = (lane & j) != 0;
      #pragma unroll
      for (int r = 0; r < R; ++r) {
        const bool desc = ((((r * 32) | lane) & k) == 0) != ASC;
        const uint64_t y = shfl_xor64(x[r], j);
        x[r] = (desc != up) ? key_max(x[r], y) : key_min(x[r], y);
      }
    }
  }
}

// ----------------------------------------------------------------------------- warp-cooperative sorted lists in shared memory
// All routines are called by a full warp with warp-uniform arguments.

// Sort a BITONIC sequence a[0..n) in shared memory descending (n a power of two >= 32).  Distances >= 64 are
// compare-exchanges between conflict-free runs of consecutive keys; the last six stages of every 64-key chunk run in
// registers.
__device__ __forceinline__ void warp_bitonic_merge_desc(uint64_t* a, int n, int lane) {
  for (int j = n >> 1; j >= 64; j >>= 1) {
    for (int t = lane; t < (n >> 1); t += 32) {
      const int lo = ((t & ~(j - 1)) << 1) | (t & (j - 1));
      const int hi = lo + j;
      const uint64_t x = a[lo], y = a[hi];
      if (x < y) { a[lo] = y; a[hi] = x; }
    }
    __syncwarp();
  }
  if (n == 32) {
    uint64_t x[1] = {a[lane]};
    reg_merge<1>(x, lane);
    a[lane] = x[0];
  } else {
    for (int c = 0; c < n; c += 64) {
      uint64_t x[2] = {a[c + lane], a[c + 32 + lane]};
      reg_merge<2>(x, lane);
      a[c + lane] = x[0]; a[c + 32 + lane] = x[1];
    }
  }
  __syncwarp();
}

// A[0..n) and B[0..nb) (shared memory) both sorted descending, nb <= n, both powers of two >= 32.
// A <- the n largest of A u B, sorted descending.  B is left untouched.
__device__ __forceinline__ void warp_merge_desc(uint64_t* A, int n, const uint64_t* B, int nb, int lane) {
  for (int t = lane; t < nb; t += 32) {
    const int i = n - nb + t;
    A[i] = key_max(A[i], B[nb - 1 - t]);
  }
  __syncwarp();
  warp_bitonic_merge_desc(A, n, lane);
}

// Merge a run of 32*R keys held in registers, sorted ASCENDING (x[r] = element r*32 + lane), into the descending list
// A[0..n) (n >= 32*R): A <- the n largest of A u run, sorted descending.
template <int R>
__device__ __forceinline__ void warp_merge_run(uint64_t* A, int n, const uint64_t (&x)[R], int lane) {
  uint64_t* tail = A + (n - 32 * R);
  if (n == 32 * R) {                                       // the whole list fits the registers
    uint64_t y[R];
    #pragma unroll
    for (int r = 0; r < R; ++r) y[r] = key_max(tail[r * 32 + lane], x[r]);
    reg_merge<R>(y, lane);
    #pragma unroll
    for (int r = 0; r < R; ++r) tail[r * 32 + lane] = y[r];
    __syncwarp();
    return;
  }
  #pragma unroll
  for (int r = 0; r < R; ++r) tail[r * 32 + lane] = key_max(tail[r * 32 + lane], x[r]);
  __syncwarp();
  warp_bitonic_merge_desc(A, n, lane);
}

// In-place merge of two descending runs A[0..len), B[0..len) (len a power of two >= 32):
//   top_only: A <- the len largest of A u B, descending (B clobbered);
//   else:     A, B <- A u B sorted descending across (A then B).
__device__ __forceinline__ void warp_merge_runs(uint64_t* A, uint64_t* B, int len, bool top_only, int lane) {
  for (int t = lane; t < len; t += 32) {
    const uint64_t a = A[t], b = B[len - 1 - t];
    A[t] = key_max(a, b);
    if (!top_only) B[len - 1 - t] = key_min(a, b);          // the low half, reversed: still bitonic
  }
  __syncwarp();
  warp_bitonic_merge_desc(A, len, lane);
  if (!top_only) warp_bitonic_merge_desc(B, len, lane);
}

// ----------------------------------------------------------------------------- staged candidates
// A selector stages the keys that pass its filter in an unsorted buffer, and from time to time sorts the staged run in
// registers and merges it into its sorted list.  The three steps below are the only copies of their rules.

// The lanes with `pass` append their keys to buf[cnt ..) in lane order; returns how many were appended (warp-uniform).
__device__ __forceinline__ int warp_append(uint64_t* buf, int cnt, bool pass, uint64_t key, int lane) {
  const unsigned m = __ballot_sync(0xffffffffu, pass);
  if (pass) buf[cnt + __popc(m & ((1u << lane) - 1))] = key;
  return __popc(m);
}

constexpr int kTopkBuf = 64;      // WarpTopK staging entries per warp
constexpr int kStage = 96;        // CtaTopK staging entries per warp: flush is attempted above 32, forced above 64

// x <- the n <= 32*R keys staged at buf, padded with empty keys, sorted ASCENDING (x[r] = element r*32 + lane).  No
// buffer stages more than kStage keys, so a register past that is empty without a look at n.
template <int R>
__device__ __forceinline__ void load_sorted_run(uint64_t (&x)[R], const uint64_t* buf, int n, int lane) {
  #pragma unroll
  for (int r = 0; r < R; ++r) x[r] = (r * 32 < kStage && r * 32 + lane < n) ? buf[r * 32 + lane] : 0ull;
  reg_sort<R, true>(x, lane);
}

// The cap: of an ascending run of 32*R keys only the kp largest can enter a list of kp slots, and they are its last
// registers.  merge(y) receives the run, or its last kp keys when it is longer than the list.
template <int R, class Merge>
__device__ __forceinline__ void merge_capped(const uint64_t (&x)[R], int kp, Merge merge) {
  if (R > 1 && kp == 32) { const uint64_t y[1] = {x[R - 1]}; merge(y); }
  else if (R > 2 && kp == 64) { const uint64_t y[2] = {x[R - 2], x[R - 1]}; merge(y); }
  else merge(x);
}

// Sort the n staged keys of buf (0 < n <= 32*RMAX) into the shortest run that holds them and hand it, capped to kp, to
// merge: warp_merge_run into a list the warp owns, CtaTopK::merge_locked into the CTA's.
template <int RMAX, class Merge>
__device__ __forceinline__ void merge_staged(const uint64_t* buf, int n, int kp, int lane, Merge merge) {
  if (n <= 32) { uint64_t x[1]; load_sorted_run(x, buf, n, lane); merge(x); }
  else if (RMAX == 2 || n <= 64) { uint64_t x[2]; load_sorted_run(x, buf, n, lane); merge_capped(x, kp, merge); }
  else { uint64_t x[4]; load_sorted_run(x, buf, n, lane); merge_capped(x, kp, merge); }
}

// Per-warp top-k selector: sorted list of KP keys + an unsorted staging buffer.
// Candidates are appended with push(); when the buffer cannot take another full
// warp's worth it is sorted and merged into the list.
struct WarpTopK {
  uint64_t* list;   // [kp] descending
  uint64_t* buf;    // [kTopkBuf]
  int kp;           // power of two >= max(k, 32)... list capacity
  int k;            // wanted
  int cnt;          // entries in buf (warp-uniform)

  __device__ __forceinline__ void init(uint64_t* list_, uint64_t* buf_, int kp_, int k_, int lane) {
    list = list_; buf = buf_; kp = kp_; k = k_; cnt = 0;
    for (int i = lane; i < kp; i += 32) list[i] = 0;
    __syncwarp();
  }
  // k-th best so far (0 while fewer than k candidates were seen)
  __device__ __forceinline__ uint64_t kth() const { return list[k - 1]; }

  __device__ __forceinline__ void flush(int lane) {
    if (cnt == 0) return;
    merge_staged<2>(buf, cnt, kp, lane, [&](const auto& x) { warp_merge_run(list, kp, x, lane); });
    cnt = 0;
  }
  // pass: this lane has a candidate.  Returns true if a flush happened (threshold may have risen).
  __device__ __forceinline__ bool push(bool pass, uint64_t key, int lane) {
    const int n = warp_append(buf, cnt, pass, key, lane);
    if (n == 0) return false;
    cnt += n;
    __syncwarp();
    if (cnt > kTopkBuf - 32) { flush(lane); return true; }
    return false;
  }
};

// CTA-wide top-k selector: ONE sorted list of kp keys shared by all warps of the CTA (so its
// k-th entry is the true running k-th best of everything merged so far), one staging buffer
// per warp.  A warp whose buffer is more than half full sorts it privately (in registers), then takes the
// CTA lock and merges it into the shared list; the other warps keep scanning against the
// (slightly stale, always valid) threshold in *thr.  Exact: a candidate is only ever dropped
// when k better ones are already in the list.
// The selector owns its shared memory: a kernel reserves bytes(nw, kp) at an 8-byte aligned offset and hands the
// address to init(), which lays out  thr | lock, drain counter | rep[nw] | list[kp] | nw staging buffers of kStage keys.
struct CtaTopK {
  uint64_t* list;               // [kp] descending, shared by the CTA
  unsigned long long* thr;      // k-th best of `list` (0 while fewer than k merged)
  int* lock;                    // lock[0] = the list lock, lock[1] = append counter of cta_drain
  uint64_t* buf;                // [kStage] this warp's staging buffer
  int kp, k, cnt;

  static constexpr size_t bytes(int nw, int kp) { return 8 * (2 + (size_t)nw + (size_t)kp + (size_t)nw * kStage); }
  // the quick start's report of each warp; the staging buffers of all warps, scratch once their keys are in registers
  __device__ __forceinline__ uint64_t* rep() const { return reinterpret_cast<uint64_t*>(thr) + 2; }
  __device__ __forceinline__ uint64_t* scratch() const { return list + kp; }

  // call from every thread of the CTA (nw warps), then __syncthreads()
  __device__ __forceinline__ void init(void* smem, int nw, int warp, int kp_, int k_) {
    thr = reinterpret_cast<unsigned long long*>(smem);
    lock = reinterpret_cast<int*>(thr + 1);
    list = rep() + nw;
    kp = kp_; k = k_; cnt = 0;
    buf = scratch() + (size_t)warp * kStage;
    for (int i = threadIdx.x; i < kp; i += blockDim.x) list[i] = 0;
    if (threadIdx.x == 0) { *thr = 0ull; lock[0] = 0; lock[1] = 0; }
  }
  __device__ __forceinline__ uint64_t threshold() const { return *reinterpret_cast<volatile unsigned long long*>(thr); }

  // x: a run sorted ASCENDING in registers (32*R <= kp keys).  Merge it into the list under the lock.
  template <int R>
  __device__ __forceinline__ void merge_locked(const uint64_t (&x)[R], int lane) {
    const uint64_t top = (uint64_t)__shfl_sync(0xffffffffu, (unsigned long long)x[R - 1], 31);   // best staged key
    if (top < threshold()) return;                            // nothing staged can still be in the top k (the bound only rises;
                                                              // '<': the quick-start bound is itself a staged key)
    // Acquire with the warp CONVERGED: lane 0 tries, the outcome is broadcast, every lane leaves the loop together.
    // (`if (lane == 0) while (CAS) ;` leaves lane 0 on its own path; the profiler then showed most of the shuffles and
    // __syncwarps of the critical section taking the WARPSYNC.COLLECTIVE slow path.)  The sleep
    // backs off: a spinning CAS competes with the holder for the shared-memory pipe.
    for (unsigned ns = 32;;) {
      int got = 0;
      if (lane == 0) got = atomicCAS(lock, 0, 1) == 0;
      if (__shfl_sync(0xffffffffu, got, 0)) break;
      __nanosleep(ns);
      if (ns < 512) ns <<= 1;
    }
    __syncwarp();
    __threadfence_block();
    if (top > list[k - 1]) {                                  // warp-uniform
      warp_merge_run<R>(list, kp, x, lane);
      if (lane == 0) atomicMax(thr, (unsigned long long)list[k - 1]);   // monotone: cta_quickstart may have set a higher bound
    }
    __threadfence_block();
    __syncwarp();
    if (lane == 0) atomicExch(lock, 0);
  }
  // force == false: if another warp holds the lock, do nothing -- the caller keeps scanning and retries at its next
  // push (a warp that waits for the lock does no work AND its spinning slows the holder down).
  __device__ __forceinline__ void flush(int lane, bool force) {
    if (cnt == 0) return;
    if (!force) {                                              // one lane looks, all lanes agree (a per-lane read could split the warp)
      int busy = 0;
      if (lane == 0) busy = *reinterpret_cast<volatile int*>(lock);
      if (__shfl_sync(0xffffffffu, busy, 0)) return;
    }
    merge_staged<4>(buf, cnt, kp, lane, [&](const auto& x) { merge_locked(x, lane); });
    __syncwarp();
    cnt = 0;
  }
  __device__ __forceinline__ void push(bool pass, uint64_t key, int lane) {
    const int n = warp_append(buf, cnt, pass, key, lane);
    if (n == 0) return;
    cnt += n;
    __syncwarp();
    if (cnt > 32) flush(lane, cnt > kStage - 32);
  }
  // Threshold quick start (every thread calls it; this warp has staged its first 32*R keys, R = 1 or 2, zeros for
  // missing vectors).  Each warp sorts its own keys in registers and reports its q-th best, q = ceil(k / nw); the
  // minimum of those nw values is a valid lower bound of the CTA's k-th best (at least nw * q >= k staged keys are
  // >= it), published after ONE barrier -- no cross-warp merge at all (the merge tree of cta_bootstrap costs log2(nw)
  // + 3 barriers).  Each warp keeps the keys >= the bound staged; they reach the list
  // through the ordinary flushes.  k > 32 * R * nw: no bound can be given, everything stays staged.
  __device__ __forceinline__ void cta_quickstart(int nw, int R, int lane, int warp) {
    uint64_t x[2] = {buf[lane], R == 2 ? buf[lane + 32] : 0ull};
    reg_sort<2>(x, lane);                                            // descending: x[0] = ranks 0..31, x[1] = ranks 32..63
    const int q = (k + nw - 1) / nw;
    uint64_t mine = 0ull;
    if (q <= 32 * R) {
      const uint64_t a = (uint64_t)__shfl_sync(0xffffffffu, (unsigned long long)x[0], (q - 1) & 31);
      const uint64_t b = (uint64_t)__shfl_sync(0xffffffffu, (unsigned long long)x[1], (q - 1) & 31);
      mine = q <= 32 ? a : b;
    }
    if (lane == 0) rep()[warp] = mine;                               // written once per CTA
    __syncthreads();
    uint64_t bound = rep()[lane < nw ? lane : 0];
    #pragma unroll 1
    for (int o = 16; o > 0; o >>= 1) bound = key_min(bound, shfl_xor64(bound, o));
    if (threadIdx.x == 0) atomicMax(thr, (unsigned long long)bound);
    // keep what can still matter: keys >= bound (the bound is itself one of the keys), a prefix of the sorted run
    const bool k0 = x[0] != 0ull && x[0] >= bound, k1 = x[1] != 0ull && x[1] >= bound;
    const unsigned m0 = __ballot_sync(0xffffffffu, k0), m1 = __ballot_sync(0xffffffffu, k1);
    if (k0) buf[lane] = x[0];
    if (k1) buf[32 + lane] = x[1];
    cnt = __popc(m0) + __popc(m1);
    __syncwarp();
  }
  // Whole-CTA bootstrap (every thread calls it; every warp has staged exactly 32*R keys, R = 1 or 2, zeros for
  // missing vectors): each warp sorts its run in registers, the runs are merged pairwise in a log2(nw)-level tree
  // (runs are capped at kp keys), and warp 0 merges the survivor into the list and publishes the threshold --
  // log2(nw) + 3 barriers instead of a CTA-wide bitonic sort (45 barriers for 512 keys) or nw lock-serialised flushes.
  // The staging area of all warps (nw * kStage keys) is used as nw runs 64 keys apart; nw a power of two.
  __device__ __forceinline__ void cta_bootstrap(int nw, int R, int lane, int warp) {
    uint64_t* scratch = this->scratch();
    int len;                                                         // run length per warp
    uint64_t x[2];
    if (R == 1) {
      uint64_t y[1] = {buf[lane]};
      reg_sort<1>(y, lane);
      x[0] = y[0]; x[1] = 0ull;
      len = 32;
    } else {
      x[0] = buf[lane]; x[1] = buf[lane + 32];
      reg_sort<2>(x, lane);
      len = kp < 64 ? 32 : 64;                                      // kp == 32: only the top half can matter
    }
    __syncthreads();                                                 // every warp holds its run in registers
    uint64_t* mine = scratch + (size_t)warp * 64;
    mine[lane] = x[0];
    if (len == 64) mine[lane + 32] = x[1];
    __syncthreads();
    for (int s = 1; s < nw; s <<= 1) {
      const bool top_only = 2 * len > kp;
      if ((warp & (2 * s - 1)) == 0 && warp + s < nw) {
        uint64_t* A = scratch + (size_t)warp * 64;
        uint64_t* B = scratch + (size_t)(warp + s) * 64;
        warp_merge_runs(A, B, len, top_only, lane);
        if (!top_only && B != A + len) {                             // 32-key runs: close the gap
          for (int t = lane; t < len; t += 32) A[len + t] = B[t];
        }
      }
      if (!top_only) len <<= 1;
      __syncthreads();
    }
    if (warp == 0) {
      warp_merge_desc(list, kp, scratch, len, lane);
      if (lane == 0) atomicMax(thr, (unsigned long long)list[k - 1]);
    }
    cnt = 0;
    __syncthreads();
  }
  // End of the scan (every thread calls it): the leftovers of all warps that still beat the threshold are appended
  // to one array (most are stale by now: the threshold rose after they were staged) and warp 0 merges them, 64 at a
  // time -- three barriers, no lock, no queue of eight warps finishing together.
  __device__ __forceinline__ void cta_drain(int lane, int warp) {
    uint64_t* all = scratch();
    const uint64_t t = threshold();
    uint64_t e[3];
    #pragma unroll
    for (int c = 0; c < 3; ++c) {
      const int i = c * 32 + lane;
      const uint64_t v = i < cnt ? buf[i] : 0ull;
      e[c] = v >= t ? v : 0ull;                                      // '>=': the quick-start bound is itself a staged key
    }
    __syncthreads();                                                 // leftovers are in registers: the staging area is scratch now
    #pragma unroll
    for (int c = 0; c < 3; ++c) {                                    // warp_append behind a base reserved from the CTA's counter
      const unsigned m = __ballot_sync(0xffffffffu, e[c] != 0ull);
      if (m) {
        int base = 0;
        if (lane == 0) base = atomicAdd(lock + 1, __popc(m));
        base = __shfl_sync(0xffffffffu, base, 0);
        if (e[c] != 0ull) all[base + __popc(m & ((1u << lane) - 1))] = e[c];
      }
    }
    __syncthreads();
    if (warp == 0) {
      const int total = *reinterpret_cast<volatile int*>(lock + 1);
      for (int c0 = 0; c0 < total; c0 += 64)
        merge_staged<2>(all + c0, min(total - c0, 64), kp, lane, [&](const auto& x) { warp_merge_run(list, kp, x, lane); });
    }
    cnt = 0;
    __syncthreads();
  }
};
#endif  // __CUDACC__

}  // namespace tpq
