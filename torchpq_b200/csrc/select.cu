// Row-wise top-k of a dense matrix (fn.Topk, torchpq/fn/Topk.py:43-67, whose kernels are top1_select.cu,
// top32_select.cu and topk_select.cu).
//
// x [m, n] fp32 or fp16, row-major -> the k best (value, column) of every row, in the library's total order: value
// descending, then column ascending, +0 above -0, every NaN above +inf.  One pass over x with 128-bit streaming loads.
// A plan (plan_topk), read by the workspace size and the launch, picks one of two shapes:
//   rows:   many rows (m >= 16 per SM): one warp per row with a WarpTopK in shared memory, which writes the row's
//           values and indices itself.
//   slices: few rows: each row is cut into S column slices so that the grid covers the SMs about twice; a CTA of 8
//           warps runs a CtaTopK over its slice (quick start on its first 512 keys, cta_drain at the end).  S == 1 writes
//           values and indices; S > 1 writes each slice's sorted keys to ws [m, S, k], and topk_parts_kernel selects the
//           top k of each row's S sorted parts, reading every part only down to its first key below the threshold.
#include <cuda_fp16.h>
#include "common.cuh"

namespace tpq {

constexpr int kRowWarps = 4;          // warps (rows) per CTA of topk_rows_kernel
constexpr int kSliceWarps = 8;        // warps per CTA of topk_slices_kernel and topk_parts_kernel
constexpr int64_t kMinSliceCols = 8192;

// The selector's key of one element: make_key's order, except that every NaN, of either sign and any payload, maps to
// the largest image (above +inf; it decodes as the NaN 0x7fffffff).  score_to_ord alone would put a negative NaN below
// -inf.  A real key is never 0: the smallest image is -inf's 0x007fffff.
__device__ __forceinline__ uint64_t topk_key(float v, int64_t c) {
  const uint32_t o = v != v ? 0xFFFFFFFFu : score_to_ord(v);
  return ((uint64_t)o << 32) | (uint64_t)(0xFFFFFFFFu - (uint32_t)c);
}
__device__ __forceinline__ float elem_value(float v) { return v; }
__device__ __forceinline__ float elem_value(__half v) { return __half2float(v); }   // exact

// U 16-byte vectors of V elements per lane and step: 16 keys in registers either way.
template <class T> struct Vec;
template <> struct Vec<float>  { static constexpr int V = 4, U = 4; };
template <> struct Vec<__half> { static constexpr int V = 8, U = 2; };

template <class T>
__device__ __forceinline__ T vec_elem(const uint4& w, int e) {
  T a[Vec<T>::V];
  memcpy(a, &w, 16);
  return a[e];
}

// The out-of-line flushes: a step pushes 16 keys, and sixteen inlined copies of the sort-and-merge would crowd the
// streaming loop out of the instruction cache.  Both return the staged count left behind.
__device__ __noinline__ int warp_flush(WarpTopK tk, int lane) { tk.flush(lane); return tk.cnt; }
__device__ __noinline__ int cta_flush(CtaTopK tk, int lane, bool force) { tk.flush(lane, force); return tk.cnt; }

// WarpTopK::push and CtaTopK::push with the flush out of line and the threshold cached per step.
struct WarpSink {
  WarpTopK tk;
  uint64_t t;
  int lane;
  __device__ __forceinline__ uint64_t thr() const { return t; }
  __device__ __forceinline__ void push(bool pass, uint64_t key) {
    tk.cnt += warp_append(tk.buf, tk.cnt, pass, key, lane);
    if (tk.cnt > kTopkBuf - 32) { __syncwarp(); tk.cnt = warp_flush(tk, lane); t = tk.kth(); }
  }
  __device__ __forceinline__ void finish() { __syncwarp(); tk.cnt = warp_flush(tk, lane); }
};
struct CtaSink {
  CtaTopK tk;
  int lane;
  __device__ __forceinline__ uint64_t thr() const { return tk.threshold(); }
  __device__ __forceinline__ void push(bool pass, uint64_t key) {
    tk.cnt += warp_append(tk.buf, tk.cnt, pass, key, lane);
    if (tk.cnt > 32) { __syncwarp(); tk.cnt = cta_flush(tk, lane, tk.cnt > kStage - 32); }
  }
};

// Push the keys of p[0 .. len) (columns col0 + i) into sink; warp w of nw.  A row need not start 16-byte aligned, so
// the elements before the first 16-byte boundary (head) and after the last (tail), fewer than V each, are one scalar
// step of warp 0; the rest are 16-byte streaming loads, U per lane in flight.  Every call of sink is warp-uniform.
template <class T, class Sink>
__device__ __forceinline__ void scan_span(const T* __restrict__ p, int64_t len, int64_t col0, int w, int nw, int lane,
                                          Sink& sink) {
  constexpr int V = Vec<T>::V, U = Vec<T>::U;
  int64_t head = (int64_t)(((16u - (unsigned)(reinterpret_cast<uintptr_t>(p) & 15u)) & 15u) / sizeof(T));
  if (head > len) head = len;
  const int64_t nv = (len - head) / V;
  const int64_t body_end = head + nv * V;
  if (w == 0 && len > 0) {
    const int64_t tail = len - body_end;
    const int64_t i = lane < head ? lane : body_end + (lane - head);
    const uint64_t key = lane < head + tail ? topk_key(elem_value(p[i]), col0 + i) : 0ull;
    const bool pass = key > sink.thr();
    if (__any_sync(0xffffffffu, pass)) sink.push(pass, key);
  }
  const uint4* vp = reinterpret_cast<const uint4*>(p + head);
  for (int64_t v0 = (int64_t)w * 32 * U; v0 < nv; v0 += (int64_t)nw * 32 * U) {
    uint4 r[U];
    #pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t v = v0 + u * 32 + lane;
      r[u] = v < nv ? __ldcs(vp + v) : make_uint4(0u, 0u, 0u, 0u);
    }
    const uint64_t t = sink.thr();
    uint64_t key[U * V];
    bool any = false;
    #pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t v = v0 + u * 32 + lane;
      #pragma unroll
      for (int e = 0; e < V; ++e) {
        const int64_t i = head + v * V + e;
        key[u * V + e] = v < nv ? topk_key(elem_value(vec_elem<T>(r[u], e)), col0 + i) : 0ull;
        any |= key[u * V + e] > t;
      }
    }
    if (__any_sync(0xffffffffu, any)) {                  // rare once the threshold has risen
      #pragma unroll
      for (int j = 0; j < U * V; ++j) sink.push(key[j] > t, key[j]);
    }
  }
}

// key -> (value, column); the missing entries of a row shorter than k are (-inf, -1)
__device__ __forceinline__ void put_key(float* values, int64_t* indices, size_t o, uint64_t key) {
  values[o] = key ? key_score(key) : -INFINITY;
  indices[o] = key ? (int64_t)key_addr(key) : -1;
}

// grid ceil(m / 4), 128 threads: warp w of CTA b owns row 4b + w.  Shared memory: 4 x (list [kp] | staging [64]).
template <class T>
__global__ void __launch_bounds__(32 * kRowWarps)
topk_rows_kernel(const T* __restrict__ x, int64_t m, int64_t n, int k, int kp,
                 float* __restrict__ values, int64_t* __restrict__ indices) {
  extern __shared__ __align__(16) uint8_t smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t r = (int64_t)blockIdx.x * kRowWarps + warp;
  if (r >= m) return;                                    // whole warp exits together
  uint64_t* base = reinterpret_cast<uint64_t*>(smem) + (size_t)warp * (kp + kTopkBuf);
  WarpSink s{{}, 0ull, lane};
  s.tk.init(base, base + kp, kp, k, lane);
  scan_span(x + (size_t)r * n, n, 0, 0, 1, lane, s);
  s.finish();
  for (int i = lane; i < k; i += 32) put_key(values, indices, (size_t)r * k + i, s.tk.list[i]);
}

// grid (m, S), 256 threads: CTA (r, s) selects over columns [s * slice_cols, (s + 1) * slice_cols) of row r.
// keys_out == nullptr (S == 1): writes values / indices; else the sorted keys to keys_out[(r * S + s) * k ..].
template <class T>
__global__ void __launch_bounds__(32 * kSliceWarps)
topk_slices_kernel(const T* __restrict__ x, int64_t n, int k, int kp, int64_t slice_cols,
                   uint64_t* __restrict__ keys_out, float* __restrict__ values, int64_t* __restrict__ indices) {
  extern __shared__ __align__(16) uint8_t smem[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t r = blockIdx.x, s = blockIdx.y;
  const int64_t c0 = s * slice_cols, c1 = c0 + slice_cols < n ? c0 + slice_cols : n;
  const T* row = x + (size_t)r * n;
  CtaSink sink{{}, lane};
  CtaTopK& tk = sink.tk;
  tk.init(smem, kSliceWarps, warp, kp, k);
  // quick start: warp w stages the slice's columns c0 + 64w .. c0 + 64w + 63 (scalar loads; 512 of the slice's keys)
  #pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int64_t c = c0 + warp * 64 + h * 32 + lane;
    tk.buf[h * 32 + lane] = c < c1 ? topk_key(elem_value(row[c]), c) : 0ull;
  }
  tk.cnt = 64;
  __syncthreads();                                       // init's list and threshold before the quick start
  tk.cta_quickstart(kSliceWarps, 2, lane, warp);
  const int64_t qs = c0 + 64 * kSliceWarps < c1 ? c0 + 64 * kSliceWarps : c1;
  scan_span(row + qs, c1 - qs, qs, warp, kSliceWarps, lane, sink);
  tk.cta_drain(lane, warp);
  for (int i = tid; i < k; i += 32 * kSliceWarps) {
    if (keys_out) keys_out[((size_t)r * gridDim.y + s) * k + i] = tk.list[i];
    else put_key(values, indices, (size_t)r * k + i, tk.list[i]);
  }
}

// grid m, 256 threads: the top k of row r's S sorted parts keys[r, 0 .. S, 0 .. k).  Warp w takes parts w, w + 8, ...
// and reads each 32 keys at a time, down to its first key that fails the threshold: the part is sorted and the
// threshold only rises, so nothing after that key can pass.  The column is the key's address.
__global__ void __launch_bounds__(32 * kSliceWarps)
topk_parts_kernel(const uint64_t* __restrict__ keys, int S, int k, int kp,
                  float* __restrict__ values, int64_t* __restrict__ indices) {
  extern __shared__ __align__(16) uint8_t smem[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t r = blockIdx.x;
  CtaSink sink{{}, lane};
  CtaTopK& tk = sink.tk;
  tk.init(smem, kSliceWarps, warp, kp, k);
  __syncthreads();
  const uint64_t* row = keys + (size_t)r * S * k;
  for (int p = warp; p < S; p += kSliceWarps) {
    const uint64_t* part = row + (size_t)p * k;
    for (int i0 = 0; i0 < k; i0 += 32) {
      const uint64_t key = i0 + lane < k ? __ldcg(part + i0 + lane) : 0ull;
      const bool pass = key > sink.thr();
      if (__any_sync(0xffffffffu, pass)) sink.push(pass, key);
      if (__any_sync(0xffffffffu, !pass)) break;
    }
  }
  tk.cta_drain(lane, warp);
  for (int i = tid; i < k; i += 32 * kSliceWarps) put_key(values, indices, (size_t)r * k + i, tk.list[i]);
}

// The plan, read by the workspace size and the launch.
//   rows:  m >= 16 rows per SM, enough warps to keep every SM streaming.  kp = 1024: 4 x 1088 keys = 34 KB per CTA.
//   S:     enough slices that m * S CTAs cover the SMs twice, each at least max(8192, 8k) columns (a slice shorter
//          than that adds more keys to the second pass than it takes reading off the first) and a multiple of 64
//          columns, so that a slice starts at the same 16-byte phase as its row.  The workspace holds m * S * k keys.
struct TopkPlan {
  bool rows;
  int kp, S;
  int64_t slice_cols;
  size_t smem, ws;
};

static TopkPlan plan_topk(int64_t m, int64_t n, int k) {
  TopkPlan P{};
  P.kp = list_capacity(k);
  const int sms = device_sm_count();
  P.rows = m >= 16 * (int64_t)sms;
  P.S = 1;
  P.slice_cols = n;
  if (P.rows) {
    P.smem = (size_t)kRowWarps * (P.kp + kTopkBuf) * 8;
    return P;
  }
  P.smem = CtaTopK::bytes(kSliceWarps, P.kp);
  const int64_t min_cols = k * 8 > kMinSliceCols ? (int64_t)k * 8 : kMinSliceCols;
  int64_t S = (2 * (int64_t)sms + m - 1) / m;
  if (S > n / min_cols) S = n / min_cols;
  if (S > 1) {
    const int64_t per = ((n + S - 1) / S + 63) / 64 * 64;
    P.S = (int)((n + per - 1) / per);
    P.slice_cols = per;
  }
  if (P.S > 1) P.ws = (size_t)m * P.S * k * 8;
  return P;
}

template <class T>
static int launch_topk(const TopkPlan& P, const T* x, int64_t m, int64_t n, int k, float* values, int64_t* indices,
                       uint64_t* ws, cudaStream_t st) {
  if (P.rows) {
    TPQ_CUDA(cudaFuncSetAttribute(topk_rows_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)P.smem));
    topk_rows_kernel<T><<<(unsigned)((m + kRowWarps - 1) / kRowWarps), 32 * kRowWarps, P.smem, st>>>(
        x, m, n, k, P.kp, values, indices);
    TPQ_LAUNCH_CHECK("topk_rows_kernel");
    return TPQ_OK;
  }
  TPQ_CUDA(cudaFuncSetAttribute(topk_slices_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)P.smem));
  topk_slices_kernel<T><<<dim3((unsigned)m, P.S), 32 * kSliceWarps, P.smem, st>>>(
      x, n, k, P.kp, P.slice_cols, P.S > 1 ? ws : nullptr, values, indices);
  TPQ_LAUNCH_CHECK("topk_slices_kernel");
  if (P.S == 1) return TPQ_OK;
  TPQ_CUDA(cudaFuncSetAttribute(topk_parts_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)P.smem));
  topk_parts_kernel<<<(unsigned)m, 32 * kSliceWarps, P.smem, st>>>(ws, P.S, k, P.kp, values, indices);
  TPQ_LAUNCH_CHECK("topk_parts_kernel");
  return TPQ_OK;
}

static bool topk_dtype(int dtype) { return dtype == TPQ_DTYPE_F32 || dtype == TPQ_DTYPE_F16; }
constexpr int64_t kMaxCols = int64_t(1) << 32;

}  // namespace tpq

using namespace tpq;

extern "C" size_t tpq_topk_workspace_bytes(int64_t m, int64_t n, int k, int dtype) {
  if (m <= 0 || n < 0 || n >= kMaxCols || k <= 0 || k > 1024 || !topk_dtype(dtype)) return 0;
  return plan_topk(m, n, k).ws;
}

extern "C" int tpq_topk(const void* x, int64_t m, int64_t n, int dtype, int k, float* values, int64_t* indices,
                        void* ws, size_t ws_bytes, void* stream) {
  TPQ_REQUIRE(k > 0, "tpq_topk: k must be in [1, 1024], got %d", k);
  if (k > 1024) { set_error("tpq_topk: k=%d > 1024 is not supported", k); return TPQ_ERR_UNSUPPORTED; }
  if (!topk_dtype(dtype)) { set_error("tpq_topk: unsupported dtype %d", dtype); return TPQ_ERR_UNSUPPORTED; }
  TPQ_REQUIRE(m >= 0 && n >= 0, "tpq_topk: bad sizes m=%lld n=%lld", (long long)m, (long long)n);
  if (n >= kMaxCols) {
    set_error("tpq_topk: n=%lld exceeds the 32-bit column of a key", (long long)n);
    return TPQ_ERR_UNSUPPORTED;
  }
  if (m == 0) return TPQ_OK;
  TPQ_REQUIRE((x || n == 0) && values && indices, "tpq_topk: null pointer");   // empty rows read nothing
  const TopkPlan P = plan_topk(m, n, k);
  if (P.ws > 0 && (!ws || ws_bytes < P.ws)) {
    set_error("tpq_topk: workspace too small (%zu < %zu)", ws_bytes, P.ws);
    return TPQ_ERR_WORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  uint64_t* keys = reinterpret_cast<uint64_t*>(ws);
  if (dtype == TPQ_DTYPE_F16)
    return launch_topk(P, reinterpret_cast<const __half*>(x), m, n, k, values, indices, keys, st);
  return launch_topk(P, reinterpret_cast<const float*>(x), m, n, k, values, indices, keys, st);
}
