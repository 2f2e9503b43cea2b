// Fused IVF list scan + top-k over the REFERENCE storage layout.
//
// Exact drop-in for the reference's inner op (same argument list, same layouts):
//   fn.IVFPQTopk.topk                       torchpq/fn/IVFPQTopk.py:54-104
//   IVFPQTopkCuda.topk                      torchpq/kernels/IVFPQTopkCuda.py:81-142
//   __global__ ivfpq_topk / ivfpq_top1      torchpq/kernels/cuda/ivfpq_topk.cu:822-971, ivfpq_top1.cu:384-455
//
// Not a port: one CTA per query, but each WARP owns 32 consecutive addresses at a
// time (one coalesced 128-byte load per 4-sub-quantizer plane) and filters against the
// CTA-wide running k-th best (so the common case is one compare + one ballot per 32
// vectors, no barrier); survivors go to a per-warp staging buffer that is merged into
// the CTA's single sorted top-k list under a lock (CtaTopK, common.cuh).  Scores are accumulated exactly as the reference
// does: fp32, sub-quantizer 0..M-1 ascending, starting from 0.f.
#include "common.cuh"

namespace tpq {

struct RefScanSmem {
  // byte offsets into dynamic shared memory
  size_t lut, seg_start, seg_size, seg_prefix, topk, total;
};

static RefScanSmem ref_scan_smem(int M, int n_probe, int nw, int kp) {
  RefScanSmem s;
  size_t off = 0;
  s.lut = off;        off += (size_t)M * 256 * sizeof(float);
  s.seg_start = off;  off += (size_t)n_probe * sizeof(int64_t);
  s.seg_size = off;   off += (size_t)n_probe * sizeof(int32_t);
  s.seg_prefix = off; off += (size_t)(n_probe + 1) * sizeof(int32_t);
  off = align_up(off, 8);
  s.topk = off;       off += CtaTopK::bytes(nw, kp);
  s.total = off;
  return s;
}

__global__ void __launch_bounds__(256)
ivfpq_topk_ref_kernel(const uint32_t* __restrict__ data,        // [M/4, n_data] words (4 codes each)
                      const float* __restrict__ precomputed,    // [M, nq, 256]
                      const uint8_t* __restrict__ is_empty,     // [n_data]
                      const int64_t* __restrict__ cell_start,   // [nq, n_probe]
                      const int64_t* __restrict__ cell_size,    // [nq, n_probe]
                      const int64_t* __restrict__ n_probe_list, // [nq]
                      int64_t n_data, int M, int nq, int n_probe, int k, int kp,
                      RefScanSmem L,
                      float* __restrict__ values, int64_t* __restrict__ address) {
  extern __shared__ __align__(16) uint8_t smem[];
  float*    lut        = reinterpret_cast<float*>(smem + L.lut);
  int64_t*  seg_start  = reinterpret_cast<int64_t*>(smem + L.seg_start);
  int32_t*  seg_size   = reinterpret_cast<int32_t*>(smem + L.seg_size);
  int32_t*  seg_prefix = reinterpret_cast<int32_t*>(smem + L.seg_prefix);

  const int q = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;

  // --- stage this query's LUT rows: precomputed[m, q, :] -> lut[m*256 ..]  (load_precomputed_v1, ivfpq_topk.cu:462-486)
  for (int i = tid; i < M * 64; i += blockDim.x) {
    int m = i >> 6, c4 = i & 63;
    reinterpret_cast<float4*>(lut)[i] =
        reinterpret_cast<const float4*>(precomputed + ((size_t)m * nq + q) * 256)[c4];
  }
  // --- probe segments.  nProbe is read as a 32-bit int (ivfpq_topk.cu:837); cell 0 is always
  //     entered (:850-856); an entry whose start equals the previous entry's start is skipped (:864-866).
  int P = (int)n_probe_list[q];
  P = max(1, min(P, n_probe));
  if (warp == 0) {
    int carry = 0;
    if (lane == 0) seg_prefix[0] = 0;
    for (int j0 = 0; j0 < P; j0 += 32) {
      int j = j0 + lane;
      int chunks = 0;
      if (j < P) {
        int64_t s = cell_start[(size_t)q * n_probe + j];
        int64_t n = cell_size[(size_t)q * n_probe + j];
        bool skip = (j > 0) && (s == cell_start[(size_t)q * n_probe + j - 1]);
        if (n < 0 || skip) n = 0;
        seg_start[j] = s;
        seg_size[j] = (int)n;
        chunks = (int)((n + 31) >> 5);
      }
      const int incl = warp_inclusive_scan(chunks, lane);
      if (j < P) seg_prefix[j + 1] = carry + incl;
      carry += __shfl_sync(0xffffffffu, incl, 31);
    }
  }
  CtaTopK tk;
  tk.init(smem + L.topk, nw, warp, kp, k);
  __syncthreads();

  const int total_chunks = seg_prefix[P];
  const int nplanes = M >> 2;
  int seg = 0;
  for (int c = warp; c < total_chunks; c += nw) {
    while (c >= seg_prefix[seg + 1]) ++seg;
    const int64_t s0 = seg_start[seg];
    const int64_t a = s0 + (int64_t)(c - seg_prefix[seg]) * 32 + lane;
    bool live = a < s0 + seg_size[seg];
    if (live) live = (is_empty[a] == 0);                       // ivfpq_topk.cu:878,883-884
    float score = 0.f;
    if (live) {
      const uint32_t* p = data + a;
      #pragma unroll 4
      for (int g = 0; g < nplanes; ++g) {                       // load_data / consume_data, ivfpq_topk.cu:650-679
        uint32_t w = __ldg(p + (size_t)g * n_data);
        const float* t = lut + (g << 10);
        score += t[w & 0xff];
        score += t[256 + ((w >> 8) & 0xff)];
        score += t[512 + ((w >> 16) & 0xff)];
        score += t[768 + (w >> 24)];
      }
    }
    const uint64_t key = make_key(score, (uint32_t)a);
    tk.push(live && key > tk.threshold(), key, lane);
  }
  tk.flush(lane, true);
  __syncthreads();
  // write-out: descending, (-inf, -1) padded  (ivfpq_topk.cu:966-970; IVFPQTopkCuda.py:118-120,142)
  for (int i = tid; i < k; i += blockDim.x) {
    uint64_t key = tk.list[i];
    values[(size_t)q * k + i]  = key ? key_score(key) : -INFINITY;
    address[(size_t)q * k + i] = key ? (int64_t)key_addr(key) : -1;
  }
}

}  // namespace tpq

using namespace tpq;

extern "C" size_t tpq_ivfpq_topk_workspace_bytes(int nq, int k) { (void)nq; (void)k; return 0; }

extern "C" int tpq_ivfpq_topk(const uint8_t* data, const float* precomputed, const uint8_t* is_empty,
                              const int64_t* cell_start, const int64_t* cell_size, const int64_t* n_probe_list,
                              int64_t n_data, int M, int nq, int n_probe, int k,
                              float* values, int64_t* address, void* ws, size_t ws_bytes, void* stream) {
  (void)ws; (void)ws_bytes;
  // the reference's asserts: IVFPQTopkCuda.py:98-114, fn/IVFPQTopk.py:64
  TPQ_REQUIRE(0 < k && k <= 1024, "k must be in (0, 1024], got %d", k);
  TPQ_REQUIRE(M > 0 && M % 4 == 0, "n_subvectors must be a positive multiple of 4, got %d", M);
  TPQ_REQUIRE(nq >= 0 && n_probe > 0, "bad n_query=%d / n_probe=%d", nq, n_probe);
  TPQ_REQUIRE(n_data >= 0 && n_data <= 0xFFFFFFFFll, "n_data=%lld exceeds the 32-bit address range", (long long)n_data);
  TPQ_REQUIRE(data && precomputed && is_empty && cell_start && cell_size && n_probe_list && values && address,
              "null pointer argument");
  TPQ_REQUIRE((reinterpret_cast<uintptr_t>(data) & 3) == 0 && (reinterpret_cast<uintptr_t>(precomputed) & 15) == 0,
              "data must be 4-byte and precomputed 16-byte aligned");
  if (nq == 0) return TPQ_OK;
  const int kp = list_capacity(k);
  int nw = 8;
  RefScanSmem L = ref_scan_smem(M, n_probe, nw, kp);
  while (L.total > kSmemLimit && nw > 1) { nw >>= 1; L = ref_scan_smem(M, n_probe, nw, kp); }
  if (L.total > kSmemLimit) {
    set_error("ivfpq_topk: M=%d, n_probe=%d, k=%d needs %zu bytes of shared memory (> 227 KB)", M, n_probe, k, L.total);
    return TPQ_ERR_UNSUPPORTED;
  }
  TPQ_CUDA(cudaFuncSetAttribute(ivfpq_topk_ref_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)L.total));
  ivfpq_topk_ref_kernel<<<nq, nw * 32, L.total, (cudaStream_t)stream>>>(
      reinterpret_cast<const uint32_t*>(data), precomputed, is_empty, cell_start, cell_size, n_probe_list,
      n_data, M, nq, n_probe, k, kp, L, values, address);
  TPQ_LAUNCH_CHECK("ivfpq_topk_ref_kernel");
  return TPQ_OK;
}
