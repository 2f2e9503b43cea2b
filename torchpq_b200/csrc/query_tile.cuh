// The query tile of the two re-rank passes (rerank.cu, refine.cu): a persistent CTA takes up to one query per warp at
// a time, scores each query's k1 candidates into keys [qt, k1] in shared memory, then each warp keeps its query's best
// k.  Only the per-candidate scoring differs between the passes; these are the two steps around it.
#pragma once
#include "common.cuh"

namespace tpq {

// Args: a pass's kernel arguments, with x [d, nq] (d passed as given), nq, k, kp (the list's slots) and keys_out.

// xs [nqt, d] <- the tile's queries, columns q0 .. q0 + nqt - 1 of A.x; every thread of the CTA takes part
template <int NT, class Args>
__device__ __forceinline__ void load_query_tile(const Args& A, float* xs, int d, int q0, int nqt, int tid) {
  for (int i = tid; i < nqt * d; i += NT) {
    const int q = i / d, e = i - q * d;
    xs[i] = A.x[(size_t)e * A.nq + q0 + q];
  }
}

// warp w < nqt: query w's k1 keys, 64 at a time, into its kp-slot list (merge_staged + warp_merge_run); its first k
// keys go to row q0 + w of A.keys_out [nq, k]
template <class Args>
__device__ __forceinline__ void select_query_tile(const Args& A, const uint64_t* keys, uint64_t* lists, int k1, int nqt,
                                                  int q0, int warp, int lane) {
  if (warp < nqt) {
    uint64_t* list = lists + (size_t)warp * A.kp;
    for (int i = lane; i < A.kp; i += 32) list[i] = 0ull;
    __syncwarp();
    const uint64_t* kq = keys + (size_t)warp * k1;
    for (int c0 = 0; c0 < k1; c0 += 64)
      merge_staged<2>(kq + c0, min(k1 - c0, 64), A.kp, lane, [&](const auto& x) { warp_merge_run(list, A.kp, x, lane); });
    uint64_t* dst = A.keys_out + (size_t)(q0 + warp) * A.k;
    for (int i = lane; i < A.k; i += 32) dst[i] = list[i];
  }
}

}  // namespace tpq
