// SQCodec.encode / decode (torchpq codec/SQCodec.py): per-dimension scalar quantization of a [d, n] fp32 matrix.
//
// 8 bits, with lower / range [d] f32 (range = upper - lower + 1e-8, as trained by the codec):
//   encode  code = clamp(rint(((x - lower) / range) * 256), 0, 255)   each step rounded on its own, rint half to even
//   decode  x'   = ((code / 256) * range) + lower                      two roundings, no fma (code / 256 is exact)
// These are the reference's torch expressions op for op, so both directions are bit-identical to it.  The reference's
// quirks follow: x == upper encodes to 256, clamped to 255; code 255 decodes to lower + 255/256 range, never to upper.
// A NaN encodes to 0 (the reference's uint8 cast of a NaN is undefined).
// 16 bits: __float2half_rn / __half2float (torch's .half() / .float(): beyond +-65504 becomes +-inf).
// 32 bits: a copy.  The decode of 8 bits is also what IVFSQIndex's scan stages into its GEMM tile (gemm_tile.cuh,
// BLoadSQ8), so the two agree by construction.
#include <cuda_fp16.h>
#include "common.cuh"

namespace tpq {

// grid (column blocks, row groups): thread per column, rows g = blockIdx.y, blockIdx.y + gridDim.y, ...
template <int BITS>
__global__ void sq_encode_kernel(const float* __restrict__ x, int d, int64_t n, const float* __restrict__ lower,
                                 const float* __restrict__ range, void* __restrict__ out) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  for (int g = blockIdx.y; g < d; g += gridDim.y) {
    const size_t i = (size_t)g * n + j;
    if (BITS == 8) {
      const float q = rintf(__fmul_rn(__fdiv_rn(__fsub_rn(x[i], lower[g]), range[g]), 256.f));
      reinterpret_cast<uint8_t*>(out)[i] = (uint8_t)fminf(fmaxf(q, 0.f), 255.f);   // fmaxf(NaN, 0) = 0
    } else {
      reinterpret_cast<__half*>(out)[i] = __float2half_rn(x[i]);
    }
  }
}

template <int BITS>
__global__ void sq_decode_kernel(const void* __restrict__ codes, int d, int64_t n, const float* __restrict__ lower,
                                 const float* __restrict__ range, float* __restrict__ out) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  for (int g = blockIdx.y; g < d; g += gridDim.y) {
    const size_t i = (size_t)g * n + j;
    if (BITS == 8) {
      const float q = __fmul_rn((float)reinterpret_cast<const uint8_t*>(codes)[i], 0.00390625f);   // code / 256, exact
      out[i] = __fadd_rn(__fmul_rn(q, range[g]), lower[g]);
    } else {
      out[i] = __half2float(reinterpret_cast<const __half*>(codes)[i]);
    }
  }
}

static int sq_check(const char* name, const void* in, int d, int64_t n, int bits, const float* lower,
                    const float* range, const void* out) {
  if (bits != 8 && bits != 16 && bits != 32) {
    set_error("%s: bits=%d is not supported (8, 16 and 32 only)", name, bits);
    return TPQ_ERR_UNSUPPORTED;
  }
  TPQ_REQUIRE(d > 0 && n >= 0, "%s: bad sizes d=%d n=%lld", name, d, (long long)n);
  TPQ_REQUIRE(n == 0 || (in && out), "%s: null input or output", name);
  TPQ_REQUIRE(bits != 8 || (lower && range), "%s: null lower or range (8 bits)", name);
  return TPQ_OK;
}

static dim3 sq_grid(int d, int64_t n) {
  return dim3((unsigned)((n + 255) / 256), (unsigned)(d < 64 ? d : 64));
}

}  // namespace tpq

using namespace tpq;

extern "C" int tpq_sq_encode(const float* x_dn, int d, int64_t n, int bits, const float* lower, const float* range,
                             void* out, void* stream) {
  if (int rc = sq_check("tpq_sq_encode", x_dn, d, n, bits, lower, range, out)) return rc;
  if (n == 0) return TPQ_OK;
  cudaStream_t st = (cudaStream_t)stream;
  if (bits == 32) {
    TPQ_CUDA(cudaMemcpyAsync(out, x_dn, (size_t)d * n * 4, cudaMemcpyDeviceToDevice, st));
    return TPQ_OK;
  }
  if (bits == 8) sq_encode_kernel<8><<<sq_grid(d, n), 256, 0, st>>>(x_dn, d, n, lower, range, out);
  else sq_encode_kernel<16><<<sq_grid(d, n), 256, 0, st>>>(x_dn, d, n, lower, range, out);
  TPQ_LAUNCH_CHECK("sq_encode_kernel");
  return TPQ_OK;
}

extern "C" int tpq_sq_decode(const void* codes, int d, int64_t n, int bits, const float* lower, const float* range,
                             float* out_dn, void* stream) {
  if (int rc = sq_check("tpq_sq_decode", codes, d, n, bits, lower, range, out_dn)) return rc;
  if (n == 0) return TPQ_OK;
  cudaStream_t st = (cudaStream_t)stream;
  if (bits == 32) {
    TPQ_CUDA(cudaMemcpyAsync(out_dn, codes, (size_t)d * n * 4, cudaMemcpyDeviceToDevice, st));
    return TPQ_OK;
  }
  if (bits == 8) sq_decode_kernel<8><<<sq_grid(d, n), 256, 0, st>>>(codes, d, n, lower, range, out_dn);
  else sq_decode_kernel<16><<<sq_grid(d, n), 256, 0, st>>>(codes, d, n, lower, range, out_dn);
  TPQ_LAUNCH_CHECK("sq_decode_kernel");
  return TPQ_OK;
}
