"""The reference's own row-wise select kernels, built into oracle/_ref/ and launched on torch tensors (TEST
INFRASTRUCTURE ONLY).

Build (python oracle/ref_select.py, run by __graft_entry__.build()): where the reference sources exist, compile
top1_select.cu, top32_select.cu and topk_select.cu unmodified, specialised the way their Python wrappers specialise
them (Top1SelectCuda.py, Top32SelectCuda.py, TopkSelectCuda.py: textual _TPB_ / _QCAP_ / _TN_ substitution, NVRTC
options --use_fast_math -lineinfo), once per (tpb, queue capacity, buffer size) that fn.Topk.__init__ constructs
(fn/Topk.py:6-41), together with a small host launcher of ours.  Only the .so files land in oracle/_ref/.

Launch: topk(x, k) restates Topk.__call__'s dispatch on k (fn/Topk.py:52-67) and each wrapper's host logic: values
[m, next_pow2(k)] filled with -inf, the grid (ceil(m / warps per block) for top1 / top32, m for topk_select), the slice
[:, :k].  The wrappers leave the indices as torch.empty; here they start at -1 so that a comparison is reproducible.
"""
import ctypes as C
import math
import os
import subprocess
import sys
import tempfile

REF = "/root/reference/torchpq/kernels/cuda"
HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref")

# (file, tpb, queue capacity, buffer size) per range of k, as fn/Topk.py:6-41 builds them
CONFIGS = {
    "top1": ("top1_select", 256, 1, 4),
    "top32": ("top32_select", 256, 1, 4),
    "top64": ("topk_select", 64, 4, 4),
    "top128": ("topk_select", 128, 4, 4),
    "top256": ("topk_select", 256, 4, 4),
    "top512": ("topk_select", 512, 2, 2),
    "top1024": ("topk_select", 1024, 2, 2),
}

LAUNCHER = r'''
#include <cuda_runtime.h>
extern "C" int ref_select_launch(const void* x, void* values, long long* indices, int m, int n, int kpow2, int fp16,
                                 void* stream) {
  const dim3 grid(%(GRID)s);
  %(CALL)s
  return (int)cudaGetLastError();
}
'''


def lib_name(tag):
    return os.path.join(OUT, f"libref_select_{tag}.so")


def available(tags=tuple(CONFIGS)) -> bool:
    return all(os.path.exists(lib_name(t)) for t in tags)


def build_select(tag):
    fname, tpb, qcap, tn = CONFIGS[tag]
    src = open(os.path.join(REF, f"{fname}.cu")).read()
    code = src.replace("_TPB_", str(tpb)).replace("_QCAP_", str(qcap)).replace("_TN_", str(tn))
    # NVRTC compiles device code only; nvcc's host pass sees __CUDA_ARCH__ undefined, takes the source's pre-Volta
    # `#if (__CUDA_ARCH__ < 700)` stand-in for __nanosleep and clashes with the runtime's declaration.  A one-line
    # prelude renames that host-pass copy; the device code and the reference text are untouched.
    code = "#ifndef __CUDA_ARCH__\n#define __nanosleep ref_host_nanosleep\n#endif\n" + code
    st = "(cudaStream_t)stream"
    if fname == "topk_select":                                   # fp32 only (TopkSelectCuda.py:66)
        grid = "m"
        call = (f"if (fp16) return -1;\n  {fname}<<<grid, {tpb}, 0, {st}>>>((const float*)x, (float*)values, indices, "
                "m, n, kpow2);")
    else:
        grid = f"(m + {tpb // 32} - 1) / {tpb // 32}"
        call = (f"if (fp16) {fname}_fp16<<<grid, {tpb}, 0, {st}>>>((const __half*)x, (__half*)values, indices, m, n, "
                f"kpow2);\n  else {fname}<<<grid, {tpb}, 0, {st}>>>((const float*)x, (float*)values, indices, m, n, "
                "kpow2);")
    code += LAUNCHER % {"GRID": grid, "CALL": call}
    os.makedirs(OUT, exist_ok=True)
    out = lib_name(tag)
    with tempfile.TemporaryDirectory() as td:
        cu = os.path.join(td, f"ref_select_{tag}.cu")
        open(cu, "w").write(code)
        subprocess.check_call(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-use_fast_math",
                               "-lineinfo", "-shared", "-Xcompiler", "-fPIC", "-w", "-o", out, cu])
    return out


def tag_of(k):
    """fn/Topk.py:52-67; None where the reference calls torch.topk."""
    if k == 1:
        return "top1"
    for cap in (32, 64, 128, 256, 512, 1024):
        if k <= cap:
            return f"top{cap}"
    return None


_libs = {}


def topk(x, k):
    """The reference's torchpq.topk(x, k) for a 2-D contiguous CUDA tensor, 1 <= k <= 1024 -> (values in x.dtype,
    indices i64).  fp16 only for k <= 32, as in the reference."""
    import torch
    tag = tag_of(k)
    assert tag is not None and x.dim() == 2 and x.is_contiguous()
    assert x.dtype == torch.float32 or (x.dtype == torch.float16 and k <= 32)
    if tag not in _libs:
        lib = C.CDLL(lib_name(tag))
        lib.ref_select_launch.restype = C.c_int
        lib.ref_select_launch.argtypes = [C.c_void_p] * 3 + [C.c_int] * 4 + [C.c_void_p]
        _libs[tag] = lib
    m, n = x.shape
    kpow2 = 1 if k == 0 else 2 ** math.ceil(math.log2(k))
    values = torch.full((m, kpow2), float("-inf"), device=x.device, dtype=x.dtype)
    indices = torch.full((m, kpow2), -1, device=x.device, dtype=torch.int64)
    rc = _libs[tag].ref_select_launch(x.data_ptr(), values.data_ptr(), indices.data_ptr(), m, n, kpow2,
                                      int(x.dtype == torch.float16),
                                      C.c_void_p(torch.cuda.current_stream(x.device).cuda_stream))
    if rc != 0:
        raise RuntimeError(f"reference select launch failed: cudaError {rc}")
    return values[:, :k], indices[:, :k]


def main():
    if not os.path.isdir(REF):
        print("oracle/_ref: reference sources not present; keeping prebuilt select kernels")
        return 0
    for tag in CONFIGS:
        if not os.path.exists(lib_name(tag)) or os.path.getmtime(lib_name(tag)) < os.path.getmtime(__file__):
            build_select(tag)
        print("built", os.path.relpath(lib_name(tag), HERE))
    return 0


if __name__ == "__main__":
    sys.exit(main())
