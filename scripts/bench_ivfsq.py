"""IVFSQIndex (8 and 16 bits) against IVFFlatIndex and IVFPQIndex (M = 64) on the same coarse codebook, one H100.

Workloads (bench.py's generators):
  * "1M":  1 M x 128 fp32 randn, 1024 cells;
  * "C3c": the clustered 10 M x 128 C3 set (Gaussian mixture), 4096 cells.
Every index trains its coarse codebook on the first 2^20 vectors with seed 0, so all four probe the same cells.
Sweep: n_probe in {8, 32, 64} x nq in {1, 100, 10000} x k in {10, 100}, smart probing off.

Reported, one JSON line per configuration:
  - ms / qps: CUDA-event time of one search, the four indexes alternated call by call (medians of --steps);
  - flop = 2 d * (live vectors scanned, summed over the queries); bytes per index = its code bytes per vector times the
    live vectors of the distinct probed cells (d for SQ8, 2 d for SQ16, 4 d for IVFFlat), with the compute bound at
    67 TFLOP/s FP32 and the memory bound at 3.35 TB/s (H100 SXM data sheet);
  - recall@k of every index against bench.exact_truth of the original vectors on the first --n-truth queries;
  - max_abs_err of each SQ index: largest |value - torch fp32 score recomputed on the decoded vector it returned|.
Per workload: each index's store bytes.  --profile: one torch.profiler run per index of the C3c, n_probe 32,
nq 10000, k 100 search, kernel time by kernel.  The card's name, power limit and max SM clock are read in the same run.

    python scripts/bench_ivfsq.py [--workloads 1M,C3c] [--steps 5] [--warmup 2] [--profile] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_ivfflat import PEAK_FP32, PEAK_HBM, alternated_ms, card, scanned, workload  # noqa: E402


def max_abs_err(ix, x, values, address):
    """Largest |value - torch fp32 euclidean score of the decoded vector at the returned address|."""
    ok = address >= 0
    nq, k = address.shape
    b = ix.get_data_by_address(address.clamp(min=0).flatten()).view(ix.d_vector, nq, k)
    dot = (x[:, :, None] * b).sum(0)
    ref = 2 * dot - (x * x).sum(0)[:, None] - (b * b).sum(0)
    return float((values - ref)[ok].abs().max().item())


def profile_ms(fn):
    from torch.profiler import profile, ProfilerActivity
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    by = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            key = e.name.split("(")[0]
            by[key] = by.get(key, 0.0) + e.device_time_total / 1e3
    return {k: round(v, 3) for k, v in sorted(by.items(), key=lambda kv: -kv[1])}, round(sum(by.values()), 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="1M,C3c")
    ap.add_argument("--n-truth", type=int, default=1000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_ivfsq.py measures on a CUDA device"
    import bench
    import torchpq_b200 as T

    dev = torch.device("cuda:0")
    lines = [{"card": card()}]
    print(json.dumps(lines[-1]), flush=True)
    for wname in args.workloads.split(","):
        t0 = time.time()
        d, n, C, base, x = workload(wname, dev)
        idx = {"ivfsq8": T.IVFSQIndex(d, C, bits=8, device=str(dev)),
               "ivfsq16": T.IVFSQIndex(d, C, bits=16, device=str(dev)),
               "ivfflat": T.IVFFlatIndex(d, C, device=str(dev)),
               "ivfpq": T.IVFPQIndex(d, 64, C, device=str(dev))}
        for ix in idx.values():
            ix.train(base[:, :1 << 20], seed=0)
            ix.add(base)
        cb = idx["ivfflat"].vq_codec.codebook
        assert all(torch.equal(ix.vq_codec.codebook, cb) for ix in idx.values())
        per_vec = {"ivfsq8": d, "ivfsq16": 2 * d, "ivfflat": 4 * d, "ivfpq": 64}
        xt = x[:, :args.n_truth].contiguous()
        truth = {k: bench.exact_truth(base, xt, k, "euclidean") for k in (10, 100)}
        lines.append({"workload": wname, "n": n, "d": d, "n_cells": C, "build_s": round(time.time() - t0, 1),
                      "store_bytes": {name: ix._storage.numel() * ix._storage.element_size() for name, ix in idx.items()}})
        print(json.dumps(lines[-1]), flush=True)
        for n_probe in (8, 32, 64):
            for ix in idx.values():
                ix.n_probe, ix.use_smart_probing = n_probe, False
            for nq in (1, 100, 10_000):
                xq = x[:, :nq].contiguous()
                total, distinct = scanned(idx["ivfflat"], xq, n_probe, False)
                flop = 2 * d * total
                for k in (10, 100):
                    names = list(idx)
                    ms = alternated_ms([(lambda ix=ix: ix.search(xq, k=k)) for ix in idx.values()], args.steps,
                                       args.warmup)
                    line = {"workload": wname, "n_probe": n_probe, "nq": nq, "k": k, "flop": flop,
                            "compute_bound_ms": round(flop / PEAK_FP32 * 1e3, 4)}
                    for name, t in zip(names, ms):
                        line[f"{name}_ms"] = round(t, 3)
                        line[f"{name}_qps"] = round(nq / t * 1e3)
                        line[f"{name}_memory_bound_ms"] = round(per_vec[name] * distinct / PEAK_HBM * 1e3, 4)
                    line["sq8_over_flat"] = round(ms[0] / ms[2], 3)
                    if nq == 10_000:
                        for name, ix in idx.items():
                            v, i, a = ix.search(xt, k=k, return_address=True)
                            line[f"recall_{name}"] = round(bench.recall(i, truth[k]), 4)
                            if name.startswith("ivfsq"):
                                line[f"max_abs_err_{name}"] = max_abs_err(ix, xt[:, :100], v[:100], a[:100])
                    lines.append(line)
                    print(json.dumps(line), flush=True)
        if args.profile and wname == "C3c":
            for name, ix in idx.items():
                ix.n_probe = 32
                kernel_ms, total_ms = profile_ms(lambda: ix.search(x, k=100))
                lines.append({"profile": f"{name} C3c n_probe=32 nq=10000 k=100 smart=off", "kernel_ms": kernel_ms,
                              "total_kernel_ms": total_ms})
                print(json.dumps(lines[-1]), flush=True)
        del idx, base, x
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
