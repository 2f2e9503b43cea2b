"""IVFFlatIndex against IVFPQIndex trained on the same data and seed, one H100: time, QPS, bounds, recall.

Workloads (bench.py's generators):
  * "1M":  1 M x 128 fp32 randn, 1024 cells;
  * "C3c": the clustered 10 M x 128 C3 set (Gaussian mixture), 4096 cells.
Both indexes train their coarse codebook on the first 2^20 vectors with seed 0 (IVFPQIndex: M = 64), so they probe the
same cells.  Sweep: n_probe in {8, 32, 64} x nq in {1, 100, 10000} x k in {10, 100} x smart probing off / on.

Reported, one JSON line per configuration:
  - ms / qps: CUDA-event time of one search, IVFFlatIndex and IVFPQIndex alternated call by call (medians of --steps);
  - flop = 2 d * (live vectors scanned, summed over the queries) and bytes = 4 d * (live vectors of the distinct probed
    cells), the compute bound at 67 TFLOP/s FP32 and the memory bound at 3.35 TB/s (H100 SXM data sheet), the larger
    one and the share of it the search reached (bound / ms);
  - recall@k of both indexes against bench.exact_truth (bench.recall) on the first --n-truth queries;
  - max_abs_err: largest |value - torch fp32 recomputation of the score of the returned vector| over those queries.
--profile: one torch.profiler run of the C3c, n_probe 32, nq 10000, k 100 search (smart probing off), kernel time by
kernel.  The card's name, power limit and max SM clock are read in the same run.

    python scripts/bench_ivfflat.py [--workloads 1M,C3c] [--steps 5] [--warmup 2] [--profile] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK_FP32 = 67e12          # H100 SXM data sheet, FP32 (non-tensor)
PEAK_HBM = 3.35e12         # H100 SXM data sheet, HBM3


def card():
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else "unknown"


def alternated_ms(fns, steps, warmup):
    """Median CUDA-event ms of each fn, the fns called in turn, one call each per step."""
    for _ in range(warmup):
        for f in fns:
            f()
    torch.cuda.synchronize()
    times = [[] for _ in fns]
    for _ in range(steps):
        for t, f in zip(times, fns):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            f()
            b.record()
            b.synchronize()
            t.append(a.elapsed_time(b))
    return [statistics.median(t) for t in times]


def scanned(ix, x, n_probe, smart):
    """(live vectors scanned summed over the queries, live vectors of the distinct probed cells)."""
    import torchpq_b200 as T
    xp = T.fn.normalize(x) if ix.distance == "cosine" else x
    _, cells, npl = T.fn.coarse_probe(xp.contiguous(), ix.vq_codec.codebook, n_probe, smart, ix.smart_probing_temperature)
    P = npl.clamp(1, n_probe)
    used = torch.arange(n_probe, device=x.device)[None, :] < P[:, None]
    live = ix._cell_size                                                  # no removals: live == cell_size
    total = int(live[cells][used].sum().item())
    distinct = int(live[torch.unique(cells[used])].sum().item())
    return total, distinct


def max_abs_err(base, x, values, ids):
    """Largest |value - torch fp32 score| of the returned vectors (ids = column of base)."""
    ok = ids >= 0
    b = base[:, ids.clamp(min=0)]                                          # [d, nq, k]
    dot = (x[:, :, None] * b).sum(0)
    ref = 2 * dot - (x * x).sum(0)[:, None] - (b * b).sum(0)
    return float((values - ref)[ok].abs().max().item())


def workload(name, dev):
    import bench
    if name == "1M":
        d, n, C = 128, 1_000_000, 1024
        centres = None
    else:
        d, n, C = 128, 10_000_000, 4096
        centres = bench.cluster_centres(d, C, dev)
    base = bench.gen_base(d, n, dev, centres=centres)
    x = bench.gen_queries(d, 10_000, 1, dev, centres=centres)[0].to(dev)
    return d, n, C, base, x


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="1M,C3c")
    ap.add_argument("--n-truth", type=int, default=1000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_ivfflat.py measures on a CUDA device"
    import bench
    import torchpq_b200 as T

    dev = torch.device("cuda:0")
    lines = [{"card": card()}]
    print(json.dumps(lines[-1]), flush=True)
    for wname in args.workloads.split(","):
        t0 = time.time()
        d, n, C, base, x = workload(wname, dev)
        fl = T.IVFFlatIndex(d, C, device=str(dev))
        fl.train(base[:, :1 << 20], seed=0)
        fl.add(base)
        pq = T.IVFPQIndex(d, 64, C, device=str(dev))
        pq.train(base[:, :1 << 20], seed=0)
        pq.add(base)
        assert torch.equal(fl.vq_codec.codebook, pq.vq_codec.codebook)
        xt = x[:, :args.n_truth].contiguous()
        truth = {k: bench.exact_truth(base, xt, k, "euclidean") for k in (10, 100)}
        lines.append({"workload": wname, "n": n, "d": d, "n_cells": C, "build_s": round(time.time() - t0, 1)})
        print(json.dumps(lines[-1]), flush=True)
        for smart in (False, True):
            for n_probe in (8, 32, 64):
                for ix in (fl, pq):
                    ix.n_probe, ix.use_smart_probing = n_probe, smart
                for nq in (1, 100, 10_000):
                    xq = x[:, :nq].contiguous()
                    total, distinct = scanned(fl, xq, n_probe, smart)
                    flop, byt = 2 * d * total, 4 * d * distinct
                    bound_ms = max(flop / PEAK_FP32, byt / PEAK_HBM) * 1e3
                    for k in (10, 100):
                        ms_fl, ms_pq = alternated_ms([lambda: fl.search(xq, k=k), lambda: pq.search(xq, k=k)],
                                                     args.steps, args.warmup)
                        line = {"workload": wname, "smart": smart, "n_probe": n_probe, "nq": nq, "k": k,
                                "ivfflat_ms": round(ms_fl, 3), "ivfflat_qps": round(nq / ms_fl * 1e3),
                                "ivfpq_ms": round(ms_pq, 3), "ivfpq_qps": round(nq / ms_pq * 1e3),
                                "flop": flop, "bytes": byt,
                                "bound": "compute" if flop / PEAK_FP32 >= byt / PEAK_HBM else "memory",
                                "bound_ms": round(bound_ms, 4), "share_of_bound": round(bound_ms / ms_fl, 4)}
                        if nq == 10_000:
                            vf, i_fl = fl.search(xt, k=k)
                            _, i_pq = pq.search(xt, k=k)
                            line.update({"recall_ivfflat": round(bench.recall(i_fl, truth[k]), 4),
                                         "recall_ivfpq": round(bench.recall(i_pq, truth[k]), 4),
                                         "max_abs_err": max_abs_err(base, xt[:, :100], vf[:100], i_fl[:100])})
                        lines.append(line)
                        print(json.dumps(line), flush=True)
        if args.profile and wname == "C3c":
            fl.n_probe, fl.use_smart_probing = 32, False
            fl.search(x, k=100)
            torch.cuda.synchronize()
            from torch.profiler import profile, ProfilerActivity
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                fl.search(x, k=100)
                torch.cuda.synchronize()
            by = {}
            for e in prof.events():
                if e.device_type == torch.autograd.DeviceType.CUDA:
                    key = e.name.split("<")[0].split("(")[0]
                    by[key] = by.get(key, 0.0) + e.device_time_total / 1e3
            lines.append({"profile": "C3c n_probe=32 nq=10000 k=100 smart=off",
                          "kernel_ms": {k: round(v, 3) for k, v in sorted(by.items(), key=lambda kv: -kv[1])},
                          "total_kernel_ms": round(sum(by.values()), 3)})
            print(json.dumps(lines[-1]), flush=True)
        del fl, pq, base, x
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
