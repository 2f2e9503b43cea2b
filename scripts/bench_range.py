"""range_search against search on the same index, one H100: time, results per query, bounds, and where the time goes.

Workloads (bench.py's generators, as scripts/bench_ivfflat.py):
  * "1M":  1 M x 128 fp32 randn in a FlatIndex (every query scores every vector);
  * "C3c": the clustered 10 M x 128 C3 set in an IVFFlatIndex, 4096 cells, n_probe 32, smart probing off;
  * "C3c-pq" / "C3c-res": the same set in an IVFPQIndex with M = 64 (search runs cell-major there), plain / residual.
nq = 10 000.  Thresholds: for r in {10, 100, 1000}, the median over the queries of search(k = r)'s r-th value, so a
query gets about r results.

Reported, one JSON line per (workload, r):
  - results per query, mean and max;
  - range_ms / search_ms: CUDA-event time of range_search and of search(k = min(r, 1024)), alternated call by call
    (medians of --steps);
  - flop = 2 d * (vectors scored) and bytes = 4 d * (store vectors read) + 16 B per match (written, then sorted), the
    FP32 compute bound at 67 TFLOP/s and the memory bound at 3.35 TB/s (H100 SXM data sheet), and the share of the
    larger one that range_search reached.  IVFPQ: bytes = M * (vectors scanned, summed over the queries) + 12 B per
    match (the key and the query written by the kernel), against the memory bound;
  - rerun_ms: the same range_search with the first match buffer lowered to 256 entries per query, which forces the one
    re-run (the total is then known exactly and the second pass writes every match).
--profile: one torch.profiler run per workload at r = 100, kernel time split into the match kernel, the ordering (the
sorts and the CSR assembly) and the copy of the count; IVFPQ adds the range kernel's own CUDA-event time
(tpq_profile_scan_ms) and its share of the memory bound.  The card's name, power limit and max SM clock are read in the
same run.

    python scripts/bench_range.py [--workloads 1M,C3c,C3c-pq,C3c-res] [--steps 5] [--warmup 2] [--profile] [--out FILE]
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


def profile_split(fn):
    """Kernel ms of one call of fn under torch.profiler: the match kernel, the ordering, the count's copy, the rest."""
    from torch.profiler import profile, ProfilerActivity
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    split = {"match_kernel": 0.0, "ordering": 0.0, "count_copy": 0.0, "other": 0.0}
    names = {}
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        ms = e.device_time_total / 1e3
        n = e.name
        if "range_kernel" in n:
            key = "match_kernel"
        elif "Memcpy DtoH" in n or "Memcpy Device -> Host" in n or "DtoH" in n:
            key = "count_copy"
        elif "probe" in n or "pairs" in n or "plan_kernel" in n or "gather_kernel" in n or "norm" in n or "coarse" in n or "Memset" in n \
                or "Memcpy DtoD" in n or "Memcpy Device -> Device" in n or "col_" in n:
            key = "other"
        else:
            key = "ordering"                     # the torch sorts, searchsorted, the key decode and the id gather
        split[key] += ms
        short = n.split("<")[0].split("(")[0][:60]
        names[short] = names.get(short, 0.0) + ms
    return {k: round(v, 3) for k, v in split.items()}, \
        {k: round(v, 3) for k, v in sorted(names.items(), key=lambda kv: -kv[1])[:12]}


def scan_event_ms(fn, steps):
    """Median over `steps` calls of fn of the summed CUDA-event time of its scan-kernel launches (tpq_profile_*)."""
    import ctypes as C
    import torchpq_b200 as T
    L = T._lib.lib
    out = []
    for _ in range(steps):
        L.tpq_profile_enable(1)
        fn()
        ms, n = C.c_float(), C.c_int()
        T._lib.check(L.tpq_profile_scan_ms(C.byref(ms), C.byref(n)))
        L.tpq_profile_enable(0)
        out.append(ms.value)
    return sorted(out)[len(out) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="1M,C3c")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_range.py measures on a CUDA device"
    import torchpq_b200 as T
    from torchpq_b200 import _range

    dev = torch.device("cuda:0")
    lines = [{"card": card()}]
    print(json.dumps(lines[-1]), flush=True)
    for wname in args.workloads.split(","):
        t0 = time.time()
        pq = wname in ("C3c-pq", "C3c-res")
        d, n, C, base, x = workload("C3c" if pq else wname, dev)
        M = 64
        if pq:
            ix = T.IVFPQIndex(d, M, C, device=str(dev), pq_use_residual=wname == "C3c-res")
            ix.train(base[:, :1 << 20], seed=0)
            ix.add(base)
            ix.n_probe, ix.use_smart_probing = 32, False
            scored, store = scanned(ix, x, 32, False)
        elif wname == "1M":
            ix = T.FlatIndex(d, initial_size=n, device=str(dev))
            ix.add(base)
            scored, store = n * x.shape[1], n
        else:
            ix = T.IVFFlatIndex(d, C, device=str(dev))
            ix.train(base[:, :1 << 20], seed=0)
            ix.add(base)
            ix.n_probe, ix.use_smart_probing = 32, False
            scored, store = scanned(ix, x, 32, False)
        nq = x.shape[1]
        lines.append({"workload": wname, "index": type(ix).__name__, "n": n, "d": d, "nq": nq,
                      "build_s": round(time.time() - t0, 1)})
        print(json.dumps(lines[-1]), flush=True)
        for r in (10, 100, 1000):
            k = min(r, 1024)
            v, _ = ix.search(x, k=k)
            t = float(v[:, r - 1].median())
            lims, _, _ = ix.range_search(x, t)
            per_q = (lims[1:] - lims[:-1]).float()
            nnz = int(lims[-1])
            ms_range, ms_search = alternated_ms([lambda: ix.range_search(x, t), lambda: ix.search(x, k=k)],
                                                args.steps, args.warmup)
            if pq:                                   # ADC lookups: no FP32 GEMM; every scanned code is read once
                flop, byt = 0, M * scored + 12 * nnz
            else:
                flop, byt = 2 * d * scored, 4 * d * store + 16 * nnz
            bound_ms = max(flop / PEAK_FP32, byt / PEAK_HBM) * 1e3
            first = _range._FIRST_CAP_PER_QUERY
            _range._FIRST_CAP_PER_QUERY = 256
            forced = _range.first_cap(nq, 1 << 62) < nnz
            ms_rerun = alternated_ms([lambda: ix.range_search(x, t, max_results=1 << 62)], args.steps, args.warmup)[0]
            _range._FIRST_CAP_PER_QUERY = first
            line = {"workload": wname, "r": r, "threshold": t, "results_mean": round(float(per_q.mean()), 1),
                    "results_max": int(per_q.max()), "nnz": nnz, "range_ms": round(ms_range, 3),
                    f"search_k{k}_ms": round(ms_search, 3), "flop": flop, "bytes": byt,
                    "bound": "compute" if flop / PEAK_FP32 >= byt / PEAK_HBM else "memory",
                    "bound_ms": round(bound_ms, 4), "share_of_bound": round(bound_ms / ms_range, 4),
                    "achieved_tflops": round(flop / ms_range / 1e9, 2),
                    "rerun_ms": round(ms_rerun, 3), "rerun_forced": forced}
            lines.append(line)
            print(json.dumps(line), flush=True)
            if args.profile and r == 100:
                split, top = profile_split(lambda: ix.range_search(x, t))
                lines.append({"profile": f"{wname} r=100 range_search", "split_ms": split, "kernels_ms": top})
                if pq:
                    kern_ms = scan_event_ms(lambda: ix.range_search(x, t), args.steps)
                    lines[-1].update({"range_kernel_event_ms": round(kern_ms, 3),
                                      "range_kernel_share_of_hbm": round(M * scored / PEAK_HBM * 1e3 / kern_ms, 4)})
                print(json.dumps(lines[-1]), flush=True)
                split, top = profile_split(lambda: ix.search(x, k=100))
                lines.append({"profile": f"{wname} search k=100", "kernels_ms": top})
                print(json.dumps(lines[-1]), flush=True)
        del ix, base, x
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
