"""IVFPQ4Index (4-bit PQ codes) beside IVFPQIndex (8-bit) at equal code bytes on the clustered C3c set, one H100:
time, QPS, recall and the scan's code-byte bandwidth.

Set: 10 M x 128 fp32, Gaussian-mixture (bench.py's clustered C3 generator), 4096 cells, euclidean, no smart probing.
Every index shares one coarse codebook (trained with the IVFPQ M = 32 index on the first 2^20 vectors, seed 0), so
they probe the same cells; each trains its own PQ codebook on the same 2^20 vectors (25 Lloyd iterations, 256 or 16
codewords).  Configurations, code bytes per vector in brackets:
  IVFPQ  M = 32 (32 B)   IVFPQ4 M = 64 (32 B)   IVFPQ  M = 64 (64 B)   IVFPQ4 M = 128 (64 B)
  RefineFlatIndex(IVFPQ4 M = 64, k_factor = 1)   (the first pass's ids re-scored exactly on stored fp32 vectors)
Sweep: n_probe in {8, 32, 64} x nq in {1, 100, 10 000} x k in {10, 100}.  Each point times every configuration in
--rounds alternating rounds of --steps calls (CUDA events) and reports the median round.
Reported per point, one JSON line per configuration: ms per call, qps, and for the scan the code bytes it reads
(sum over queries of the live items of the probed cells x code bytes) over the call time.  Per (configuration,
n_probe): recall@1/10/100 = the fraction of the first --n-truth queries whose exact nearest neighbour (bench.exact_truth)
is among the first 1/10/100 results of a k = 100 search.  Then --profile: torch.profiler's kernel times of one
IVFPQ4 M = 64 and one IVFPQ M = 32 search (nq 10 000, n_probe 32, k 100).
The card's name, power limit and SM clock are read in the same run.

    python scripts/bench_ivfpq4.py [--n 10000000] [--rounds 5] [--steps 3] [--out FILE] [--profile]
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


def card():
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else "unknown"


def event_ms(fn, steps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / steps


def train_pq(ix, xt, n_codewords, seed=1):
    """ix's PQ codebook: n_codewords-means of the sub-vectors of xt (ix's coarse codebook is already set)."""
    from torchpq_b200 import build
    sub = xt.reshape(ix.n_subvectors, ix.d_subvector, xt.shape[1]).contiguous()
    ix.pq_codec.set_codebook(build.multi_kmeans(sub, n_codewords, 25, seed=seed).contiguous())
    ix._state_changed()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--n-truth", type=int, default=1000)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_ivfpq4.py measures on a CUDA device"
    import bench
    import torchpq_b200 as T

    dev = torch.device("cuda:0")
    d, C = 128, 4096
    info = {"card": card(), "n": args.n, "d": d, "n_cells": C}
    t0 = time.time()
    centres = bench.cluster_centres(d, C, dev)
    base = bench.gen_base(d, args.n, dev, centres=centres)
    xall = bench.gen_queries(d, 10_000, 1, dev, centres=centres)[0].to(dev)
    xt_train = base[:, :1 << 20].contiguous()
    pq32 = T.IVFPQIndex(d, 32, C, device=str(dev))
    pq32.train(xt_train, seed=0)
    vq = pq32.vq_codec.codebook
    pq64 = T.IVFPQIndex(d, 64, C, device=str(dev))
    p4_64 = T.IVFPQ4Index(d, 64, C, device=str(dev))
    p4_128 = T.IVFPQ4Index(d, 128, C, device=str(dev))
    for ix, K in ((pq64, 256), (p4_64, 16), (p4_128, 16)):
        ix.vq_codec.set_codebook(vq.clone())
        train_pq(ix, xt_train, K)
    rf = T.RefineFlatIndex(p4_64, k_factor=1)
    pq32.add(base)
    pq64.add(base)
    rf.add(base)                                                         # fills p4_64 and the refine store
    p4_128.add(base)
    configs = {"IVFPQ M=32 (32 B)": pq32, "IVFPQ4 M=64 (32 B)": p4_64, "IVFPQ M=64 (64 B)": pq64,
               "IVFPQ4 M=128 (64 B)": p4_128, "Refine(IVFPQ4 M=64, k_factor=1)": rf}
    code_bytes = {"IVFPQ M=32 (32 B)": 32, "IVFPQ4 M=64 (32 B)": 32, "IVFPQ M=64 (64 B)": 64, "IVFPQ4 M=128 (64 B)": 64,
                  "Refine(IVFPQ4 M=64, k_factor=1)": 32}
    for ix in (pq32, pq64, p4_64, p4_128):
        ix.use_smart_probing = False
    info["build_s"] = round(time.time() - t0, 1)
    info["index_code_bytes"] = {name: args.n * b for name, b in code_bytes.items()}
    xt = xall[:, :args.n_truth].contiguous()
    truth = bench.exact_truth(base, xt, 1, "euclidean")[:, 0]
    del base, xt_train
    torch.cuda.empty_cache()
    print(json.dumps(info), flush=True)
    lines = [info]

    def set_probe(n_probe):
        for ix in (pq32, pq64, p4_64, p4_128):
            ix.n_probe = n_probe

    def emit(line):
        lines.append(line)
        print(json.dumps(line), flush=True)

    cell_size = pq32._cell_size
    for n_probe in (8, 32, 64):
        set_probe(n_probe)
        for name, ix in configs.items():
            ids = ix.search(xt, k=100)[1]
            rec = {f"recall@{r}": round(float((ids[:, :r] == truth[:, None]).any(1).float().mean()), 4) for r in (1, 10, 100)}
            emit({"config": name, "n_probe": n_probe, "recall_queries": args.n_truth, **rec})
        for nq in (1, 100, 10_000):
            x = xall[:, :nq].contiguous()
            cells = T.fn.coarse_probe(x, vq, n_probe, False)[1]
            scanned = int(cell_size[cells].sum().item())                  # live items of the probed cells (no holes here)
            for k in (10, 100):
                runs = {name: [] for name in configs}
                for ix in configs.values():                              # warm every shape (and build the caches)
                    ix.search(x, k=k)
                torch.cuda.synchronize()
                for _ in range(args.rounds):
                    for name, ix in configs.items():
                        runs[name].append(event_ms(lambda: ix.search(x, k=k), args.steps))
                for name in configs:
                    ms = statistics.median(runs[name])
                    emit({"config": name, "n_probe": n_probe, "nq": nq, "k": k, "ms": round(ms, 4),
                          "qps": round(nq / ms * 1e3, 1), "scanned_items": scanned,
                          "code_GBps": round(scanned * code_bytes[name] / ms / 1e6, 1),
                          "spread_ms": [round(min(runs[name]), 4), round(max(runs[name]), 4)]})
    if args.profile:
        from torch.profiler import profile, ProfilerActivity
        set_probe(32)
        x = xall.contiguous()
        for name in ("IVFPQ4 M=64 (32 B)", "IVFPQ M=32 (32 B)", "IVFPQ4 M=128 (64 B)"):
            ix = configs[name]
            ix.search(x, k=100)
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(3):
                    ix.search(x, k=100)
                torch.cuda.synchronize()
            kern = {}
            for e in prof.key_averages():
                t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
                if t:
                    kern[e.key[:60]] = round(t / 3 / 1e3, 3)
            emit({"profile": name, "n_probe": 32, "nq": 10_000, "k": 100, "kernel_ms_per_search": kern})
    if args.out:
        with open(args.out, "w") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
