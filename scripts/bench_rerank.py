"""IVFPQRIndex against IVFPQIndex on a clustered C3-shaped set, one H100: recall, QPS and the time of each pass.

Set: 10 M x 128 fp32, Gaussian-mixture (bench.py's clustered C3 generator), 4096 cells, n_probe 32 (no smart probing),
M = 64, Mr = 64, use_residual, euclidean; codebooks trained on the first 2^20 vectors; 10 000 queries, k = 100.
Ground truth: FlatIndex's exact nearest neighbour of the first --n-truth queries.  The plain IVFPQIndex holds the same
first-level codebooks and the first M/4 word planes of the same store, so its search is the re-ranked index's first pass.

Reported, one JSON line per configuration (plain, then k_factor 1, 2, 4, 8):
  - recall@1/10/100: fraction of truth queries whose true nearest neighbour is in the first 1/10/100 results;
  - QPS and ms per 10 000-query search (CUDA events, --steps calls after --warmup);
  - first_pass_ms (IVFPQIndex.search at depth k1) and rerank_ms (IVFPQRIndex.rerank on those candidates alone),
    rerank_share = rerank_ms / (first_pass_ms + rerank_ms);
  - rerank sector bytes: one 32-byte sector per code word read, (M + Mr)/4 words per live candidate, plus the 8-byte
    candidate addresses; over rerank_ms, against the 3.35 TB/s HBM3 data-sheet figure.
The card's name, power limit and SM clock are read in the same run.

    python scripts/bench_rerank.py [--n 10000000] [--nq 10000] [--steps 5] [--warmup 2] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK_HBM = 3.35e12         # H100 SXM data sheet, HBM3


def card():
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else "unknown"


def cuda_ms(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / steps


def recall_at(ids, truth, r):
    return float((ids[:, :r] == truth[:, None]).any(1).float().mean())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--nq", type=int, default=10_000)
    ap.add_argument("--n-truth", type=int, default=1000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_rerank.py measures on a CUDA device"
    import bench
    import torchpq_b200 as T

    dev = torch.device("cuda:0")
    d, C, M, Mr, n_probe, k = 128, 4096, 64, 64, 32, 100
    info = {"card": card(), "n": args.n, "d": d, "n_cells": C, "M": M, "Mr": Mr, "n_probe": n_probe, "k": k,
            "nq": args.nq}
    t0 = time.time()
    centres = bench.cluster_centres(d, C, dev)
    base = bench.gen_base(d, args.n, dev, centres=centres)
    x = bench.gen_queries(d, args.nq, 1, dev, centres=centres)[0].to(dev)
    rx = T.IVFPQRIndex(d, M, Mr, C, use_residual=True, device=str(dev))
    rx.train(base[:, :1 << 20], seed=0)
    rx.add(base)
    rx.n_probe, rx.use_smart_probing = n_probe, False
    plain = T.IVFPQIndex(d, M, C, initial_size=1, device=str(dev))
    plain.load_state_dict({"_storage": rx._storage[:M // 4].contiguous(), "_is_empty": rx._is_empty.clone(),
                           "_cell_start": rx._cell_start.clone(), "_cell_size": rx._cell_size.clone(),
                           "_cell_capacity": rx._cell_capacity.clone(), "_address2id": rx._address2id.clone(),
                           "vq_codec.kmeans.centroids": rx.vq_codec.codebook, "vq_codec._is_trained": torch.tensor(True),
                           "pq_codec.kmeans.centroids": rx.pq_codec.codebook, "pq_codec._is_trained": torch.tensor(True)})
    plain.n_probe, plain.use_smart_probing = n_probe, False
    info["build_s"] = round(time.time() - t0, 1)

    flat = T.FlatIndex(d, device=str(dev))
    flat.add(base)
    xt = x[:, :args.n_truth].contiguous()
    truth = flat.search(xt, k=1)[1][:, 0]
    del flat
    torch.cuda.empty_cache()
    print(json.dumps(info), flush=True)

    lines = []
    ms = cuda_ms(lambda: plain.search(x, k=k), args.steps, args.warmup)
    ids = plain.search(xt, k=k)[1]
    lines.append({"index": "IVFPQIndex", "ms": round(ms, 3), "qps": round(args.nq / ms * 1e3),
                  **{f"recall@{r}": round(recall_at(ids, truth, r), 4) for r in (1, 10, 100)}})
    print(json.dumps(lines[-1]), flush=True)
    W = (M + Mr) // 4
    for kf in (1, 2, 4, 8):
        rx.k_factor = kf
        k1 = min(1024, max(k, kf * k))
        ms = cuda_ms(lambda: rx.search(x, k=k), args.steps, args.warmup)
        first_ms = cuda_ms(lambda: T.IVFPQIndex.search(rx, x, k1, return_address=True), args.steps, args.warmup)
        cand = T.IVFPQIndex.search(rx, x, k1, return_address=True)[2]
        rr_ms = cuda_ms(lambda: rx.rerank(x, cand, k), args.steps, args.warmup)
        live = int((cand >= 0).sum().item())
        sector_bytes = live * W * 32 + cand.numel() * 8
        ids = rx.search(xt, k=k)[1]
        lines.append({"index": "IVFPQRIndex", "k_factor": kf, "k1": k1, "ms": round(ms, 3), "qps": round(args.nq / ms * 1e3),
                      **{f"recall@{r}": round(recall_at(ids, truth, r), 4) for r in (1, 10, 100)},
                      "first_pass_ms": round(first_ms, 3), "rerank_ms": round(rr_ms, 3),
                      "rerank_share": round(rr_ms / (first_ms + rr_ms), 4), "live_candidates": live,
                      "rerank_sector_GBps": round(sector_bytes / rr_ms / 1e6, 1),
                      "rerank_sector_share_of_3.35TBps": round(sector_bytes / rr_ms / 1e-3 / PEAK_HBM, 4)})
        print(json.dumps(lines[-1]), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            for line in [info] + lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
