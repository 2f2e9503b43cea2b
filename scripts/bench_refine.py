"""RefineFlatIndex over IVFPQIndex against the plain IVFPQIndex and IVFFlatIndex on a clustered C3-shaped set, one H100:
recall, QPS and the time of each pass.

Set: 10 M x 128 fp32, Gaussian-mixture (bench.py's clustered C3 generator), 4096 cells, n_probe 32 (no smart probing),
euclidean; 10 000 queries, k = 100.  The IVFPQIndex (M = 64) trains on the first 2^20 vectors with seed 0; the
RefineFlatIndex wraps that same IVFPQIndex, so its first pass is exactly the plain index's search.  The IVFFlatIndex
shares the IVFPQIndex's coarse codebook, so it probes the same cells.
Ground truth: bench.exact_truth's nearest neighbour of the first --n-truth queries.  exact_truth ranks with
2ab - a^2 - b^2, the refine pass with -sum(dif^2), so near-ties can differ by one rank.

Reported, one JSON line per configuration (IVFPQIndex, RefineFlatIndex at k_factor 1, 2, 4, IVFFlatIndex):
  - recall@1/10/100: fraction of truth queries whose true nearest neighbour is in the first 1/10/100 results;
  - QPS and ms per 10 000-query search (CUDA events, --steps calls after --warmup);
  - first_pass_ms (the IVFPQIndex's search at depth k1) and refine_ms (RefineFlatIndex.refine on those ids alone, id
    map lookup included), each timed alone;
  - refine bytes: 4 d per live candidate plus 8 per candidate address, over refine_ms, against the 3.35 TB/s HBM3
    data-sheet figure.
The card's name, power limit and SM clock are read in the same run.

    python scripts/bench_refine.py [--n 10000000] [--nq 10000] [--steps 5] [--warmup 2] [--out FILE]
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
    assert torch.cuda.is_available(), "bench_refine.py measures on a CUDA device"
    import bench
    import torchpq_b200 as T
    from torchpq_b200.modules import k1_of

    dev = torch.device("cuda:0")
    d, C, M, n_probe, k = 128, 4096, 64, 32, 100
    info = {"card": card(), "n": args.n, "d": d, "n_cells": C, "M": M, "n_probe": n_probe, "k": k, "nq": args.nq}
    t0 = time.time()
    centres = bench.cluster_centres(d, C, dev)
    base = bench.gen_base(d, args.n, dev, centres=centres)
    x = bench.gen_queries(d, args.nq, 1, dev, centres=centres)[0].to(dev)
    plain = T.IVFPQIndex(d, M, C, device=str(dev))
    rf = T.RefineFlatIndex(plain)
    rf.train(base[:, :1 << 20], seed=0)
    rf.add(base)
    plain.n_probe, plain.use_smart_probing = n_probe, False
    flat_ivf = T.IVFFlatIndex(d, C, device=str(dev))
    flat_ivf.vq_codec.set_codebook(plain.vq_codec.codebook)
    flat_ivf.add(base)
    flat_ivf.n_probe, flat_ivf.use_smart_probing = n_probe, False
    info["build_s"] = round(time.time() - t0, 1)
    xt = x[:, :args.n_truth].contiguous()
    truth = bench.exact_truth(base, xt, 1, "euclidean")[:, 0]
    del base
    torch.cuda.empty_cache()
    print(json.dumps(info), flush=True)

    lines = []

    def report(name, search, extra=None):
        ms = cuda_ms(lambda: search(x), args.steps, args.warmup)
        ids = search(xt)[1]
        lines.append({"index": name, **(extra or {}), "ms": round(ms, 3), "qps": round(args.nq / ms * 1e3),
                      **{f"recall@{r}": round(recall_at(ids, truth, r), 4) for r in (1, 10, 100)}})

    report("IVFPQIndex", lambda q: plain.search(q, k=k))
    print(json.dumps(lines[-1]), flush=True)
    for kf in (1, 2, 4):
        rf.k_factor = kf
        k1 = k1_of(k, kf)
        report("RefineFlatIndex", lambda q: rf.search(q, k=k), {"k_factor": kf, "k1": k1})
        first_ms = cuda_ms(lambda: plain.search(x, k1), args.steps, args.warmup)
        cand = plain.search(x, k1)[1]
        ref_ms = cuda_ms(lambda: rf.refine(x, cand, k), args.steps, args.warmup)
        live = int((rf._addresses_of(cand) >= 0).sum().item())
        nbytes = live * 4 * d + cand.numel() * 8
        lines[-1].update({"first_pass_ms": round(first_ms, 3), "refine_ms": round(ref_ms, 3),
                          "refine_share": round(ref_ms / (first_ms + ref_ms), 4), "live_candidates": live,
                          "refine_GBps": round(nbytes / ref_ms / 1e6, 1),
                          "refine_share_of_3.35TBps": round(nbytes / ref_ms / 1e-3 / PEAK_HBM, 4)})
        print(json.dumps(lines[-1]), flush=True)
    report("IVFFlatIndex", lambda q: flat_ivf.search(q, k=k))
    print(json.dumps(lines[-1]), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            for line in [info] + lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
