"""Time FlatIndex.search (tpq_flat_search) against the torch brute force of bench.exact_truth on one H100.

For n in {1 M, 10 M} x d = 128 (euclidean), nq in {1, 100, 10 000} and k in {1, 10, 100, 1024}: CUDA-event time of
`--steps` search calls after `--warmup` warm-ups, alternating ours and torch's call by call; QPS, achieved FP32 FLOP/s
(2 d n nq over the call's time) against the 67 TFLOP/s data-sheet figure and the base read (4 d n bytes) against
3.35 TB/s, naming the larger of the two lower bounds; and, at the timed size, agreement: identical id sets on rows
without a tie at rank k, values within 1e-5 relative.  One JSON line per shape on stdout (and in --out).

    python scripts/bench_flat.py [--ns 1000000,10000000] [--nqs 1,100,10000] [--ks 1,10,100,1024] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK_FP32 = 67e12          # H100 SXM data sheet, dense FP32
PEAK_HBM = 3.35e12         # H100 SXM data sheet, HBM3


def card():
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else "unknown"


def torch_brute(base, x, k, chunk):
    """bench.exact_truth's loop (fp32 GEMM + topk per chunk, running merge), returning values as well as ids."""
    best_v = torch.full((x.shape[1], k), -float("inf"), device=x.device)
    best_i = torch.zeros((x.shape[1], k), dtype=torch.long, device=x.device)
    x2 = (x ** 2).sum(0)[:, None]
    for s in range(0, base.shape[1], chunk):
        b = base[:, s:s + chunk]
        sim = 2 * (x.T @ b) - x2 - (b ** 2).sum(0)[None, :]
        v, i = torch.topk(sim, min(k, sim.shape[1]), dim=1)
        cat_v = torch.cat([best_v, v], 1)
        cat_i = torch.cat([best_i, i + s], 1)
        sel = torch.topk(cat_v, k, dim=1).indices
        best_v, best_i = torch.gather(cat_v, 1, sel), torch.gather(cat_i, 1, sel)
    return best_v, best_i


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ns", default="1000000,10000000")
    ap.add_argument("--nqs", default="1,100,10000")
    ap.add_argument("--ks", default="1,10,100,1024")
    ap.add_argument("--d", type=int, default=128)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_flat needs a CUDA device"
    import torchpq_b200 as T
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    gpu = card()
    print(f"# card: {gpu}", flush=True)
    out = open(a.out, "w") if a.out else None
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(0)
    d = a.d
    for n in (int(s) for s in a.ns.split(",")):
        ix = T.FlatIndex(d, initial_size=n, device="cuda:0")
        ix.add(torch.randn(d, n, generator=g, device=dev))
        base = ix._storage.view(d, -1)[:, :n]
        for nq in (int(s) for s in a.nqs.split(",")):
            x = torch.randn(d, nq, generator=g, device=dev)
            chunk = max(4096, min(1 << 20, (1 << 29) // max(1, nq)))          # sim chunk <= 2 GB
            for k in (int(s) for s in a.ks.split(",")):
                ours = lambda: ix.search(x, k=k)
                ref = lambda: torch_brute(base, x, k, chunk)
                for _ in range(a.warmup):
                    ours(); ref()
                ev = [[torch.cuda.Event(enable_timing=True) for _ in range(4)] for _ in range(a.steps)]
                for e in ev:                                                  # alternate ours and torch's, call by call
                    e[0].record(); ours(); e[1].record()
                    e[2].record(); ref(); e[3].record()
                torch.cuda.synchronize()
                t_ours = sum(e[0].elapsed_time(e[1]) for e in ev) / a.steps / 1e3
                t_ref = sum(e[2].elapsed_time(e[3]) for e in ev) / a.steps / 1e3
                # agreement at the timed size: rows whose rank-k value is not tied with rank k+1
                v, i = ix.search(x, k=k)
                tv, ti = torch_brute(base, x, min(k + 1, n), chunk)
                rel = ((v - tv[:, :k]).abs() / tv[:, :k].abs().clamp_min(1e-30)).max().item()
                free = (tv[:, k - 1] - tv[:, k]).abs() > 4e-5 * tv[:, k - 1].abs() if k < n else torch.ones_like(tv[:, 0], dtype=torch.bool)
                same = (i.sort(1).values == ti[:, :k].sort(1).values).all(1)
                flops, byts = 2.0 * d * n * nq, 4.0 * d * n
                bound = "compute" if flops / PEAK_FP32 > byts / PEAK_HBM else "memory"
                r = dict(n=n, d=d, nq=nq, k=k, search_ms=round(t_ours * 1e3, 4), torch_ms=round(t_ref * 1e3, 4),
                         speedup=round(t_ref / t_ours, 3), qps=round(nq / t_ours, 1),
                         tflops=round(flops / t_ours / 1e12, 2), frac_fp32_peak=round(flops / t_ours / PEAK_FP32, 3),
                         tbps=round(byts / t_ours / 1e12, 3), frac_hbm_peak=round(byts / t_ours / PEAK_HBM, 3),
                         bound=bound, max_rel_value_diff=rel, tie_free_rows=int(free.sum().item()),
                         id_sets_equal_on_tie_free=bool(same[free].all().item()), gpu=gpu)
                line = json.dumps(r)
                print(line, flush=True)
                if out:
                    out.write(line + "\n")
                    out.flush()
        del ix, base
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
