"""Time torchpq_b200.topk (tpq_topk) against torch.topk on one H100.

Shapes: 10 000 x 4 096 (k = 32), 10 000 x 65 536 (k = 100), 100 x 10^6 (k = 1024), 1 x 10^8 (k = 1, 100, 1024), an
ascending 1 x 10^8 row (k = 1024: every element passes the filter), and 10 000 x 65 536 in fp16 (k = 100).  Per shape:
CUDA-event time of `--steps` calls after `--warmup` warm-ups, alternating ours and torch.topk's call by call on the
same tensor; the time of each of our kernels (select, then the second pass over the slices' sorted parts where the
plan has one) from a separate torch.profiler run; the read (m n elem bytes) over our time against 3.35 TB/s; and
agreement with torch.topk (equal values column by column, equal indices on rows without a tie among the top k + 1).
One JSON line per shape on stdout (and in --out), each with the card's name, power limit and maximum SM clock.

    python scripts/bench_topk.py [--steps 20] [--warmup 3] [--only NAME,...] [--out FILE]
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

PEAK_HBM = 3.35e12         # H100 SXM data sheet, HBM3

SHAPES = [  # name, m, n, k, dtype, kind
    ("probe_10000x4096_k32", 10000, 4096, 32, torch.float32, "randn"),
    ("10000x65536_k100", 10000, 65536, 100, torch.float32, "randn"),
    ("100x1e6_k1024", 100, 10 ** 6, 1024, torch.float32, "randn"),
    ("1x1e8_k1", 1, 10 ** 8, 1, torch.float32, "randn"),
    ("1x1e8_k100", 1, 10 ** 8, 100, torch.float32, "randn"),
    ("1x1e8_k1024", 1, 10 ** 8, 1024, torch.float32, "randn"),
    ("1x1e8_k1024_ascending", 1, 10 ** 8, 1024, torch.float32, "ascending"),
    ("10000x65536_k100_fp16", 10000, 65536, 100, torch.float16, "randn"),
]


def card():
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else "unknown"


def make(m, n, dtype, kind):
    g = torch.Generator(device="cuda").manual_seed(m + n)
    if kind == "ascending":
        return torch.arange(m * n, device="cuda", dtype=torch.float32).reshape(m, n).to(dtype)
    return torch.randn(m, n, device="cuda", generator=g).to(dtype)


def alternate(fns, steps):
    """CUDA-event time (ms per call) of each fn, called in turn `steps` times."""
    ev = [[(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
          for _ in fns]
    for s in range(steps):
        for f, e in zip(fns, ev):
            e[s][0].record()
            f()
            e[s][1].record()
    torch.cuda.synchronize()
    return [sorted(a.elapsed_time(b) for a, b in e)[steps // 2] for e in ev]      # median


def stage_times(fn, steps):
    """Mean device time (ms) per call of each of our kernels, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        if "topk_" in e.key and "kernel" in e.key:
            name = e.key.split("topk_")[1].split("_kernel")[0]
            t = getattr(e, "device_time_total", None)
            if t is None:
                t = e.cuda_time_total
            out[f"topk_{name}_kernel"] = round(t / 1000.0 / steps, 4)
    return out


def agreement(x, v, i, k):
    tv, ti = torch.topk(x, k, dim=1)
    t = torch.topk(x.float(), min(k + 1, x.shape[1]), dim=1).values
    rows = (t[:, 1:] != t[:, :-1]).all(1)
    return {"values_equal": bool(torch.equal(v, tv)), "tie_free_rows": int(rows.sum()),
            "indices_equal_on_tie_free_rows": bool(torch.equal(i[rows], ti[rows]))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--only", default=None)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_topk needs a CUDA device"
    import torchpq_b200 as T
    gpu = card()
    only = set(a.only.split(",")) if a.only else None
    lines = []
    for name, m, n, k, dtype, kind in SHAPES:
        if only and name not in only:
            continue
        x = make(m, n, dtype, kind)
        ours = lambda: T.topk(x, k=k)                   # noqa: E731
        ref = lambda: torch.topk(x, k, dim=1)           # noqa: E731
        for _ in range(a.warmup):
            ours()
            ref()
        torch.cuda.synchronize()
        t_ours, t_torch = alternate([ours, ref], a.steps)
        stages = stage_times(ours, max(3, a.steps // 4))
        v, i = ours()
        nbytes = m * n * x.element_size()
        rec = {"shape": name, "m": m, "n": n, "k": k, "dtype": str(dtype).split(".")[1], "rows": kind,
               "ours_ms": round(t_ours, 4), "torch_topk_ms": round(t_torch, 4),
               "speedup_vs_torch_topk": round(t_torch / t_ours, 2), "stages_ms": stages,
               "read_bytes": nbytes, "read_TBps": round(nbytes / (t_ours * 1e-3) / 1e12, 3),
               "read_share_of_3.35TBps": round(nbytes / (t_ours * 1e-3) / PEAK_HBM, 3),
               "agreement": agreement(x, v, i, k), "gpu": gpu, "steps": a.steps, "warmup": a.warmup}
        line = json.dumps(rec)
        print(line, flush=True)
        lines.append(line)
        del x, v, i
        torch.cuda.empty_cache()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
