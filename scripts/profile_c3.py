#!/usr/bin/env python3
"""Per-kernel device times of a search step on a bench.py workload (default C3), with torch.profiler.

    python scripts/profile_c3.py --out DIR [--workload c3] [--steps 5] [--tag NAME]

Builds the workload's index as bench.py does, warms up, then
  * times `steps` strictly serial search steps with CUDA events (profiler off), and the scan stage inside them with the
    library's scan-launch events (bench.py's `roofline.scan_ms_per_launch`);
  * profiles `steps` more steps with CUDA activities and sums each kernel's device time per step.
Writes DIR/profile_<tag>.json: the card, the step and scan-stage times, the step time outside the scan stage, and every
kernel's ms per step, split into the scan stage's kernels and the rest.  TPQ_B200_LIB selects another build of the
library (e.g. a parent commit's) for an A/B on the same machine.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402

# kernels launched inside the scan stage's profiling events (tpq_profile_*): the query-major scan, or the cell-major
# path's LUTs, pair list, plan, pass 1, cell scan, select and re-run
SCAN_STAGE = ("ivfpq_scan_kernel", "ivfpq_cell_scan_kernel", "cell_lut_kernel", "cell_pairs_count_kernel",
              "cell_pairs_scatter_kernel", "cell_plan_kernel", "cell_select_kernel", "lut_kernel")


def short_name(name):
    """'void tpq::ivfpq_scan_kernel<64, 8, 2, 0, false>(tpq::ScanArgs, ...)' -> 'ivfpq_scan_kernel<64, 8, 2, 0, false>'"""
    n = name.split("(")[0]
    if n.startswith("void "):
        n = n[5:]
    return n.replace("tpq::", "")


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--out", required=True, help="output directory")
    ap.add_argument("--workload", default="c3", choices=list(bench.WORKLOADS))
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--nq", type=int, default=10000)
    ap.add_argument("--tag", default=None, help="file name suffix (default: the workload)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "profile_c3.py needs a CUDA device"
    from torch.profiler import ProfilerActivity, profile

    dev = torch.device("cuda:0")
    wl = bench.WORKLOADS[args.workload]
    N, d, M, C, n_probe, k, distance, n_train, desc = wl
    clustered = args.workload in bench.CLUSTERED
    centres = bench.cluster_centres(d, C, dev) if clustered else None
    index, base = bench.build_index(wl, dev, clustered=clustered)
    del base
    torch.cuda.empty_cache()
    index.layout()
    xs = [x.to(dev) for x in bench.gen_queries(d, args.nq, 4, dev, centres=centres)]

    def step(i):
        return index.search(xs[i % len(xs)], k=k)

    sampler = bench.ClockSampler(0)
    try:
        for i in range(args.warmup):
            step(i)
        bench.scan_profile_begin()
        step_ms = bench.cuda_time(step, args.steps, warmup=0, device=dev)
        scan_ms, launches = bench.scan_profile_end()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for i in range(args.steps):
                step(i)
            torch.cuda.synchronize(dev)
    finally:
        clocks = sampler.stop()

    per_kernel = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        if t <= 0:
            continue
        name = short_name(ev.key)
        per_kernel[name] = per_kernel.get(name, 0.0) + t / 1e3 / args.steps          # us -> ms per step
    in_scan = {n: v for n, v in per_kernel.items() if n.split("<")[0] in SCAN_STAGE}
    other = {n: v for n, v in per_kernel.items() if n not in in_scan}
    scan_per_step = scan_ms / args.steps if launches else None
    out = {
        "workload": f"{args.workload}: {desc}", "n_query_per_step": args.nq, "steps": args.steps,
        "card": {"gpu_name": clocks.get("gpu_name"), "power_limit_w": clocks.get("power_limit_w"),
                 "sm_mhz_median": clocks.get("sm_mhz"), "clock_reasons": clocks.get("reasons")},
        "step_ms": step_ms,
        "scan_stage_ms_per_step": scan_per_step,
        "outside_scan_stage_ms_per_step": step_ms - scan_per_step if scan_per_step is not None else None,
        "kernels_scan_stage_ms_per_step": dict(sorted(in_scan.items(), key=lambda kv: -kv[1])),
        "kernels_other_ms_per_step": dict(sorted(other.items(), key=lambda kv: -kv[1])),
        "kernel_sum_scan_stage_ms": sum(in_scan.values()), "kernel_sum_other_ms": sum(other.values()),
    }
    os.makedirs(args.out, exist_ok=True)
    path = os.path.join(args.out, f"profile_{args.tag or args.workload}.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps({"step_ms": out["step_ms"], "scan_stage_ms": scan_per_step,
                      "outside_scan_stage_ms": out["outside_scan_stage_ms_per_step"],
                      "top": list(out["kernels_scan_stage_ms_per_step"].items())[:3], "file": path}))


if __name__ == "__main__":
    main()
