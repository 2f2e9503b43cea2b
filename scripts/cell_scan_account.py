#!/usr/bin/env python3
"""Where ivfpq_cell_scan_kernel's time goes on a bench.py workload (default C3): per-phase warp-cycles, the two
ablations that bound a gain, and the kernel's shapes.  Needs the -DTPQ_DEBUG_KNOBS build:

    make -C torchpq_b200/csrc dbg
    TPQ_B200_LIB=torchpq_b200/libtpq_b200_dbg.so python scripts/cell_scan_account.py --out DIR [--workload c3]

Builds the workload's index as bench.py does, then for every configuration (the debug build reads the knobs once per
search, so they are switched inside one process):
  * profiles `steps` serial search steps with torch.profiler and takes the cell-scan kernel's device time per step;
  * runs one more step with the phase buffer set and reads the kernel's cycle account: each phase's share of all
    warps' cycles from kernel entry to exit.
Configurations: the product shape 12x7; TPQ_CELL_ABLATE=1 (no refills: every pair of an item reuses the first three
LUTs, which leaves the scoring time of this kernel shape), =2 (no survivors: neither the pair tail nor the window
flush runs), =3 (both);
TPQ_CELL_CFG=14x6 and 16x5.  The ablations give WRONG search results on purpose; only their times mean anything.
Writes DIR/cell_scan_account_<workload>.json and prints one line per configuration.
"""
import argparse
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402
import torchpq_b200 as T  # noqa: E402

PHASES = ("item_prologue", "mbar_wait", "scoring", "release_issue", "pair_tail", "window_flush")
CONFIGS = (("12x7", {}), ("12x7 no refills", {"TPQ_CELL_ABLATE": "1"}), ("12x7 no survivors", {"TPQ_CELL_ABLATE": "2"}),
           ("12x7 no refills, no survivors", {"TPQ_CELL_ABLATE": "3"}),
           ("14x6", {"TPQ_CELL_CFG": "14x6"}), ("16x5", {"TPQ_CELL_CFG": "16x5"}))
KNOBS = ("TPQ_CELL_ABLATE", "TPQ_CELL_CFG")


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--out", required=True, help="output directory")
    ap.add_argument("--workload", default="c3", choices=list(bench.WORKLOADS))
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--nq", type=int, default=10000)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "cell_scan_account.py needs a CUDA device"
    lib = T._lib.lib
    assert hasattr(lib, "tpq_debug_set_phase_buffer"), "set TPQ_B200_LIB to the -DTPQ_DEBUG_KNOBS build (make dbg)"
    set_phase = lib.tpq_debug_set_phase_buffer
    set_phase.restype, set_phase.argtypes = ctypes.c_int, [ctypes.c_void_p]
    from torch.profiler import ProfilerActivity, profile

    dev = torch.device("cuda:0")
    wl = bench.WORKLOADS[args.workload]
    d, k = wl[1], wl[5]
    clustered = args.workload in bench.CLUSTERED
    centres = bench.cluster_centres(d, wl[3], dev) if clustered else None
    index, base = bench.build_index(wl, dev, clustered=clustered)
    del base
    torch.cuda.empty_cache()
    index.layout()
    xs = [x.to(dev) for x in bench.gen_queries(d, args.nq, 4, dev, centres=centres)]
    phase = torch.zeros(16, dtype=torch.int64, device=dev)

    def step(i):
        return index.search(xs[i % len(xs)], k=k)

    rows = []
    sampler = bench.ClockSampler(0)
    try:
        for tag, env in CONFIGS:
            for name in KNOBS:
                os.environ.pop(name, None)
            os.environ.update(env)
            for i in range(2):
                step(i)
            torch.cuda.synchronize(dev)
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for i in range(args.steps):
                    step(i)
                torch.cuda.synchronize(dev)
            kern_ms = 0.0
            for ev in prof.key_averages():
                if "ivfpq_cell_scan_kernel" in ev.key:
                    kern_ms += ev.device_time_total / 1e3 / args.steps
            phase.zero_()
            set_phase(ctypes.c_void_p(phase.data_ptr()))
            step(0)
            torch.cuda.synchronize(dev)
            set_phase(ctypes.c_void_p(0))
            p = phase.cpu().tolist()[8:]
            total = max(1, p[7])
            row = {"config": tag, "cell_scan_kernel_ms": kern_ms, "warps": p[6], "cycles_per_warp": total / max(1, p[6]),
                   "phase_share": {n: p[j] / total for j, n in enumerate(PHASES)}}
            rows.append(row)
            print(json.dumps(row), flush=True)
    finally:
        for name in KNOBS:
            os.environ.pop(name, None)
        clocks = sampler.stop()
    out = {"workload": f"{args.workload}: {wl[8]}", "n_query_per_step": args.nq, "steps": args.steps,
           "card": {"gpu_name": clocks.get("gpu_name"), "power_limit_w": clocks.get("power_limit_w"),
                    "sm_mhz_median": clocks.get("sm_mhz"), "clock_reasons": clocks.get("reasons")},
           "configs": rows}
    os.makedirs(args.out, exist_ok=True)
    path = os.path.join(args.out, f"cell_scan_account_{args.workload}.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps({"card": out["card"], "file": path}))


if __name__ == "__main__":
    main()
