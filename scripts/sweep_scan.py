"""Experiment driver (GPU box): time the scan kernel on one workload, optionally as one rank of a cell-sharded
index emulated on this GPU, with the per-phase cycle counters of the -DTPQ_DEBUG_KNOBS build.

usage: TPQ_B200_LIB=torchpq_b200/libtpq_b200_dbg.so python scripts/sweep_scan.py <workload> [shard_world ...]
       (knobs of the debug build: TPQ_SCAN_CFG=8x2|8x3|16x1|4x4, TPQ_BOOT_R=1|2, TPQ_BOOT_MODE=1 (merge tree, this build's
        default) | 0 (one-barrier quick start, the product library's bootstrap), TPQ_LUT_MODE=staged, TPQ_RES_MODE=staged2|staged3,
        TPQ_CELL_CFG=14x6|16x5 (shape of the cell-major kernel; scripts/cell_scan_account.py sweeps it with its cycle account))
Prints one JSON line per configuration and appends them to gpurun_out/sweep_scan.jsonl."""
import ctypes, json, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import bench
import torchpq_b200 as T

wl_name = sys.argv[1] if len(sys.argv) > 1 else "c3"
shards = [int(a) for a in sys.argv[2:]] or [1]
nq = int(os.environ.get("NQ", "10000"))
wl = bench.WORKLOADS[wl_name]
dev = torch.device("cuda:0")
index, base = bench.build_index(wl, dev, vq_iters=4, pq_iters=4)
del base
k = wl[5]
xs = [x.to(dev) for x in bench.gen_queries(wl[1], nq, 4, dev)]
lib = T._lib.lib
dbg = hasattr(lib, "tpq_debug_set_phase_buffer") or "dbg" in os.environ.get("TPQ_B200_LIB", "")
phase = torch.zeros(16, dtype=torch.int64, device=dev)     # [8..15]: the cell-major kernel's account (cell_scan_account.py)
if dbg:
    f = lib.tpq_debug_set_phase_buffer
    f.restype, f.argtypes = ctypes.c_int, [ctypes.c_void_p]
os.makedirs("gpurun_out", exist_ok=True)
for shard in shards:
    index.set_shard(0, shard)
    for smart in (True,):
        index.use_smart_probing = smart
        for i in range(3):
            index.search(xs[i], k=k)
        torch.cuda.synchronize()
        if dbg:
            phase.zero_(); f(ctypes.c_void_p(phase.data_ptr()))
        lib.tpq_profile_enable(1)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        reps = 8
        for i in range(reps):
            index.search(xs[i % 4], k=k)
        e1.record(); torch.cuda.synchronize()
        ms, n = ctypes.c_float(0), ctypes.c_int(0)
        lib.tpq_profile_scan_ms(ctypes.byref(ms), ctypes.byref(n))
        lib.tpq_profile_enable(0)
        rec = {"workload": wl_name, "nq": nq, "shard_world": shard, "scan_ms": ms.value / max(1, n.value),
               "search_ms": e0.elapsed_time(e1) / reps, "cfg": os.environ.get("TPQ_SCAN_CFG", "default"),
               "boot_r": os.environ.get("TPQ_BOOT_R", "2"), "lut_mode": os.environ.get("TPQ_LUT_MODE", "default")}
        if dbg:
            f(ctypes.c_void_p(0))
            p = phase.cpu().tolist()
            ctas = max(1, p[4])
            rec["phase_cycles_per_cta"] = {"prologue_lut": p[0] / ctas, "bootstrap": p[1] / ctas, "scan": p[2] / ctas,
                                           "drain": p[3] / ctas, "ctas": p[4]}
        print(json.dumps(rec), flush=True)
        with open("gpurun_out/sweep_scan.jsonl", "a") as fo:
            fo.write(json.dumps(rec) + "\n")
