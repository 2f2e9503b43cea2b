"""Secondary measurements on one H100 (results -> aux_bench.json, see the end of the file):
C5 MultiKMeans assignment (GB/s vs HBM roofline), compute_centroids, pq_decode, search QPS on C2 / C4, and (`kmeans`)
the KMeans assignment for large k and d (TFLOP/s vs the TF32 data-sheet rate), its centroid update and a full fit.
CUDA events, 3 warm-ups, inputs larger than L2 where the workload allows."""
import json, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torchpq_b200 as T
import bench

dev = torch.device("cuda:0")
out = {}
peak = json.load(open(os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json")))["hbm_gbs"] \
    if os.path.exists(os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json")) else 3350.0


def timeit(fn, reps=5, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def card():
    """GPU name and enforced power limit, recorded beside the numbers they qualify."""
    import subprocess
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
        return {"gpu_name": q[0], "power_limit_w": float(q[1])}
    except Exception as e:                                             # the numbers stay, marked as unqualified
        return {"gpu_name": torch.cuda.get_device_name(0), "power_limit_w": None, "note": repr(e)}


which = sys.argv[1:] or ["c5", "centroids", "decode", "c2", "c4"]
if "kmeans" in which:
    # KMeans at the C3 coarse-quantizer shape and the reference benchmark's largest shape (benchmark/turing/kmeans):
    # assignment on the streaming TF32 wgmma kernel vs the exact fp32 kernel, the centroid update, and a full fit by
    # the reference benchmark's protocol (15 iterations, tol = 0, random init).
    TF32_PEAK = 495.0                                                  # H100 SXM dense TF32 data-sheet TFLOP/s
    res = {"card": card()}
    for l, d, n, k in ((1, 128, 1 << 20, 4096), (1, 256, 1 << 20, 16384)):
        torch.manual_seed(0)
        data = torch.randn(l, d, n, device=dev)
        cent = data[:, :, :k].contiguous()
        flop = 2.0 * l * n * d * k
        r = {"shape_l_d_n_k": [l, d, n, k], "gemm_form_tflop": flop / 1e12}
        for name, f in (("tf32_wide", lambda: T.fn.kmeans_assign(data, cent, exact_values=False)),
                        ("tf32_wide_exact_values", lambda: T.fn.kmeans_assign(data, cent, exact_values=True)),
                        ("exact_fp32", lambda: T.fn.max_sim(data, cent, exact=True))):
            ms = timeit(f, reps=3, warm=1)
            r[name] = {"ms": ms, "tflops_gemm_form": flop / ms / 1e9, "frac_of_tf32_peak": flop / ms / 1e9 / TF32_PEAK}
        se, le = T.fn.max_sim(data, cent, exact=True)
        st, lt = T.fn.kmeans_assign(data, cent, exact_values=True)
        diff = lt != le
        r["label_agreement_vs_exact"] = float((~diff).float().mean())
        r["max_rel_sim_gap_where_labels_differ"] = float(((se - st) / se.abs())[diff].max()) if diff.any() else 0.0
        r["maxsims_bit_identical_where_labels_agree"] = bool(torch.equal(st[~diff], se[~diff]))
        ms = timeit(lambda: T.fn.compute_centroids(data, le, k), reps=3, warm=1)
        r["compute_centroids_ms"] = ms
        x = data[0]
        km = T.KMeans(k, max_iter=15, tol=0.0, init_mode="random")
        km.fit(x)                                                      # warm-up
        torch.cuda.synchronize(); t0 = time.perf_counter()
        km.fit(x)
        torch.cuda.synchronize()
        r["kmeans_fit_15_iter_s"] = time.perf_counter() - t0
        r["kmeans_fit_iterations"] = km.n_iter_
        out[f"kmeans_d{d}_k{k}"] = r
        print(r, flush=True)
        del data, cent, se, le, st, lt, x
    out["kmeans_card"] = res["card"]
if "c5" in which or "centroids" in which:
    l, d, n, k = 64, 64, 1_000_000, 256
    data = torch.randn(l, d, n, device=dev)
    cent = data[:, :, :k].contiguous()
    if "c5" in which:
        byts = 4 * l * d * n + 4 * l * d * k + 12 * l * n
        for exact, ev, name, kern in ((False, False, "c5_max_sim_tc", "assign_tc_kernel (wgmma TF32, TF32-derived maxsim)"),
                                      (False, True, "c5_max_sim_tc_exact_values", "assign_tc_kernel (wgmma TF32 + exact fp32 maxsim)"),
                                      (True, True, "c5_max_sim_exact", "max_sim_kernel (fp32 SIMT, exact)")):
            if exact and "c5fast" in which:
                continue
            ms = timeit(lambda: T.fn.max_sim(data, cent, exact=exact, exact_values=ev), reps=3, warm=1)
            out[name] = {"ms": ms, "algorithmic_GB": byts / 1e9, "GBps": byts / ms / 1e6, "frac_of_hbm_peak": byts / ms / 1e6 / peak,
                         "tflops_gemm_form": 2.0 * l * n * d * k / ms / 1e9, "kernel": kern}
            print(out[name], flush=True)
        st, lt = T.fn.max_sim(data[:2], cent[:2], exact=False)          # exact fp32 similarity of the chosen centroid
        se, le = T.fn.max_sim(data[:2], cent[:2], exact=True)
        out["c5_label_agreement_tc_vs_exact"] = float((lt == le).float().mean())
        diff = lt != le                                                  # where labels differ: how much worse the choice is
        out["c5_max_rel_sim_gap_where_labels_differ"] = float(((se - st) / se.abs())[diff].max()) if diff.any() else 0.0
        print({k: out[k] for k in ("c5_label_agreement_tc_vs_exact", "c5_max_rel_sim_gap_where_labels_differ")}, flush=True)
    if "centroids" in which:
        lab = T.fn.max_sim(data, cent)[1]
        ms = timeit(lambda: T.fn.compute_centroids(data, lab, k), reps=3, warm=1)
        byts = 4 * l * d * n + 8 * l * n + 4 * l * d * k
        out["c5_compute_centroids"] = {"ms": ms, "algorithmic_GB": byts / 1e9, "GBps": byts / ms / 1e6, "frac_of_hbm_peak": byts / ms / 1e6 / peak}
        print(out["c5_compute_centroids"], flush=True)
    del data
if "decode" in which:
    M, dsub, n = 64, 2, 10_000_000
    cb = torch.randn(M, dsub, 256, device=dev)
    code = torch.randint(0, 256, (M, n), dtype=torch.uint8, device=dev)
    ms = timeit(lambda: T.fn.pq_decode(cb, code))
    byts = M * n + 4 * M * dsub * n
    out["pq_decode_10M"] = {"ms": ms, "algorithmic_GB": byts / 1e9, "GBps": byts / ms / 1e6, "frac_of_hbm_peak": byts / ms / 1e6 / peak}
    print(out["pq_decode_10M"], flush=True)
    del code
for name in ("c2", "c4"):
    if name not in which:
        continue
    wl = bench.WORKLOADS[name]
    index, base = bench.build_index(wl, dev)
    nq = 10000 if name == "c2" else 1000
    xs = [x.to(dev) for x in bench.gen_queries(wl[1], nq, 4, dev)]
    k = wl[5]
    T._lib.lib.tpq_profile_enable(0)
    i = [0]
    def step():
        index.search(xs[i[0] % 4], k=k); i[0] += 1
    ms = timeit(step, reps=10)
    truth = bench.exact_truth(base, xs[0][:, :500].contiguous(), k, wl[6])
    rec = bench.recall(index.search(xs[0][:, :500].contiguous(), k=k)[1], truth)
    out[f"{name}_search"] = {"nq": nq, "ms_per_batch": ms, "qps": nq / ms * 1e3, "recall_at_100": rec, "workload": wl[8]}
    print(out[f"{name}_search"], flush=True)
    del index, base
if "c3sweep" in which or "build" in which:
    wl = bench.WORKLOADS["c3"]
    torch.cuda.synchronize(); t0 = time.perf_counter()
    index, base = bench.build_index(wl, dev)
    torch.cuda.synchronize(); t_build = time.perf_counter() - t0
    out["c3_build"] = {"seconds_total": t_build, "what": "gen 10M x 128 randn + train (4+4 Lloyd iters on 1M) + encode 10M + container_add",
                       "reference_T4_sift1m": "train 4.45 s + add 10.72 s for 1M (BASELINE.md)"}
    # add path alone: encode + place 1M fresh vectors into an empty index with the trained codebooks
    from torchpq_b200 import build
    ix2 = T.IVFPQIndex(wl[1], wl[2], wl[3], initial_size=4096, device="cuda:0")
    ix2.vq_codec.set_codebook(index.vq_codec.codebook); ix2.pq_codec.set_codebook(index.pq_codec.codebook)
    xb = base[:, :1_000_000].contiguous()
    torch.cuda.synchronize(); t0 = time.perf_counter()
    ix2.add(xb)
    torch.cuda.synchronize(); out["add_1M"] = {"seconds": time.perf_counter() - t0, "vectors_per_s": 1e6 / (time.perf_counter() - t0)}
    print(out["c3_build"], out["add_1M"], flush=True)
    del ix2, xb
    if "c3sweep" in which:
        k = wl[5]
        res = {}
        for nq in (1, 10, 100, 1000, 10000):
            xs = [x.to(dev) for x in bench.gen_queries(wl[1], nq, 4, dev)]
            i = [0]
            def step():
                index.search(xs[i[0] % 4], k=k); i[0] += 1
            ms = timeit(step, reps=20)
            res[nq] = {"ms_per_batch": ms, "qps": nq / ms * 1e3}
        out["c3_batch_size_sweep"] = res
        print(res, flush=True)
    del index, base
if "c3res" in which:
    # residual IVFPQ on the C3 shape (reference: 72k q/s vs 120k q/s plain on T4/Sift1M, BASELINE.md)
    wl = bench.WORKLOADS["c3"]
    N, d, M, Cn, n_probe, k = wl[0], wl[1], wl[2], wl[3], wl[4], wl[5]
    from torchpq_b200 import build
    base = bench.gen_base(d, N, dev)
    tmp = T.IVFPQIndex(d, M, Cn, initial_size=1, device="cuda:0", pq_use_residual=True)
    build.train(tmp, base[:, :wl[7]].contiguous(), seed=0, vq_iters=4, pq_iters=4)
    cl, co = [], []
    for s0 in range(0, N, 1 << 20):
        c, q = build.encode(tmp, base[:, s0:s0 + (1 << 20)].contiguous()); cl.append(c); co.append(q)
    cells, codes = torch.cat(cl), torch.cat(co, 1)
    index = T.IVFPQIndex(d, M, Cn, initial_size=int(torch.bincount(cells, minlength=Cn).max().item()), device="cuda:0", pq_use_residual=True)
    index.vq_codec.set_codebook(tmp.vq_codec.codebook); index.pq_codec.set_codebook(tmp.pq_codec.codebook)
    build.container_add(index, codes, cells)
    index.n_probe = n_probe
    xs = [x.to(dev) for x in bench.gen_queries(d, 10000, 4, dev)]
    i = [0]
    def step():
        index.search(xs[i[0] % 4], k=k); i[0] += 1
    ms = timeit(step, reps=10)
    truth = bench.exact_truth(base, xs[0][:, :500].contiguous(), k, "euclidean")
    rec = bench.recall(index.search(xs[0][:, :500].contiguous(), k=k)[1], truth)
    out["c3_residual_search"] = {"nq": 10000, "ms_per_batch": ms, "qps": 1e4 / ms * 1e3, "recall_at_100": rec}
    print(out["c3_residual_search"], flush=True)
    del index, base, tmp
os.makedirs("gpurun_out", exist_ok=True)
json.dump(out, open("gpurun_out/aux_bench.json", "w"), indent=1)
