"""Request coalescing (pb_search + pb_index_set_coalescing) under the deployment it is for: T host threads, each issuing
single-query searches in a loop on one handle.  Config B, generated on the device with bench.py's generator: 1M docs x
300 tokens x 128-d, 4-bit residuals, K = 2^18 (the batched variant), 32-token queries, centroid_score_threshold 0.4.
The threads draw from a shared pool of queries, with
  uniform   top_k 10, n_ivf_probe 8, n_full_scores 4096 for every request
  mixed     the 8 tuples of tools/bench_search_params.py: top_k in {10, 100}, n_ivf_probe in {8, 32}, n_full_scores
            in {1024, 4096}
each without subsets and with a subset per request (--subset-docs ids each), and the handle set to
  off       coalescing off: every call is a batch of one (what concurrent callers got before)
  on0       max_queries / max_inflight as given, max_wait_us 0
  on200     the same with max_wait_us 200
Every cell runs --seconds of wall clock per run, --runs runs, the three settings alternating inside a run.  Reported
per cell: queries/s (median, min, max over the runs), p50 / p99 request latency in ms over all runs, the batch-size
histogram, and how many requests failed or differed from the serial run of the same request (warm-up included; the
messages of failed requests are listed once each).  The threads call pb_search through ctypes with buffers prepared beforehand, so the interpreter adds little between calls; ctypes releases the GIL
during a call.  Prints one JSON line with the card and its power limit.

Run from the repository root on an H100: python tools/bench_coalesce.py"""
import argparse
import ctypes as C
import json
import os
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--threads", type=int, nargs="+", default=[1, 8, 32, 64])
    ap.add_argument("--pool", type=int, default=64)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--max-queries", type=int, default=32)
    ap.add_argument("--max-inflight", type=int, default=2)
    ap.add_argument("--subset-docs", type=int, default=10000)
    ap.add_argument("--docs-total", type=int, default=1000000)
    ap.add_argument("--log2k", type=int, default=18)
    a = ap.parse_args()
    sys.argv = [sys.argv[0], "--docs-total", str(a.docs_total), "--log2k", str(a.log2k), "--batch", str(a.pool)]
    import bench
    import torch
    import next_plaid_b200 as npb
    args = bench.parse_args()
    dev = torch.device("cuda", 0)
    G = bench.corpus_globals(args, dev)
    sh = bench.build_shard(args, G, 0, 1, dev)
    gpu = bench.open_shard(npb, args, G, sh, 0, 0)
    del sh["codes"]
    torch.cuda.empty_cache()
    L = npb.load_library()
    qs = [np.ascontiguousarray(q, np.float32) for q in bench.make_queries(args, G, dev, a.pool, seed=args.seed + 11)]
    rng = np.random.default_rng(6)
    uniform = [npb.SearchParameters(top_k=10, n_ivf_probe=8, n_full_scores=4096, centroid_score_threshold=args.threshold)
               for _ in qs]
    mixed = [npb.SearchParameters(top_k=int(rng.choice([10, 100])), n_ivf_probe=int(rng.choice([8, 32])),
                                  n_full_scores=int(rng.choice([1024, 4096])), centroid_score_threshold=args.threshold)
             for _ in qs]
    D = sh["D"]
    subsets = [np.sort(rng.choice(D, min(a.subset_docs, D), replace=False)).astype(np.int64) for _ in qs]
    P = lambda x: x.ctypes.data_as(C.c_void_p)  # noqa: E731

    def workload(params, with_subsets):
        """the pool as ready-made pb_search arguments, and the serial results they must reproduce"""
        items = []
        for j, (q, p) in enumerate(zip(qs, params)):
            s = subsets[j] if with_subsets else None
            items.append((P(q), q.shape[0], p._c(), None if s is None else P(s), 0 if s is None else len(s), p.top_k))
        ref = []
        ids, sc, cn = np.zeros(128, np.int64), np.zeros(128, np.float32), C.c_int32()
        for qp, nt, pc, sp, ns, _ in items:
            assert L.pb_search(gpu._h, qp, nt, C.byref(pc), sp, ns, P(ids), P(sc), C.byref(cn)) == 0
            ref.append((ids[:cn.value].tobytes(), sc[:cn.value].tobytes()))
        return items, ref

    def run_cell(T, items, ref, seconds):
        lat, n_done, n_failed, n_differ = [[] for _ in range(T)], [0] * T, [0] * T, [0] * T
        gate = threading.Barrier(T + 1)
        deadline = [0.0]

        def body(t):
            ids, sc, cn = np.zeros(128, np.int64), np.zeros(128, np.float32), C.c_int32()
            pi, ps, pc = P(ids), P(sc), C.byref(cn)
            gate.wait()
            i = t * 7
            while True:
                j = i % len(items)
                qp, nt, par, sp, ns, _ = items[j]
                t0 = time.perf_counter()
                if t0 >= deadline[0]:
                    break
                st = L.pb_search(gpu._h, qp, nt, C.byref(par), sp, ns, pi, ps, pc)
                lat[t].append(time.perf_counter() - t0)
                c = cn.value
                if st != 0:
                    n_failed[t] += 1
                    errors.setdefault(L.pb_last_error().decode("utf-8", "replace"), st)
                elif (ids[:c].tobytes(), sc[:c].tobytes()) != ref[j]:
                    n_differ[t] += 1
                n_done[t] += 1
                i += 1
        ths = [threading.Thread(target=body, args=(t,)) for t in range(T)]
        [t.start() for t in ths]
        deadline[0] = time.perf_counter() + seconds
        t0 = time.perf_counter()
        gate.wait()
        [t.join() for t in ths]
        wall = time.perf_counter() - t0
        return sum(n_done) / wall, [x for per in lat for x in per], sum(n_failed), sum(n_differ)

    errors = {}                                              # message -> status of every failed request
    modes = dict(off=(1, 0), on0=(a.max_queries, 0), on200=(a.max_queries, 200))
    cells = []
    for wname, params in (("uniform", uniform), ("mixed", mixed)):
        for with_subsets in (False, True):
            items, ref = workload(params, with_subsets)
            for T in a.threads:
                acc = {m: dict(qps=[], lat=[], failed=0, differ=0, hist=[0] * 8, batches=0, requests=0) for m in modes}
                for run in range(a.runs + 1):                 # run 0 warms up every setting of the cell
                    for m, (mq, wait) in modes.items():
                        gpu.set_coalescing(mq, max_wait_us=wait, max_inflight=a.max_inflight)
                        gpu.coalesce_stats(reset=True)
                        qps, lat, failed, differ = run_cell(T, items, ref, a.seconds if run else min(a.seconds, 0.3))
                        st = gpu.coalesce_stats()
                        acc[m]["failed"] += failed
                        acc[m]["differ"] += differ
                        if run:
                            acc[m]["qps"].append(qps)
                            acc[m]["lat"] += lat
                            acc[m]["hist"] = [x + y for x, y in zip(acc[m]["hist"], st["batch_hist"])]
                            acc[m]["batches"] += st["n_batches"]
                            acc[m]["requests"] += st["n_requests"]
                for m, v in acc.items():
                    lat = np.array(v["lat"]) * 1e3
                    cells.append(dict(
                        workload=wname, subsets=with_subsets, threads=T, mode=m,
                        qps=dict(median=round(float(np.median(v["qps"])), 1), min=round(min(v["qps"]), 1),
                                 max=round(max(v["qps"]), 1)),
                        p50_ms=round(float(np.percentile(lat, 50)), 3), p99_ms=round(float(np.percentile(lat, 99)), 3),
                        batch_hist=v["hist"],
                        mean_batch=round(v["requests"] / v["batches"], 2) if v["batches"] else None,
                        failed=v["failed"], differ=v["differ"], identical=v["failed"] + v["differ"] == 0))
    gpu.set_coalescing(1)
    gpu.close()
    info = bench.gpu_info(0)
    print(json.dumps(dict(workload="B", docs=D, K=G["K"], pool=a.pool, runs=a.runs, seconds=a.seconds,
                          max_queries=a.max_queries, max_inflight=a.max_inflight, subset_docs=a.subset_docs,
                          cells=cells, errors=errors, gpu=info["name"], power_limit_w=info["power_limit_w"])), flush=True)


if __name__ == "__main__":
    main()
