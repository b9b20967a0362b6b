"""Per-query subsets (pb_search_batch_subsets) against the ways a server could serve the same filtered requests without
it.  Two workloads, generated on the device with bench.py's generator (32-token queries, top_k 100, n_full_scores 4096,
centroid_score_threshold 0.4, the default centroid_batch_size of 100 000):
  B      config B: 1M docs x 300 tokens x 128-d, 4-bit residuals, K = 2^18 (the batched variant: subsets intersect)
  dense  200k docs x 300 tokens, K = 2^16 (the dense variant: eligible centroids and the scaled n_ivf_probe)
32 queries, each with its own random subset of 10 % of the docs, are searched as
  subsets   one pb_search_batch_subsets call
  serial    32 batch-of-1 pb_search_batch calls, one after another
  threads   the same 32 calls from 8 host threads
  shared    one pb_search_batch with a single shared 10 % subset (the ceiling: one subset row for the batch)
Every form is checked to return identical ids and scores (shared: against pb_search_batch_subsets with that one subset
for every query).  Wall clock around the calls with host buffers; --runs runs of each form, alternating, after one
warm-up round; median, min and max queries/s.  Prints one JSON line per workload with the card and its power limit.

Run from the repository root on an H100: python tools/bench_subsets.py [--workloads B,dense]"""
import argparse
import json
import os
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

WORKLOADS = {"B": dict(docs_total=1_000_000, log2k=18), "dense": dict(docs_total=200_000, log2k=16)}


def run_workload(name, a):
    w = WORKLOADS[name]
    sys.argv = [sys.argv[0], "--docs-total", str(w["docs_total"]), "--log2k", str(w["log2k"]), "--batch", "32"]
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
    D = sh["D"]
    p = npb.SearchParameters(top_k=args.top_k, n_ivf_probe=args.n_ivf_probe, n_full_scores=args.n_full_scores,
                             centroid_score_threshold=args.threshold)
    qs = bench.make_queries(args, G, dev, a.queries, seed=args.seed + 7)
    rng = np.random.default_rng(5)
    subs = [np.sort(rng.choice(D, D // 10, replace=False)).astype(np.int64) for _ in qs]
    shared = subs[0]

    def key(res):
        return [(r.passage_ids.tolist(), r.scores.tobytes()) for r in res]

    def f_subsets():
        return key(gpu.search_batch_subsets(qs, p, subs))

    def f_serial():
        return key([gpu.search_batch([q], p, subset=s)[0] for q, s in zip(qs, subs)])

    def f_threads():
        out = [None] * len(qs)

        def worker(t):
            for i in range(t, len(qs), a.threads):
                out[i] = gpu.search_batch([qs[i]], p, subset=subs[i])[0]
        ths = [threading.Thread(target=worker, args=(t,)) for t in range(a.threads)]
        [t.start() for t in ths]
        [t.join() for t in ths]
        return key(out)

    def f_shared():
        return key(gpu.search_batch(qs, p, subset=shared))

    forms = dict(subsets=f_subsets, serial=f_serial, threads=f_threads, shared=f_shared)
    first = {k: f() for k, f in forms.items()}                # warm-up round, also the results compared
    identical = first["subsets"] == first["serial"] == first["threads"] and \
        first["shared"] == key(gpu.search_batch_subsets(qs, p, [shared] * len(qs)))
    qps = {k: [] for k in forms}
    for _ in range(a.runs):
        for k, f in forms.items():
            t = time.perf_counter()
            got = f()
            qps[k].append(len(qs) / (time.perf_counter() - t))
            identical = identical and got == first[k]
    gpu.close()
    info = bench.gpu_info(0)
    return dict(workload=name, docs=D, K=G["K"], batched=G["K"] > 100_000, queries=len(qs), subset_share=0.1,
                qps={k: dict(median=round(float(np.median(v)), 1), min=round(min(v), 1), max=round(max(v), 1))
                     for k, v in qps.items()},
                speedup_vs_serial=round(float(np.median(qps["subsets"]) / np.median(qps["serial"])), 2),
                speedup_vs_threads=round(float(np.median(qps["subsets"]) / np.median(qps["threads"])), 2),
                identical=bool(identical), gpu=info["name"], power_limit_w=info["power_limit_w"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="B,dense")
    ap.add_argument("--queries", type=int, default=32)
    ap.add_argument("--threads", type=int, default=8)
    ap.add_argument("--runs", type=int, default=5)
    a = ap.parse_args()
    for name in a.workloads.split(","):
        print(json.dumps(run_workload(name, a)), flush=True)


if __name__ == "__main__":
    main()
