"""Per-query search parameters (pb_search_batch_params) against the ways a server could serve the same requests without
it.  Config B, generated on the device with bench.py's generator: 1M docs x 300 tokens x 128-d, 4-bit residuals,
K = 2^18 (the batched variant), 32-token queries, centroid_score_threshold 0.4.  Each batch holds 32 queries whose
parameters are drawn from top_k in {10, 100}, n_ivf_probe in {8, 32} and n_full_scores in {1024, 4096}, served as
  mixed     one pb_search_batch_params call
  grouped   one pb_search_batch call per distinct parameter tuple (what a caller had to do before)
  single    32 batch-of-1 pb_search_batch calls
Every form is checked to return identical ids and scores.  Wall clock around the calls with host buffers; --runs runs
of each form, alternating, after one warm-up round; median, min and max queries/s.  Prints one JSON line with the card
and its power limit.

Run from the repository root on an H100: python tools/bench_search_params.py"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--queries", type=int, default=32)
    ap.add_argument("--runs", type=int, default=20)
    a = ap.parse_args()
    sys.argv = [sys.argv[0], "--docs-total", "1000000", "--log2k", "18", "--batch", str(a.queries)]
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
    qs = bench.make_queries(args, G, dev, a.queries, seed=args.seed + 11)
    rng = np.random.default_rng(6)
    ps = [npb.SearchParameters(top_k=int(rng.choice([10, 100])), n_ivf_probe=int(rng.choice([8, 32])),
                               n_full_scores=int(rng.choice([1024, 4096])), centroid_score_threshold=args.threshold)
          for _ in qs]
    tuples = {}
    for i, p in enumerate(ps):
        tuples.setdefault((p.top_k, p.n_ivf_probe, p.n_full_scores), []).append(i)

    def key(res):
        return [(r.passage_ids.tolist(), r.scores.tobytes()) for r in res]

    def f_mixed():
        return key(gpu.search_batch_params(qs, ps))

    def f_grouped():
        out = [None] * len(qs)
        for idx in tuples.values():
            for i, r in zip(idx, gpu.search_batch([qs[i] for i in idx], ps[idx[0]])):
                out[i] = r
        return key(out)

    def f_single():
        return key([gpu.search_batch([q], p)[0] for q, p in zip(qs, ps)])

    forms = dict(mixed=f_mixed, grouped=f_grouped, single=f_single)
    first = {k: f() for k, f in forms.items()}                # warm-up round, also the results compared
    identical = first["mixed"] == first["grouped"] == first["single"]
    qps = {k: [] for k in forms}
    for _ in range(a.runs):
        for k, f in forms.items():
            t = time.perf_counter()
            got = f()
            qps[k].append(len(qs) / (time.perf_counter() - t))
            identical = identical and got == first[k]
    gpu.close()
    info = bench.gpu_info(0)
    print(json.dumps(dict(
        workload="B", docs=sh["D"], K=G["K"], queries=len(qs), distinct_tuples=len(tuples),
        qps={k: dict(median=round(float(np.median(v)), 1), min=round(min(v), 1), max=round(max(v), 1))
             for k, v in qps.items()},
        speedup_vs_grouped=round(float(np.median(qps["mixed"]) / np.median(qps["grouped"])), 2),
        speedup_vs_single=round(float(np.median(qps["mixed"]) / np.median(qps["single"])), 2),
        identical=bool(identical), gpu=info["name"], power_limit_w=info["power_limit_w"])), flush=True)


if __name__ == "__main__":
    main()
