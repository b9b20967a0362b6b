"""The device row cache of a host-tier handle (DESIGN.md 4s) on the config-B corpus (1M docs x 300 tokens x 128-d, 4-bit
residuals, K = 2^18, bench.py's generator; batches of 32 queries of 32 tokens, top_k 100, n_full_scores 4096).

Arms, in one process on one GPU, alternated within each run: a resident handle, and one host-tier handle with cache
budgets of 0, 25, 50 and 100 % of its rows.  For each host arm: the budget is set afresh (counts start at zero), --warm
batches of the same source are searched, the cache is filled by counts, and then the --steps timed batches run.

Two query sources, each a query from nq tokens of one source doc as bench.py builds them (docs of the generator's first
chunk, the docs it decodes):
  uniform   source docs drawn uniformly, as bench.py draws them
  zipf      source docs drawn with P(rank r) ~ 1 / r (s = 1) over a seeded permutation of those docs, so that
            popularity is not tied to position

Prints one JSON line: per source and arm the queries/s of each run (median, min, max), the hit rate of the timed
batches (hit_docs / staged_docs), the staging kernels' device time per batch (pb_last_staging_stats, a separate
profiled pass), the fill time and cached share, the handle's device bytes after the fill (pb_index_memory), and whether
every arm returned the resident arm's ids and scores; with the card's name and power limit.

Run from the repository root on an H100: python tools/bench_row_cache.py [--docs-total 1000000]"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

SHARES = (0.0, 0.25, 0.5, 1.0)


def queries_of(bench, args, G, dev, src, seed):
    """bench.make_queries for the given source docs (of the first chunk)"""
    import torch
    _, chunk, _ = bench.chunk_layout(args, 1)
    codes, res = bench.gen_chunk(args, G, 0, chunk, dev)
    T, nbits, dim = args.doclen, args.nbits, args.dim
    rng = np.random.default_rng(seed)
    shifts = torch.tensor([8 - nbits * (j + 1) for j in range(8 // nbits)], device=dev, dtype=torch.int32)
    w = G["bucket_weights"]
    w_rev = torch.stack([w[bench._bitrev(f, nbits)] for f in range(1 << nbits)])
    out = []
    for d in src:
        tok = torch.from_numpy(rng.integers(0, T, size=args.nq)).to(dev) + int(d) * T
        fields = ((res[tok].to(torch.int32).unsqueeze(-1) >> shifts) & ((1 << nbits) - 1)).reshape(args.nq, dim)
        v = G["centroids"][codes[tok]] + w_rev[fields.to(torch.int64)]
        v = (v / v.norm(dim=1, keepdim=True).clamp_min(1e-12)).cpu().numpy()
        noise = rng.standard_normal(v.shape).astype(np.float32)
        noise /= np.linalg.norm(noise, axis=1, keepdims=True)
        q = v + args.query_noise * noise
        out.append(np.ascontiguousarray(q / np.linalg.norm(q, axis=1, keepdims=True), np.float32))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs-total", type=int, default=1_000_000)
    ap.add_argument("--steps", type=int, default=20, help="timed batches per arm and run")
    ap.add_argument("--warm", type=int, default=20, help="batches searched before the fill by counts")
    ap.add_argument("--runs", type=int, default=2, help="runs per source, the arms alternated within each")
    ap.add_argument("--batch", type=int, default=32)
    a = ap.parse_args()
    sys.argv = [sys.argv[0], "--docs-total", str(a.docs_total), "--batch", str(a.batch)]
    import bench
    import torch
    import next_plaid_b200 as npb
    args = bench.parse_args()
    dev = torch.device("cuda", 0)
    G = bench.corpus_globals(args, dev)
    sh = bench.build_shard(args, G, 0, 1, dev)
    packed = args.dim * args.nbits // 8
    rows = sh["N"] * packed
    _, chunk, _ = bench.chunk_layout(args, 1)
    perm = np.random.default_rng(7).permutation(chunk)
    zipf_p = 1.0 / np.arange(1, chunk + 1)
    zipf_p /= zipf_p.sum()

    def batches(source, n, seed):
        rng = np.random.default_rng(seed)
        out = []
        for s in range(n):
            src = rng.integers(0, chunk, a.batch) if source == "uniform" else perm[rng.choice(chunk, a.batch, p=zipf_p)]
            out.append(queries_of(bench, args, G, dev, src, seed * 1000 + s))
        return out

    p = npb.SearchParameters(top_k=args.top_k, n_ivf_probe=args.n_ivf_probe, n_full_scores=args.n_full_scores,
                             centroid_score_threshold=args.threshold)

    def open_tier(host):
        return npb.MmapIndex.from_device_pointers(
            args.dim, args.nbits, G["K"], sh["D"], sh["N"], G["centroids"].data_ptr(), G["bucket_weights"].data_ptr(),
            sh["codes"].data_ptr(), sh["residuals"].data_ptr(), sh["doc_lengths"].data_ptr(), None, None,
            adopt_residuals=not host, host_residuals=host)

    res, host = open_tier(False), open_tier(True)
    base_bytes = host.memory_usage()["device_bytes"]

    def search(h, qsets):
        return [[(r.passage_ids.tolist(), r.scores.tobytes()) for r in h.search_batch(qs, p)] for qs in qsets]

    out, identical = {}, True
    for source, seed in (("uniform", 11), ("zipf", 12)):
        warm, timed = batches(source, a.warm, seed), batches(source, a.steps, seed + 100)
        want = search(res, timed)                                         # also the resident arm's warm-up
        arms = {"resident": dict(qps=[])}
        arms.update({f"host_{int(s * 100)}": dict(qps=[], hit_rate=[], fill_ms=[], cached_share=[]) for s in SHARES})
        for _ in range(a.runs):
            for name, arm in arms.items():
                h = res if name == "resident" else host
                if h is host:
                    share = int(name.split("_")[1]) / 100
                    host.set_row_cache(0)                                  # counts start at zero
                    if share:
                        host.set_row_cache(int(rows * share))
                    search(host, warm)
                    if share:
                        host.fill_row_cache()
                        st = host.row_cache_stats(reset=True)
                        arm["fill_ms"].append(round(st["last_fill_ms"], 1))
                        arm["cached_share"].append(round(st["cached_bytes"] / rows, 4))
                        arm["device_bytes"] = host.memory_usage()["device_bytes"]
                torch.cuda.synchronize(dev)
                t = time.perf_counter()
                got = search(h, timed)
                arm["qps"].append(round(a.batch * a.steps / (time.perf_counter() - t), 1))
                identical &= got == want
                if h is host and share:
                    st = host.row_cache_stats(reset=True)
                    arm["hit_rate"].append(round(st["hit_docs"] / max(st["staged_docs"], 1), 4))
                if h is host and "staging_ms" not in arm:               # profiled, outside the timed window
                    host.set_profiling(True)
                    ms = []
                    for qs in timed[:5]:
                        host.search_batch(qs, p)
                        ms.append(host.last_staging_stats()["ms"])
                    host.set_profiling(False)
                    arm["staging_ms"] = round(float(np.median(ms)), 2)
        for arm in arms.values():
            v = arm["qps"]
            arm["qps"] = dict(median=round(float(np.median(v)), 1), min=min(v), max=max(v), runs=v)
        out[source] = arms
    host.set_row_cache(0)
    assert host.memory_usage()["device_bytes"] == base_bytes
    res.close()
    host.close()
    info = bench.gpu_info(0)
    print(json.dumps({
        "workload": f"{sh['D']} docs x {args.doclen} tok, dim {args.dim}, nbits {args.nbits}, K 2^{args.log2k}, batch "
                    f"{a.batch} x {args.nq} tok, top_k {args.top_k}, n_full_scores {args.n_full_scores}",
        "rows_bytes": rows, "host_device_bytes_without_cache": base_bytes, "steps": a.steps, "warm": a.warm,
        "runs": a.runs, "sources": out, "identical": bool(identical),
        "gpu": info["name"], "power_limit_w": info["power_limit_w"]}))


if __name__ == "__main__":
    main()
