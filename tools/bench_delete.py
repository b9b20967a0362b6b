"""Incremental delete on the config-B corpus (1M docs x 300 tokens x 128-d, 4-bit residuals, K = 2^18, built on the
device exactly as bench.py builds it): pb_index_delete of 10 000 docs -- scattered, the oldest (the whole index moves)
and the newest (nothing moves) -- against pb_index_close + pb_index_open of the filtered device arrays.  Checks that the
deleted handle and the fresh open return identical searches on 64 queries and prints one JSON line.

  delete_ms   host clock around pb_index_delete (the call ends synchronised), median of --repeats
  compact_ms, ivf_ms, norms_ms
              device time of the in-place compaction, the inverted-file kernels and the k_min_vnorm pass, from the
              library's CUDA events (pb_set_profiling) in a separate profiled call
  reopen_ms   close + open of the filtered device arrays

Run from the repository root on an H100: python tools/bench_delete.py [--docs-total 1000000] [--del-docs 10000]"""
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
    ap.add_argument("--docs-total", type=int, default=1_000_000)
    ap.add_argument("--del-docs", type=int, default=10_000)
    ap.add_argument("--queries", type=int, default=64)
    ap.add_argument("--repeats", type=int, default=2)
    a = ap.parse_args()
    sys.argv = [sys.argv[0], "--docs-total", str(a.docs_total)]
    import bench
    import torch
    import next_plaid_b200 as npb
    args = bench.parse_args()
    dev = torch.device("cuda", 0)
    G = bench.corpus_globals(args, dev)
    K, T, dim, nbits = G["K"], args.doclen, args.dim, args.nbits
    per_rank, _, _ = bench.chunk_layout(args, 1)
    qs = bench.make_queries(args, G, dev, a.queries, seed=11)
    p = npb.SearchParameters(top_k=100, n_ivf_probe=8, n_full_scores=4096)
    n = a.del_docs
    patterns = {
        "scattered": np.sort(np.random.default_rng(5).choice(per_rank, n, replace=False)).astype(np.int64),
        "oldest": np.arange(n, dtype=np.int64),
        "newest": np.arange(per_rank - n, per_rank, dtype=np.int64),
    }

    def open_arrays(keep=None):
        sh = bench.build_shard(args, G, 0, 1, dev)
        codes, res, dl = sh["codes"], sh["residuals"], sh["doc_lengths"]
        del sh
        if keep is not None:
            kd = torch.from_numpy(keep).to(dev)
            kt = torch.repeat_interleave(kd, dl)
            codes, res, dl = codes[kt], res[kt], dl[kd]
            del kd, kt
        torch.cuda.empty_cache()
        D, N = len(dl), len(codes)
        t0 = time.perf_counter()
        ix = npb.MmapIndex.from_device_pointers(dim, nbits, K, D, N, G["centroids"].data_ptr(),
                                                G["bucket_weights"].data_ptr(), codes.data_ptr(), res.data_ptr(),
                                                dl.data_ptr(), None, None)
        torch.cuda.synchronize(dev)
        ms = (time.perf_counter() - t0) * 1e3
        del codes, res, dl
        torch.cuda.empty_cache()
        return ix, ms

    def search(ix):
        return [(r.passage_ids.tolist(), r.scores.tobytes()) for r in ix.search_batch(qs, p)]

    # warm-up: one delete on a small index (modules, CUB)
    small, _ = open_arrays(np.arange(per_rank) < 2000)
    small.delete(range(0, 2000, 3))
    small.close()
    torch.cuda.empty_cache()
    out = {}
    for name, ids in patterns.items():
        runs, res_del = [], None
        for rep in range(a.repeats):
            ix, _ = open_arrays()
            torch.cuda.synchronize(dev)
            t0 = time.perf_counter()
            got = ix.delete(ids)
            runs.append((time.perf_counter() - t0) * 1e3)
            assert got == n
            if rep == 0:
                res_del = search(ix)
            ix.close()
            torch.cuda.empty_cache()
        ix, _ = open_arrays()
        ix.set_profiling(True)
        ix.delete(ids)
        prof = ix.last_delete_ms()
        ix.close()
        torch.cuda.empty_cache()
        keep = np.ones(per_rank, bool)
        keep[ids] = False
        reopen, res_fresh = [], None
        for rep in range(a.repeats):
            fresh, ms_open = open_arrays(keep)
            if res_fresh is None:
                res_fresh = search(fresh)
            torch.cuda.synchronize(dev)
            t0 = time.perf_counter()
            fresh.close()
            reopen.append(ms_open + (time.perf_counter() - t0) * 1e3)
            torch.cuda.empty_cache()
        out[name] = dict(delete_ms=float(np.median(runs)), **prof, reopen_ms=float(np.median(reopen)),
                         parity=bool(res_del == res_fresh))
    info = bench.gpu_info(0)
    print(json.dumps({
        "workload": f"{per_rank} docs x {T} tok, delete of {n} docs, dim {dim}, nbits {nbits}, K 2^{args.log2k}",
        **out, "gpu": info["name"], "power_limit_w": info["power_limit_w"]}))


if __name__ == "__main__":
    main()
