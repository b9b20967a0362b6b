"""Host-tier search (PB_OPEN_HOST_RESIDUALS) against resident search on the config-B corpus (1M docs x 300 tokens x
128-d, 4-bit residuals, K = 2^18, bench.py's generator; batches of 32 queries of 32 tokens, top_k 100, n_full_scores
4096).  The corpus is generated on the device as bench.py does; the resident handle uses that residual array in place,
the host-tier handle copies it into about 19 GB of pinned host memory.  No larger corpus is built: the point of the tier
is capacity, and what one GPU could hold in this mode is arithmetic (DESIGN.md 4j), not something this tool measures.

In one process on one GPU it prints one JSON line with
  open_s / memory      time to open each tier (host clock, the call ends synchronised) and its memory_usage()
  qps                  queries/s of each tier with lanes 1 and 2: --steps batches per run (wall clock around search
                       calls with host buffers), --runs runs per tier alternating resident / host; median, min and max
  identical            whether both tiers returned the same ids and scores on every timed query
  staging              a separate profiled pass: the staging kernels' device time and GB/s per batch
                       (pb_last_staging_stats), next to a plain pinned cudaMemcpy H2D of the same byte count
  repeat_share         the share of staged docs that another query of the same batch also kept (traced calls)
  gpu, power_limit_w   what the numbers were measured on

Run from the repository root on an H100: python tools/bench_host_residuals.py [--docs-total 1000000]"""
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
    ap.add_argument("--steps", type=int, default=20, help="batches per timed run")
    ap.add_argument("--runs", type=int, default=3, help="timed runs per tier and lane setting (alternating)")
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
    qsets = [bench.make_queries(args, G, dev, a.batch, seed=100 + s) for s in range(a.steps)]
    p = npb.SearchParameters(top_k=args.top_k, n_ivf_probe=args.n_ivf_probe, n_full_scores=args.n_full_scores,
                             centroid_score_threshold=args.threshold)

    def open_tier(host):
        torch.cuda.synchronize(dev)
        t = time.perf_counter()
        h = npb.MmapIndex.from_device_pointers(
            args.dim, args.nbits, G["K"], sh["D"], sh["N"], G["centroids"].data_ptr(), G["bucket_weights"].data_ptr(),
            sh["codes"].data_ptr(), sh["residuals"].data_ptr(), sh["doc_lengths"].data_ptr(), None, None,
            adopt_residuals=not host, host_residuals=host)
        return h, time.perf_counter() - t

    res, t_res = open_tier(False)
    host, t_host = open_tier(True)
    tiers = dict(resident=res, host=host)
    out = dict(open_s=dict(resident=round(t_res, 2), host=round(t_host, 2)),
               memory={k: h.memory_usage() for k, h in tiers.items()})

    def run(h):
        got = []
        t = time.perf_counter()
        for qs in qsets:
            got.append([(r.passage_ids.tolist(), r.scores.tobytes()) for r in h.search_batch(qs, p)])
        return a.batch * a.steps / (time.perf_counter() - t), got

    identical = True
    qps = {}
    for lanes in (1, 2):
        for h in tiers.values():
            h.set_lanes(lanes)
            run(h)                                                 # warm-up: modules, workspaces, staging buffers
        rates = {k: [] for k in tiers}
        for _ in range(a.runs):
            want = None
            for k, h in tiers.items():
                r, got = run(h)
                rates[k].append(r)
                if want is None:
                    want = got
                identical &= got == want
        for k, v in rates.items():
            qps[f"{k}_lanes{lanes}"] = dict(median=round(float(np.median(v)), 1), min=round(min(v), 1),
                                            max=round(max(v), 1), runs=[round(x, 1) for x in v])
        for h in tiers.values():
            h.set_lanes(1)
    out["qps"] = qps
    out["identical"] = bool(identical)

    # staging kernels, profiled, against a plain pinned H2D copy of the same bytes per batch
    host.set_profiling(True)
    st_ms, st_bytes, st_docs = [], [], []
    for qs in qsets:
        host.search_batch(qs, p)
        s = host.last_staging_stats()
        st_ms.append(s["ms"])
        st_bytes.append(s["bytes"])
        st_docs.append(s["docs"])
    host.set_profiling(False)
    nb = int(np.median(st_bytes))
    src = torch.empty(nb, dtype=torch.uint8, pin_memory=True)
    dst = torch.empty(nb, dtype=torch.uint8, device=dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    dst.copy_(src, non_blocking=True)
    copy_ms = []
    for _ in range(5):
        e0.record()
        dst.copy_(src, non_blocking=True)
        e1.record()
        e1.synchronize()
        copy_ms.append(e0.elapsed_time(e1))
    del src, dst
    ms = float(np.median(st_ms))
    out["staging"] = dict(docs_per_batch=int(np.median(st_docs)), bytes_per_batch=nb, kernel_ms=round(ms, 3),
                          kernel_gbps=round(nb / ms / 1e6, 2) if ms > 0 else None,
                          memcpy_h2d_ms=round(float(np.median(copy_ms)), 3),
                          memcpy_h2d_gbps=round(nb / float(np.median(copy_ms)) / 1e6, 2))

    # docs kept by more than one query of a batch (staged once per query today)
    staged = repeats = 0
    for qs in qsets[:5]:
        _, tr = host.search_batch(qs, p, trace=True)
        kept = np.concatenate(tr.kept)
        staged += len(kept)
        repeats += len(kept) - len(np.unique(kept))
    out["repeat_share"] = round(repeats / max(staged, 1), 4)
    res.close()
    host.close()
    info = bench.gpu_info(0)
    print(json.dumps({
        "workload": f"{sh['D']} docs x {args.doclen} tok, dim {args.dim}, nbits {args.nbits}, K 2^{args.log2k}, batch "
                    f"{a.batch} x {args.nq} tok, top_k {args.top_k}, n_full_scores {args.n_full_scores}",
        "packed_bytes_per_token": packed, "steps": a.steps, "runs": a.runs, **out,
        "gpu": info["name"], "power_limit_w": info["power_limit_w"]}))


if __name__ == "__main__":
    main()
