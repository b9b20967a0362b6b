"""Changing a live deployment's number of ranks on the device (pb_index_add_devices / pb_index_remove_ranks) against the
remedy without it, closing the handle and loading the directory again at the new world size with load_devices.

Corpus: config B's generator (300 tokens x 128-d, 4-bit residuals, K = 2^18) written as an index directory by
tools/bench_load.py's write_directory (--docs-total documents, chunk files of 50 000 docs).  load_devices opens it over
2 ranks on device 0; then add_devices([0]) (2 -> 3 ranks) and remove_ranks([2]) (3 -> 2) alternate, --repeats times
each way, both with the balanced bounds, so every call moves data.  `open_regroup_ms` times the same two calls with
bounds that move nothing (the new rank empty after the last one, and the removal of that empty rank): what opening an
empty rank, re-forming the group and closing a rank cost by themselves.  Each call is timed with a host clock around it
and a device synchronize.  `reload_ms` times load_devices of the directory at W = 3 and W = 2, the handle closed first.
Bytes moved are computed from shapes: the moved docs' codes, residuals and per-doc lengths.  The deployment's top-100
on --queries queries must equal pb_index_load's of the directory before the first and after every step.  Prints one
JSON line with the GPU name and power limit.

Run from the repository root on an H100: python tools/bench_resize.py [--docs-total 1000000] [--dir /tmp]"""
import argparse
import json
import os
import shutil
import statistics
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402


def moved_docs(old, new):
    """documents that change rank between two bounds of the same world (sharded_rebalance.plan without kept pieces)"""
    from sharded_rebalance import plan
    return sum(hi - lo for (s, r), (lo, hi) in plan(old, new).items() if s != r)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs-total", type=int, default=1_000_000)
    ap.add_argument("--dir", default=tempfile.gettempdir(), help="where the temporary index directory is written")
    ap.add_argument("--queries", type=int, default=64)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    sys.argv = [sys.argv[0], "--docs-total", str(a.docs_total)]
    import bench
    import torch
    import next_plaid_b200 as npb
    from bench_load import write_directory
    args = bench.parse_args()
    dev = torch.device("cuda", 0)
    G = bench.corpus_globals(args, dev)
    T, packed = args.doclen, args.dim * args.nbits // 8
    _, chunk, _ = bench.chunk_layout(args, 1)
    if a.docs_total % chunk:
        raise SystemExit(f"--docs-total must be a multiple of the chunk size {chunk}")
    need = 1.2 * a.docs_total * T * (8 + packed)
    if shutil.disk_usage(a.dir).free < need:
        raise SystemExit(f"{a.dir} needs about {need / 1e9:.1f} GB free: pass --dir elsewhere or a smaller --docs-total")
    root = tempfile.mkdtemp(prefix="pb_bench_resize_", dir=a.dir)
    try:
        D, _ = write_directory(root, args, G, npb, bench, dev)
        assert D == a.docs_total
        qs = bench.make_queries(args, G, dev, a.queries, seed=11)
        del G
        torch.cuda.empty_cache()
        p = npb.SearchParameters(top_k=100, n_ivf_probe=8, n_full_scores=4096)
        res = lambda h: [(r.passage_ids.tolist(), r.scores.tobytes()) for r in h.search_batch(qs, p)]  # noqa: E731
        single = npb.MmapIndex.load(root)
        want = res(single)
        single.close()
        torch.cuda.empty_cache()

        def timed(fn):
            torch.cuda.synchronize(dev)
            t = time.perf_counter()
            r = fn()
            torch.cuda.synchronize(dev)
            return r, round((time.perf_counter() - t) * 1e3, 1)

        b2, b3 = npb.shard_bounds(root, 2), npb.shard_bounds(root, 3)
        dep = npb.MmapIndex.load_devices(root, [0, 0])
        ms = {"add_2_to_3": [], "remove_3_to_2": []}
        idle = {"add_empty_rank": [], "remove_empty_rank": []}
        try:
            parity = [res(dep) == want]
            for _ in range(a.repeats):
                got, t = timed(lambda: dep.add_devices([0]))
                assert np.array_equal(got, b3)
                ms["add_2_to_3"].append(t)
                parity.append(res(dep) == want)
                got, t = timed(lambda: dep.remove_ranks([2]))
                assert np.array_equal(got, b2)
                ms["remove_3_to_2"].append(t)
                parity.append(res(dep) == want)
            for _ in range(a.repeats):
                _, t = timed(lambda: dep.add_devices([0], list(b2) + [D]))
                idle["add_empty_rank"].append(t)
                parity.append(res(dep) == want)
                _, t = timed(lambda: dep.remove_ranks([2], b2))
                idle["remove_empty_rank"].append(t)
                parity.append(res(dep) == want)
        finally:
            dep.close()
            torch.cuda.empty_cache()
        reload = {}
        for W in (3, 2):
            h, t = timed(lambda: npb.MmapIndex.load_devices(root, [0] * W))
            h.close()
            torch.cuda.empty_cache()
            reload[f"W{W}"] = t
        n_add = moved_docs(list(b2) + [D], b3)   # the 2-rank layout with an empty third rank -> the 3-rank split
        n_rem = moved_docs(b3, list(b2) + [D])
    finally:
        shutil.rmtree(root, ignore_errors=True)
    stat = lambda v: dict(median=statistics.median(v), runs=v)  # noqa: E731
    info = bench.gpu_info(0)
    print(json.dumps({
        "workload": f"{a.docs_total} docs x {T} tok, dim {args.dim}, nbits {args.nbits}, K 2^{args.log2k}, "
                    "2 <-> 3 ranks on device 0",
        "page_cache": "warm: the directory was written by this run",
        "resize_ms": {k: stat(v) for k, v in ms.items()},
        "open_regroup_ms": {k: stat(v) for k, v in idle.items()},
        "reload_ms": reload,
        "moved_docs": dict(add=n_add, remove=n_rem),
        "moved_bytes": dict(add=n_add * (T * (4 + packed) + 16), remove=n_rem * (T * (4 + packed) + 16)),
        "top100_equals_single": dict(before=parity[0], after_every_step=all(parity[1:])),
        "gpu": torch.cuda.get_device_name(0), "power_limit_w": info["power_limit_w"]}))


if __name__ == "__main__":
    main()
