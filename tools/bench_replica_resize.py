"""Changing a live replica set's number of replicas (pb_index_add_replicas / pb_index_remove_replicas) against the remedy
without it, closing the set and loading the directory again with load_replicas at the new R.

Corpus: config B's generator (300 tokens x 128-d, 4-bit residuals, K = 2^18) written as an index directory by
tools/bench_load.py's write_directory (--docs-total documents, chunk files of 50 000 docs).  The default 1M documents
make two copies plus search workspaces fit one 80 GB card.  load_replicas opens one replica on device 0; then
add_replicas([0]) (1 -> 2) and remove_replicas([1]) (2 -> 1) alternate --repeats times.  Each call is timed with a host
clock around it and a device synchronize.  `load_replicas_ms` times load_replicas of the directory at R = 2, the set
closed first.  During one more add, a background thread searches --batch queries per call in a loop on the set: its
throughput and its largest per-call latency during the add, against the same loop with no add running.  The set's
top-100 on --queries queries must equal pb_index_load's before the first and after every step.  Prints one JSON line
with the GPU name and power limit read in the same run.

Run from the repository root on an H100: python tools/bench_replica_resize.py [--docs-total 1000000] [--dir /tmp]"""
import argparse
import json
import os
import shutil
import statistics
import sys
import tempfile
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def search_loop(h, qs, p, stop, out):
    """search_batch of qs until stop is set; (calls, queries, seconds, largest call ms) into out"""
    n, worst, t0 = 0, 0.0, time.perf_counter()
    while not stop.is_set():
        t = time.perf_counter()
        h.search_batch(qs, p)
        worst = max(worst, (time.perf_counter() - t) * 1e3)
        n += 1
    s = time.perf_counter() - t0
    out.update(calls=n, qps=round(n * len(qs) / s, 1), max_call_ms=round(worst, 2), seconds=round(s, 3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs-total", type=int, default=1_000_000)
    ap.add_argument("--dir", default=tempfile.gettempdir(), help="where the temporary index directory is written")
    ap.add_argument("--queries", type=int, default=64)
    ap.add_argument("--batch", type=int, default=32, help="queries per call of the background search loop")
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
    root = tempfile.mkdtemp(prefix="pb_bench_replica_resize_", dir=a.dir)
    try:
        D, _ = write_directory(root, args, G, npb, bench, dev)
        assert D == a.docs_total
        qs = bench.make_queries(args, G, dev, max(a.queries, a.batch), seed=11)
        del G
        torch.cuda.empty_cache()
        p = npb.SearchParameters(top_k=100, n_ivf_probe=8, n_full_scores=4096)
        res = lambda h: [(r.passage_ids.tolist(), r.scores.tobytes()) for r in h.search_batch(qs[:a.queries], p)]  # noqa: E731
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

        ms = {"add_1_to_2": [], "remove_2_to_1": []}
        rep = npb.MmapIndex.load_replicas(root, [0])
        try:
            parity = [res(rep) == want]
            for _ in range(a.repeats):
                _, t = timed(lambda: rep.add_replicas([0]))
                ms["add_1_to_2"].append(t)
                parity.append(res(rep) == want)
                _, t = timed(lambda: rep.remove_replicas([1]))
                ms["remove_2_to_1"].append(t)
                parity.append(res(rep) == want)
            mem_1 = rep.memory_usage()["device_bytes"]
            # the background loop alone, then during an add (which it ends when the add returns)
            loop = qs[:a.batch]
            quiet, busy = {}, {}
            stop = threading.Event()
            th = threading.Thread(target=search_loop, args=(rep, loop, p, stop, quiet))
            th.start()
            time.sleep(max(1.0, statistics.median(ms["add_1_to_2"]) / 1e3))
            stop.set()
            th.join()
            stop = threading.Event()
            th = threading.Thread(target=search_loop, args=(rep, loop, p, stop, busy))
            th.start()
            time.sleep(0.2)
            _, t_add = timed(lambda: rep.add_replicas([0]))
            stop.set()
            th.join()
            parity.append(res(rep) == want)
            mem_2 = rep.memory_usage()["device_bytes"]
        finally:
            rep.close()
            torch.cuda.empty_cache()
        h, t_load = timed(lambda: npb.MmapIndex.load_replicas(root, [0, 0]))
        parity.append(res(h) == want)
        h.close()
        torch.cuda.empty_cache()
    finally:
        shutil.rmtree(root, ignore_errors=True)
    stat = lambda v: dict(median=statistics.median(v), runs=v)  # noqa: E731
    info = bench.gpu_info(0)
    print(json.dumps({
        "workload": f"{a.docs_total} docs x {T} tok, dim {args.dim}, nbits {args.nbits}, K 2^{args.log2k}, "
                    "1 <-> 2 replicas on device 0",
        "page_cache": "warm: the directory was written by this run",
        "resize_ms": {k: stat(v) for k, v in ms.items()},
        "load_replicas_R2_ms": t_load,
        "replica_device_bytes": mem_2 - mem_1,
        "copy_gb_per_s": round((mem_2 - mem_1) / (stat(ms["add_1_to_2"])["median"] * 1e6), 1),
        "search_loop": dict(batch=a.batch, without_add=quiet, during_add=dict(busy, add_ms=t_add)),
        "top100_equals_single": dict(before=parity[0], after_every_step=all(parity[1:])),
        "gpu": torch.cuda.get_device_name(0), "power_limit_w": info["power_limit_w"]}))


if __name__ == "__main__":
    main()
