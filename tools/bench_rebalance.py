"""Rebalancing a doc-sharded deployment on the device (pb_index_rebalance_sharded) against the remedy without it,
reloading every rank with pb_index_load_range at the new bounds.

Corpus: config B's generator (300 tokens x 128-d, 4-bit residuals, K = 2^18) written as an index directory by
tools/bench_load.py's write_directory with --docs-total + --n-append documents (chunk files of 50 000 docs).  For each
W in --widths an in-process shard group on device 0 opens the first --docs-total documents with load_range at the
balanced split, then appends the directory's last --n-append documents, encoded, to the last rank
(pb_index_append_encoded_sharded), so the group holds the directory's documents at skewed bounds.  Then rebalance()
alternates between the balanced and the skewed bounds, --repeats times each way, so that every run moves data; each
call is timed with a host clock (it ends in a device synchronize).  `reload_ms` times load_range of every rank at the
balanced bounds, one after another (sum and slowest rank).  Bytes moved are computed from shapes: the moved docs'
codes, residuals and per-doc lengths.  The group's top-100 on --queries queries must equal pb_index_load's of the
directory before the first and after every rebalance.  Prints one JSON line with the GPU name and power limit.

Run from the repository root on an H100: python tools/bench_rebalance.py [--docs-total 1000000] [--dir /tmp]"""
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
    """documents that change rank between the two bounds (sharded_rebalance.plan without the kept pieces)"""
    from sharded_rebalance import plan
    return sum(hi - lo for (s, r), (lo, hi) in plan(old, new).items() if s != r)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs-total", type=int, default=1_000_000)
    ap.add_argument("--n-append", type=int, default=100_000)
    ap.add_argument("--dir", default=tempfile.gettempdir(), help="where the temporary index directory is written")
    ap.add_argument("--queries", type=int, default=64)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--widths", default="2,4")
    a = ap.parse_args()
    total = a.docs_total + a.n_append
    sys.argv = [sys.argv[0], "--docs-total", str(total)]
    import bench
    import torch
    import next_plaid_b200 as npb
    from bench_load import write_directory
    args = bench.parse_args()
    dev = torch.device("cuda", 0)
    G = bench.corpus_globals(args, dev)
    T, packed = args.doclen, args.dim * args.nbits // 8
    _, chunk, _ = bench.chunk_layout(args, 1)
    if a.docs_total % chunk or a.n_append % chunk:
        raise SystemExit(f"--docs-total and --n-append must be multiples of the chunk size {chunk}")
    need = 1.2 * total * T * (8 + packed)
    if shutil.disk_usage(a.dir).free < need:
        raise SystemExit(f"{a.dir} needs about {need / 1e9:.1f} GB free: pass --dir elsewhere or a smaller --docs-total")
    root = tempfile.mkdtemp(prefix="pb_bench_rebalance_", dir=a.dir)
    try:
        D, _ = write_directory(root, args, G, npb, bench, dev)
        assert D == total
        qs = bench.make_queries(args, G, dev, a.queries, seed=11)
        app = [bench.gen_chunk(args, G, c, chunk, dev) for c in range(a.docs_total // chunk, total // chunk)]
        codes = np.concatenate([x[0].cpu().numpy() for x in app])
        res = np.concatenate([x[1].cpu().numpy() for x in app])
        del app, G
        torch.cuda.empty_cache()
        p = npb.SearchParameters(top_k=100, n_ivf_probe=8, n_full_scores=4096)
        single = npb.MmapIndex.load(root)
        want = [(r.passage_ids.tolist(), r.scores.tobytes()) for r in single.search_batch(qs, p)]
        single.close()
        torch.cuda.empty_cache()

        def timed(fn):
            torch.cuda.synchronize(dev)
            t = time.perf_counter()
            r = fn()
            return r, (time.perf_counter() - t) * 1e3

        def run(W):
            base = [r * a.docs_total // W for r in range(W)] + [a.docs_total]
            grp = npb.ShardGroup([npb.MmapIndex.load_range(root, base[r], base[r + 1]) for r in range(W)])
            out = {}
            try:
                grp.append_encoded(codes, res, [T] * a.n_append)
                skewed = np.array(base[:-1] + [total], np.int64)
                balanced = npb.shard_bounds(root, W)
                parity = [[(r.passage_ids.tolist(), r.scores.tobytes()) for r in grp.search_batch(qs, p)] == want]
                ms = {"to_balanced": [], "to_skewed": []}
                cur = skewed
                for i in range(2 * a.repeats):
                    nxt, key = (balanced, "to_balanced") if i % 2 == 0 else (skewed, "to_skewed")
                    got, t = timed(lambda: grp.rebalance(nxt))
                    assert np.array_equal(got, nxt)
                    ms[key].append(round(t, 1))
                    parity.append([(r.passage_ids.tolist(), r.scores.tobytes())
                                   for r in grp.search_batch(qs, p)] == want)
                    cur = nxt
                assert np.array_equal(cur, skewed)
            finally:
                grp.close()
                torch.cuda.empty_cache()
            per = []
            for r in range(W):
                h, t = timed(lambda: npb.MmapIndex.load_range(root, int(balanced[r]), int(balanced[r + 1])))
                h.close()
                torch.cuda.empty_cache()
                per.append(t)
            n = moved_docs(skewed, balanced)
            out.update(
                bounds=dict(skewed=skewed.tolist(), balanced=balanced.tolist()),
                rebalance_ms={k: dict(median=statistics.median(v), runs=v) for k, v in ms.items()},
                reload_ms=dict(sum=round(sum(per), 1), slowest_rank=round(max(per), 1)),
                moved_docs=n, moved_bytes=n * (T * (4 + packed) + 16),
                top100_equals_single=dict(before=parity[0], after_every_rebalance=all(parity[1:])))
            return out

        groups = {f"W{W}": run(W) for W in (int(w) for w in a.widths.split(","))}
    finally:
        shutil.rmtree(root, ignore_errors=True)
    info = bench.gpu_info(0)
    print(json.dumps({
        "workload": f"{a.docs_total} docs x {T} tok + {a.n_append} appended to the last rank, dim {args.dim}, "
                    f"nbits {args.nbits}, K 2^{args.log2k}",
        "page_cache": "warm: the directory was written by this run", **groups,
        "gpu": torch.cuda.get_device_name(0), "power_limit_w": info["power_limit_w"]}))


if __name__ == "__main__":
    main()
