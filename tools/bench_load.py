"""Loading an index directory whole and as doc shards, on the config-B corpus (1M docs x 300 tokens x 128-d, 4-bit
residuals, K = 2^18, in chunk files of 50 000 docs; codes and residuals from bench.py's device generator, ivf.npy the
inverted file the library builds from them on the device).  The directory is written to a temporary directory under
--dir (about 24 GB at the default size; --docs-total scales it down) and removed at the end.

In one process on one GPU it times pb_index_load of the whole directory, then pb_index_load_range of every shard of
pb_index_dir_shard_bounds for W = 2 and 4, one shard after another, each closed before the next:

  ms           host clock around the call (it ends synchronised), median of --repeats
  chunk_bytes  bytes of chunk rows the call reads (codes <i8 and packed residuals of its tokens)
  ivf_bytes    bytes of ivf.npy it reads (the whole payload, on every rank)

and checks that a W-shard group of load_shard handles returns the same top-k ids and scores as the full load on
--queries queries (parity; queries_differing counts the queries whose results differ).  The page cache holds the
directory just written, so every number is a warm-cache load.  Prints one JSON line with the GPU name and power limit.

Run from the repository root on an H100: python tools/bench_load.py [--docs-total 1000000] [--dir /tmp]"""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402


def write_directory(path, args, G, npb, bench, dev):
    """The directory as create_index lays it out: one chunk file pair per 50 000 docs, ivf.npy from the device."""
    import torch
    per_rank, chunk, n_chunks = bench.chunk_layout(args, 1)
    T = args.doclen
    np.save(os.path.join(path, "centroids.npy"), G["centroids"].cpu().numpy())
    np.save(os.path.join(path, "bucket_weights.npy"), G["bucket_weights"].cpu().numpy())
    for c in range(n_chunks):
        codes, res = bench.gen_chunk(args, G, c, chunk, dev)
        np.save(os.path.join(path, f"{c}.codes.npy"), codes.cpu().numpy())
        np.save(os.path.join(path, f"{c}.residuals.npy"), res.cpu().numpy())
        del codes, res
        with open(os.path.join(path, f"doclens.{c}.json"), "w") as f:
            json.dump([T] * chunk, f)
        with open(os.path.join(path, f"{c}.metadata.json"), "w") as f:
            json.dump({"num_documents": chunk, "num_embeddings": chunk * T, "embedding_offset": c * chunk * T}, f)
    sh = bench.build_shard(args, G, 0, 1, dev)
    ix = bench.open_shard(npb, args, G, sh, 0, 0)
    ivf, lens = ix.export_ivf()
    ix.close()
    del sh
    torch.cuda.empty_cache()
    np.save(os.path.join(path, "ivf.npy"), ivf)
    np.save(os.path.join(path, "ivf_lengths.npy"), lens)
    with open(os.path.join(path, "metadata.json"), "w") as f:
        json.dump({"num_chunks": n_chunks, "nbits": args.nbits, "num_partitions": G["K"], "num_embeddings": per_rank * T,
                   "avg_doclen": float(T), "num_documents": per_rank, "embedding_dim": args.dim,
                   "next_plaid_compatible": True}, f)
    return per_rank, int(ivf.size) * 8


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
    args = bench.parse_args()
    dev = torch.device("cuda", 0)
    G = bench.corpus_globals(args, dev)
    T, packed = args.doclen, args.dim * args.nbits // 8
    need = a.docs_total * T * (8 + packed) * 1.15
    free = shutil.disk_usage(a.dir).free
    if free < need:
        raise SystemExit(f"{a.dir} has {free / 1e9:.1f} GB free, the directory needs about {need / 1e9:.1f} GB: "
                         "pass --dir elsewhere or a smaller --docs-total")
    path = tempfile.mkdtemp(prefix="pb_bench_load_", dir=a.dir)
    try:
        t0 = time.perf_counter()
        D, ivf_bytes = write_directory(path, args, G, npb, bench, dev)
        write_s = time.perf_counter() - t0
        qs = bench.make_queries(args, G, dev, a.queries, seed=11)
        del G
        torch.cuda.empty_cache()
        p = npb.SearchParameters(top_k=100, n_ivf_probe=8, n_full_scores=4096)

        def timed(fn):
            runs = []
            for _ in range(a.repeats):
                torch.cuda.synchronize(dev)
                t = time.perf_counter()
                h = fn()
                runs.append((time.perf_counter() - t) * 1e3)
                h.close()
                torch.cuda.empty_cache()
            return float(np.median(runs))

        npb.MmapIndex.load_range(path, 0, min(D, 1000)).close()      # warm-up: modules, CUB
        full = npb.MmapIndex.load(path)
        want = [(r.passage_ids.tolist(), r.scores.tobytes()) for r in full.search_batch(qs, p)]
        full.close()
        torch.cuda.empty_cache()
        out = {"full": dict(ms=timed(lambda: npb.MmapIndex.load(path)), chunk_bytes=D * T * (8 + packed),
                            ivf_bytes=ivf_bytes)}
        for W in (2, 4):
            b = npb.shard_bounds(path, W)
            ranks = []
            for r in range(W):
                lo, hi = int(b[r]), int(b[r + 1])
                ranks.append(dict(docs=[lo, hi], ms=timed(lambda: npb.MmapIndex.load_range(path, lo, hi)),
                                  chunk_bytes=(hi - lo) * T * (8 + packed), ivf_bytes=ivf_bytes))
            grp = npb.ShardGroup([npb.MmapIndex.load_shard(path, r, W) for r in range(W)])
            got = [(r.passage_ids.tolist(), r.scores.tobytes()) for r in grp.search_batch(qs, p)]
            grp.close()
            torch.cuda.empty_cache()
            out[f"W{W}"] = dict(ranks=ranks, max_rank_ms=max(x["ms"] for x in ranks), parity=bool(got == want),
                                queries_differing=sum(g != w for g, w in zip(got, want)))
    finally:
        shutil.rmtree(path, ignore_errors=True)
    info = bench.gpu_info(0)
    print(json.dumps({
        "workload": f"{D} docs x {T} tok, dim {args.dim}, nbits {args.nbits}, K 2^{args.log2k}, chunks of "
                    f"{bench.chunk_layout(args, 1)[1]} docs",
        "page_cache": "warm: the directory was written by this run just before", "write_s": round(write_s, 1),
        "repeats": a.repeats, **out, "gpu": info["name"], "power_limit_w": info["power_limit_w"]}))


if __name__ == "__main__":
    main()
