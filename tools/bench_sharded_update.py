"""Deletes and appends on a doc-sharded deployment against the same changes on one handle and against a reload, on the
config-B corpus written as an index directory by tools/bench_load.py's write_directory (1M docs x 300 tokens x 128-d,
4-bit residuals, K = 2^18; --docs-total scales it down).

Every configuration starts from its own hard-linked copy of the directory and runs the same four operations in order:

  delete            --n-delete scattered docs, device only          (pb_index_delete / pb_index_delete_sharded)
  append_encoded    --n-append docs x 300 tokens, already encoded   (pb_index_append_encoded / _sharded)
  delete_dir        another --n-delete scattered docs, with the directory
  append_dir        --n-append docs x 300 tokens encoded on the device, with the directory (pb_index_append / _sharded)

The configurations run one after another, so two copies of the index never share the card: `single` (pb_index_load),
then W = 2 and W = 4 (--widths) load_shard handles in one in-process shard group on device 0.  Each operation is timed with a host
clock around the call (it ends synchronised).  `reload_ms` times what a deployment without these calls does instead:
pb_index_load, or pb_index_load_range of every shard one after another (sum and slowest rank).  After every operation the
group's top-k ids and scores on --queries queries must equal the single handle's after the same operation (parity).
Prints one JSON line with the GPU name and power limit.

Run from the repository root on an H100: python tools/bench_sharded_update.py [--docs-total 1000000] [--dir /tmp]"""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs-total", type=int, default=1_000_000)
    ap.add_argument("--dir", default=tempfile.gettempdir(), help="where the temporary index directories are written")
    ap.add_argument("--queries", type=int, default=64)
    ap.add_argument("--n-delete", type=int, default=10_000)
    ap.add_argument("--n-append", type=int, default=10_000)
    ap.add_argument("--widths", default="2,4", help="group sizes to run after the single handle, e.g. 2 or 2,4")
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
    need = 2.3 * a.docs_total * T * (8 + packed)       # the directory and one configuration's rewritten files
    free = shutil.disk_usage(a.dir).free
    if free < need:
        raise SystemExit(f"{a.dir} has {free / 1e9:.1f} GB free, two directories need about {need / 1e9:.1f} GB: "
                         "pass --dir elsewhere or a smaller --docs-total")
    root = tempfile.mkdtemp(prefix="pb_bench_sharded_update_", dir=a.dir)
    pristine = os.path.join(root, "pristine")
    os.mkdir(pristine)
    try:
        D, _ = write_directory(pristine, args, G, npb, bench, dev)
        qs = bench.make_queries(args, G, dev, a.queries, seed=11)
        rng = np.random.default_rng(5)
        del1 = rng.choice(D, a.n_delete, replace=False)
        del2 = rng.choice(D - a.n_delete, a.n_delete, replace=False)
        codes, res = bench.gen_chunk(args, G, 10_000, a.n_append, dev)    # a chunk index the directory does not use
        codes, res = codes.cpu().numpy(), res.cpu().numpy()
        dl = [T] * a.n_append
        cent = G["centroids"].cpu().numpy()
        emb = [cent[codes[i * T:(i + 1) * T]] + 0.01 * rng.standard_normal((T, args.dim)).astype(np.float32)
               for i in range(a.n_append)]
        cutoffs = np.linspace(-0.02, 0.02, (1 << args.nbits) - 1).astype(np.float32)
        codec = npb.ResidualCodec(args.nbits, cent, cutoffs)
        del G
        torch.cuda.empty_cache()
        p = npb.SearchParameters(top_k=100, n_ivf_probe=8, n_full_scores=4096)
        npb.MmapIndex.load_range(pristine, 0, min(D, 1000)).close()        # warm-up: modules, CUB

        def timed(fn):
            torch.cuda.synchronize(dev)
            t = time.perf_counter()
            r = fn()
            return r, round((time.perf_counter() - t) * 1e3, 1)

        def run(W, want):
            work = os.path.join(root, f"w{W}")
            # hard links: the library replaces a directory's files by rename, never writes into them, so every
            # configuration starts from the pristine bytes without a copy of the whole directory
            shutil.copytree(pristine, work, copy_function=os.link)
            out = {}
            try:
                if W == 1:
                    ix, ms = timed(lambda: npb.MmapIndex.load(work))
                    out["reload_ms"] = ms
                else:
                    b = npb.shard_bounds(work, W)
                    per = []
                    for r in range(W):
                        h, ms = timed(lambda: npb.MmapIndex.load_range(work, int(b[r]), int(b[r + 1])))
                        h.close()
                        torch.cuda.empty_cache()
                        per.append(ms)
                    out["reload_ms"] = dict(sum=round(sum(per), 1), slowest_rank=max(per))
                    ix = npb.ShardGroup([npb.MmapIndex.load_shard(work, r, W) for r in range(W)])
                ops = [("delete", lambda: ix.delete(del1)),
                       ("append_encoded", lambda: ix.append_encoded(codes, res, dl)),
                       ("delete_dir", lambda: ix.delete(del2, index_dir=work)),
                       ("append_dir", lambda: ix.append(emb, codec, index_dir=work))]
                results = []
                for name, op in ops:
                    _, ms = timed(op)
                    got = [(r.passage_ids.tolist(), r.scores.tobytes()) for r in ix.search_batch(qs, p)]
                    results.append(got)
                    out[name] = dict(ms=ms)
                    if want is not None:
                        k = len(results) - 1
                        out[name].update(parity=bool(got == want[k]),
                                         queries_differing=sum(g != w for g, w in zip(got, want[k])))
                ix.close()
                torch.cuda.empty_cache()
                return out, results
            finally:
                shutil.rmtree(work, ignore_errors=True)

        single, want = run(1, None)
        groups = {f"W{W}": run(W, want)[0] for W in (int(w) for w in a.widths.split(","))}
        codec.close()
    finally:
        shutil.rmtree(root, ignore_errors=True)
    info = bench.gpu_info(0)
    name = torch.cuda.get_device_name(0)                 # also when nvidia-smi reports no power limit
    print(json.dumps({
        "workload": f"{D} docs x {T} tok, dim {args.dim}, nbits {args.nbits}, K 2^{args.log2k}; delete {a.n_delete} "
                    f"scattered docs, append {a.n_append} docs x {T} tok",
        "page_cache": "warm: the directory was written by this run", "single": single, **groups,
        "gpu": name, "power_limit_w": info["power_limit_w"]}))


if __name__ == "__main__":
    main()
