"""Incremental append on the config-B corpus (1M docs x 300 tokens x 128-d, 4-bit residuals, K = 2^18, built on the
device exactly as bench.py builds it): pb_index_append of 10 000 new 300-token docs, with and without
pb_index_reserve, against pb_index_close + pb_index_open of the concatenated device arrays.  Checks that the appended
handle and the fresh open return identical searches on 64 queries and prints one JSON line.

  encode_ms  pb_index_append (device encode from f32 embeddings) minus pb_index_append_encoded of the same codes
  merge_ms   device time of the inverted-file merge kernels (k_ivf_offsets, k_ivf_merge_old, k_ivf_merge_new), from a
             separate torch.profiler run
  rest_ms    append_ms - encode_ms - merge_ms (capacity, narrowing, distinct codes, norms, pair sort, host syncs)

Run from the repository root on an H100: python tools/bench_append.py [--docs-total 1000000] [--new-docs 10000]"""
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
    ap.add_argument("--new-docs", type=int, default=10_000)
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
    per_rank, chunk, n_chunks = bench.chunk_layout(args, 1)
    # the new docs: the generator's chunk after the last one, decoded to f32 embeddings c + w (which encode back to
    # those codes unless a token sits on a tie)
    new_codes, new_res = bench.gen_chunk(args, G, n_chunks, a.new_docs, dev)
    new_dl = torch.full((a.new_docs,), T, dtype=torch.int64, device=dev)
    shifts = torch.tensor([8 - nbits * (j + 1) for j in range(8 // nbits)], device=dev, dtype=torch.int32)
    w = G["bucket_weights"]
    w_rev = torch.stack([w[bench._bitrev(f, nbits)] for f in range(1 << nbits)])
    fields = ((new_res.to(torch.int32).unsqueeze(-1) >> shifts) & ((1 << nbits) - 1)).reshape(-1, dim)
    emb = (G["centroids"][new_codes] + w_rev[fields.to(torch.int64)]).contiguous()
    del fields
    # bucket cutoffs of the generator's weights: quantiles i / 2^nbits of N(0, res_sigma^2)
    nb = 1 << nbits
    cut = (args.res_sigma * torch.special.ndtri(torch.arange(1, nb, dtype=torch.float64) / nb)).to(torch.float32).numpy()
    codec = npb.ResidualCodec(nbits, G["centroids"].cpu().numpy(), cut)
    qs = bench.make_queries(args, G, dev, a.queries, seed=11)
    p = npb.SearchParameters(top_k=100, n_ivf_probe=8, n_full_scores=4096)

    def open_base():
        sh = bench.build_shard(args, G, 0, 1, dev)
        ix = npb.MmapIndex.from_device_pointers(dim, nbits, K, sh["D"], sh["N"], G["centroids"].data_ptr(),
                                                G["bucket_weights"].data_ptr(), sh["codes"].data_ptr(),
                                                sh["residuals"].data_ptr(), sh["doc_lengths"].data_ptr(), None, None)
        del sh
        torch.cuda.empty_cache()
        return ix

    def timed(f):
        torch.cuda.synchronize(dev)
        t0 = time.perf_counter()
        r = f()
        torch.cuda.synchronize(dev)
        return (time.perf_counter() - t0) * 1e3, r

    from next_plaid_b200.index import _check
    L = npb.load_library()
    import ctypes as C
    n_new_tok = a.new_docs * T

    def append_codec(ix):
        first = C.c_int64()
        _check(L.pb_index_append(ix._h, codec._h, emb.data_ptr(), new_dl.data_ptr(), a.new_docs, 1, None, 0,
                                           C.byref(first)))

    def append_encoded(ix):
        first = C.c_int64()
        _check(L.pb_index_append_encoded(ix._h, new_codes.data_ptr(), new_res.data_ptr(), new_dl.data_ptr(),
                                                   a.new_docs, 1, C.byref(first)))

    def search(ix):
        return [(r.passage_ids.tolist(), r.scores.tobytes()) for r in ix.search_batch(qs, p)]

    out = {}
    results = {}
    # warm-up: one append of each kind on a small index opened from the same generator (modules, CUB, cuBLAS-free)
    small = npb.MmapIndex.from_device_pointers(dim, nbits, K, a.new_docs, n_new_tok, G["centroids"].data_ptr(),
                                               G["bucket_weights"].data_ptr(), new_codes.data_ptr(), new_res.data_ptr(),
                                               new_dl.data_ptr(), None, None)
    append_codec(small)
    append_encoded(small)
    small.close()
    for mode in ("growth", "reserve"):
        runs = []
        for rep in range(a.repeats):
            for kind, fn in (("codec", append_codec), ("encoded", append_encoded)):
                ix = open_base()
                if mode == "reserve":
                    ix.reserve(per_rank + a.new_docs, (per_rank + a.new_docs) * T)
                ms, _ = timed(lambda: fn(ix))
                runs.append((kind, ms))
                if kind == "encoded" and rep == 0:
                    results[mode] = search(ix)
                ix.close()
                torch.cuda.empty_cache()
        out[mode] = {"append_ms": float(np.median([m for k, m in runs if k == "codec"])),
                     "append_encoded_ms": float(np.median([m for k, m in runs if k == "encoded"]))}
        out[mode]["encode_ms"] = out[mode]["append_ms"] - out[mode]["append_encoded_ms"]
    # merge kernels' device time, in a profiled run of its own
    ix = open_base()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        append_encoded(ix)
        torch.cuda.synchronize(dev)
    merge_us = sum(e.device_time_total for e in prof.key_averages()
                   if any(k in e.key for k in ("k_ivf_merge_old", "k_ivf_merge_new", "k_ivf_offsets")))
    ix.close()
    torch.cuda.empty_cache()
    for mode in out:
        out[mode]["merge_ms"] = merge_us / 1e3
        out[mode]["rest_ms"] = out[mode]["append_ms"] - out[mode]["encode_ms"] - out[mode]["merge_ms"]
        out[mode]["tokens_per_s"] = n_new_tok / (out[mode]["append_ms"] / 1e3)
    # close + open of the concatenated device arrays
    reopen, fresh_res = [], None
    for rep in range(a.repeats):
        sh = bench.build_shard(args, G, 0, 1, dev)
        codes, res = torch.cat([sh["codes"], new_codes]), torch.cat([sh["residuals"], new_res])
        dl = torch.cat([sh["doc_lengths"], new_dl])
        del sh
        torch.cuda.empty_cache()
        ms_open, fresh = timed(lambda: npb.MmapIndex.from_device_pointers(
            dim, nbits, K, per_rank + a.new_docs, (per_rank + a.new_docs) * T, G["centroids"].data_ptr(),
            G["bucket_weights"].data_ptr(), codes.data_ptr(), res.data_ptr(), dl.data_ptr(), None, None))
        del codes, res, dl
        torch.cuda.empty_cache()
        if fresh_res is None:
            fresh_res = search(fresh)
        ms_close, _ = timed(fresh.close)
        reopen.append(ms_open + ms_close)
    info = bench.gpu_info(0)
    print(json.dumps({
        "workload": f"{per_rank} docs x {T} tok + append of {a.new_docs} docs, dim {dim}, nbits {nbits}, K 2^{args.log2k}",
        "append_growth": out["growth"], "append_reserved": out["reserve"],
        "reopen_ms": float(np.median(reopen)),
        "parity": bool(results["growth"] == fresh_res and results["reserve"] == fresh_res),
        "gpu": info["name"], "power_limit_w": info["power_limit_w"]}))


if __name__ == "__main__":
    main()
