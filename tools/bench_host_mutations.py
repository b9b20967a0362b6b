"""Appends and deletes on a mutable host-tier handle (PB_OPEN_HOST_RESIDUALS | PB_OPEN_HOST_MUTABLE, DESIGN.md 4r) on
the config-B corpus (1M docs x 300 tokens x 128-d, 4-bit residuals, K = 2^18, bench.py's generator), against closing
the handle and opening a host-tier handle on the resulting arrays, which is what such a handle cost before.

One handle goes through, each step timed with a host clock around a call that ends synchronised:
  append_encoded      10 000 docs x 300 tokens, encoded, from device memory (a copy of docs [0, 10 000))
  delete_newest       those 10 000 docs again
  append_codec        10 000 docs x 300 tokens of random unit vectors, encoded on the device with a codec
  delete_newest_2     those again
  reserve             capacity for one more append of 10 000 docs; pinned bytes before and after
  append_codec_reserved   the codec append once more, into the reserved capacity (pinned bytes it added), then
                      delete_newest_3 of those docs
  append_reserved     the encoded append once more, into the reserved capacity (pinned bytes it added)
  delete_scattered    10 000 docs spread over the index (every 101st)
  delete_oldest       the 10 000 oldest docs
Then reopen_s: a host-tier open on the resulting arrays, and `identical`: 64 queries (two batches of 32, top_k 100)
give the same ids and scores on the mutated handle and on that fresh open.

Run from the repository root on an H100: python tools/bench_host_mutations.py [--docs-total 1000000]"""
import argparse
import ctypes
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
    a = ap.parse_args()
    sys.argv = [sys.argv[0], "--docs-total", str(a.docs_total), "--batch", "32"]
    import bench
    import torch
    import next_plaid_b200 as npb
    args = bench.parse_args()
    dev = torch.device("cuda", 0)
    G = bench.corpus_globals(args, dev)
    sh = bench.build_shard(args, G, 0, 1, dev)
    L = npb.load_library()
    from next_plaid_b200.index import _check as check
    n = a.new_docs
    D0 = sh["D"]
    doff = torch.zeros(D0 + 1, dtype=torch.int64, device=dev)
    doff[1:] = torch.cumsum(sh["doc_lengths"], 0)
    t_new = int(doff[n])
    qsets = [bench.make_queries(args, G, dev, 32, seed=500 + s) for s in range(2)]
    p = npb.SearchParameters(top_k=args.top_k, n_ivf_probe=args.n_ivf_probe, n_full_scores=args.n_full_scores,
                             centroid_score_threshold=args.threshold)

    def timed(f):
        torch.cuda.synchronize(dev)
        t = time.perf_counter()
        r = f()
        torch.cuda.synchronize(dev)
        return r, round(time.perf_counter() - t, 3)

    def open_host(codes, res, dl, D, N, mutable):
        return npb.MmapIndex.from_device_pointers(
            args.dim, args.nbits, G["K"], D, N, G["centroids"].data_ptr(), G["bucket_weights"].data_ptr(),
            codes.data_ptr(), res.data_ptr(), dl.data_ptr(), None, None, host_residuals=True, mutable=mutable)

    h, open_s = timed(lambda: open_host(sh["codes"], sh["residuals"], sh["doc_lengths"], D0, sh["N"], True))
    out = dict(open_s=open_s, host_bytes_open=h.memory_usage()["host_bytes"])

    def append_encoded():
        first = ctypes.c_int64()
        check(L.pb_index_append_encoded(h._h, sh["codes"].data_ptr(), sh["residuals"].data_ptr(),
                                             sh["doc_lengths"].data_ptr(), n, 1, ctypes.byref(first)))

    _, out["append_encoded_s"] = timed(append_encoded)
    out["host_bytes_after_append"] = h.memory_usage()["host_bytes"]
    _, out["delete_newest_s"] = timed(lambda: h.delete(list(range(D0, D0 + n))))

    # codec append: random unit vectors, cutoffs halfway between the sorted bucket weights
    ws = np.sort(G["bucket_weights"].float().cpu().numpy())
    codec = npb.ResidualCodec(args.nbits, G["centroids"].float().cpu().numpy(),
                              ((ws[1:] + ws[:-1]) / 2).astype(np.float32))
    x = torch.randn(n * args.doclen, args.dim, device=dev)
    x /= x.norm(dim=1, keepdim=True)
    dl_new = torch.full((n,), args.doclen, dtype=torch.int64, device=dev)

    def append_codec():
        first = ctypes.c_int64()
        check(L.pb_index_append(h._h, codec._h, x.data_ptr(), dl_new.data_ptr(), n, 1, None, 0,
                                     ctypes.byref(first)))

    _, out["append_codec_s"] = timed(append_codec)
    _, out["delete_newest_2_s"] = timed(lambda: h.delete(list(range(D0, D0 + n))))
    before = h.memory_usage()["host_bytes"]
    _, out["reserve_s"] = timed(lambda: h.reserve(D0 + n, sh["N"] + max(t_new, n * args.doclen)))
    out["host_bytes_reserve"] = [before, h.memory_usage()["host_bytes"]]
    _, out["append_codec_reserved_s"] = timed(append_codec)
    out["append_codec_reserved_added_pinned_bytes"] = h.memory_usage()["host_bytes"] - out["host_bytes_reserve"][1]
    _, out["delete_newest_3_s"] = timed(lambda: h.delete(list(range(D0, D0 + n))))
    codec.close()
    del x
    _, out["append_reserved_s"] = timed(append_encoded)
    out["append_reserved_added_pinned_bytes"] = h.memory_usage()["host_bytes"] - out["host_bytes_reserve"][1]
    scattered = list(range(0, D0, max(D0 // n, 1)))[:n]
    _, out["delete_scattered_s"] = timed(lambda: h.delete(scattered))
    _, out["delete_oldest_s"] = timed(lambda: h.delete(list(range(n))))

    # the resulting arrays: docs [0, D0) then a copy of [0, n), minus the scattered ones, minus the n oldest after that
    docs = torch.cat([torch.arange(D0, device=dev), torch.arange(n, device=dev)])
    keep = torch.ones(len(docs), dtype=torch.bool, device=dev)
    keep[torch.tensor(scattered, device=dev)] = False
    docs = docs[keep][n:]
    lens = sh["doc_lengths"][docs]
    tok = torch.repeat_interleave(doff[docs], lens) + (torch.arange(int(lens.sum()), device=dev) -
                                                       torch.repeat_interleave(torch.cumsum(lens, 0) - lens, lens))
    codes, res = sh["codes"][tok], sh["residuals"][tok]
    del tok
    h2, out["reopen_s"] = timed(lambda: open_host(codes, res, lens, len(docs), len(codes), False))
    identical = h.num_documents() == h2.num_documents() and h.num_embeddings() == h2.num_embeddings()
    for qs in qsets:
        a1 = h.search_batch(qs, p)
        a2 = h2.search_batch(qs, p)
        identical &= [(r.passage_ids.tolist(), r.scores.tobytes()) for r in a1] == \
                     [(r.passage_ids.tolist(), r.scores.tobytes()) for r in a2]
    out["identical"] = bool(identical)
    out["host_bytes_end"] = h.memory_usage()["host_bytes"]
    h.close()
    h2.close()
    info = bench.gpu_info(0)
    print(json.dumps({
        "workload": f"{D0} docs x {args.doclen} tok, dim {args.dim}, nbits {args.nbits}, K 2^{args.log2k}; "
                    f"{n} new docs x {args.doclen} tok", **out,
        "gpu": info["name"], "power_limit_w": info["power_limit_w"]}))


if __name__ == "__main__":
    main()
