"""N-rank NCCL check of pb_index_rebalance_sharded (run under torchrun on N >= 2 GPUs of one box; NCCL does not put two
ranks on one device):
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 \\
        --master-port 29515 tests/gpu_sharded_rebalance_check.py
Every rank opens its shard of one index, joins the communicator and runs the same sequence: skewed bounds to balanced,
explicit bounds that move documents across several ranks and empty a rank, appends to the last rank followed by a
rebalance, and a delete followed by another.  After each step every rank's handle must equal a fresh open of its range
(document and token counts, inverted file with its base, decompressed rows), and the group's searches must equal, bit
for bit, the CPU oracle.  Rejected calls (bad bounds, ranks passing different bounds) must fail on every rank with the
same status and change nothing.  Exit status 0 on every rank when all checks hold."""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

NBITS, K, DIM = 2, 256, 128


def main():
    import torch
    import torch.distributed as dist
    import next_plaid_b200 as npb
    from oracle import oracle
    import sharded_update as su
    from ivf_delete import delete_ivf
    from ivf_merge import merge_ivf
    from ivf_slice import ivf_slice, shard_bounds
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    L = npb.load_library()
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    bad = []

    docs = oracle.synthetic_corpus(2400, 40, dim=DIM, seed=71, ragged=True)
    flat = np.concatenate(docs, 0)
    cent = flat[np.random.default_rng(3).choice(len(flat), K, replace=False)].copy()
    art = oracle.prepare_codec_artifacts(docs, cent, NBITS, 3)
    codes_all, packed_all, dl_all = oracle.encode_documents(docs, art, NBITS)
    dl_all = np.asarray(dl_all, np.int64)
    off_all = np.concatenate([[0], np.cumsum(dl_all)]).astype(np.int64)
    qs, _ = oracle.synthetic_queries(docs, 6, nq=32, seed=12)
    D = 1800
    st = dict(codes=codes_all[:off_all[D]], packed=packed_all[:off_all[D]], dl=dl_all[:D])
    st["ivf"], st["lens"] = oracle.build_ivf(st["codes"], st["dl"], K)
    bounds = np.array([0] + [5 * r for r in range(1, world)] + [D], np.int64)    # almost everything on the last rank

    def open_range(b, e):
        off = np.concatenate([[0], np.cumsum(st["dl"])]).astype(np.int64)
        iv, ln = ivf_slice(st["ivf"], st["lens"], b, e)
        return npb.MmapIndex.from_arrays(art.centroids, art.bucket_weights, st["codes"][off[b]:off[e]],
                                         st["packed"][off[b]:off[e]], st["dl"][b:e], iv, ln, NBITS, device=local,
                                         doc_id_base=b)

    def check(h, what):
        b, e = int(bounds[rank]), int(bounds[rank + 1])
        fresh = open_range(b, e)
        x, y = h.export_ivf(), fresh.export_ivf()
        same = (h.num_documents(), h.num_embeddings()) == (fresh.num_documents(), fresh.num_embeddings()) and \
            np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1])
        if same and e > b:
            ids = sorted({b, e - 1, (b + e) // 2})
            same = all(np.array_equal(u, v) for u, v in zip(h.decompress_documents(ids), fresh.decompress_documents(ids)))
        if not same:
            bad.append(f"rank {rank}: handle differs from a fresh open after {what}")
        fresh.close()
        ix = oracle.Index(art.centroids, art.bucket_weights, art.bucket_cutoffs, st["codes"], st["packed"], st["dl"],
                          st["ivf"], st["lens"], NBITS)
        for cbs in (100_000, 100):
            pg = npb.SearchParameters(top_k=10, n_ivf_probe=8, n_full_scores=256, centroid_batch_size=cbs)
            po = oracle.SearchParameters(top_k=10, n_ivf_probe=8, n_full_scores=256, centroid_batch_size=cbs)
            for q, r in zip(qs, h.search_batch(qs, pg)):
                w = oracle.search_one(ix, q, po)
                if r.passage_ids.tolist() != w.passage_ids.tolist() or not np.array_equal(r.scores, w.scores):
                    bad.append(f"rank {rank}: search differs from the oracle after {what} (cbs={cbs})")
                    break

    def rebalance(h, want, what):
        nonlocal bounds
        got = h.rebalance_sharded(want)
        expect = shard_bounds(st["dl"], world) if want is None else np.asarray(want, np.int64)
        if not np.array_equal(got, expect):
            bad.append(f"rank {rank}: {what} applied {got.tolist()}, expected {expect.tolist()}")
        bounds = got
        check(h, what)

    h = open_range(int(bounds[rank]), int(bounds[rank + 1]))
    uid = [npb.comm_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(uid, src=0)
    h.comm_init(uid[0], rank, world)
    check(h, "open")
    rebalance(h, None, "skewed to balanced")
    rebalance(h, [0] + [1700] * (world - 1) + [D], "the last rank to rank 0")
    rebalance(h, [0] + [0] * (world - 1) + [D], "everything on the last rank")
    rebalance(h, None, "back to balanced")

    # appends to the last rank, then a rebalance; a delete, then another
    nxt = D
    for m in (150, 100):
        t0, t1 = int(off_all[nxt]), int(off_all[nxt + m])
        first = C.c_int64()
        last = rank == world - 1
        dl = np.ascontiguousarray(dl_all[nxt:nxt + m])
        c_, p_ = np.ascontiguousarray(codes_all[t0:t1]), np.ascontiguousarray(packed_all[t0:t1])
        npb.index._check(L.pb_index_append_encoded_sharded(h._h, npb.index._ptr(c_) if last else None,
                                                           npb.index._ptr(p_) if last else None,
                                                           npb.index._ptr(dl), m, 0, C.byref(first)))
        st["ivf"], st["lens"] = merge_ivf(st["ivf"], st["lens"], codes_all[t0:t1], dl, len(st["dl"]), K)
        st["codes"] = np.concatenate([st["codes"], codes_all[t0:t1]])
        st["packed"] = np.concatenate([st["packed"], packed_all[t0:t1]])
        st["dl"] = np.concatenate([st["dl"], dl])
        bounds = bounds.copy()
        bounds[-1] += m
        nxt += m
    check(h, "appends")
    rebalance(h, None, "rebalance after appends")
    ids = np.random.default_rng(5).choice(len(st["dl"]), 200, replace=False).astype(np.int64)
    cnt = C.c_int64()
    npb.index._check(L.pb_index_delete_sharded(h._h, npb.index._ptr(ids), len(ids), None, C.byref(cnt)))
    gone = su.deleted_set(ids, len(st["dl"]))
    keep = ~np.isin(np.arange(len(st["dl"])), gone)
    tok = np.repeat(keep, st["dl"])
    st["ivf"], st["lens"] = delete_ivf(st["ivf"], st["lens"], gone, len(st["dl"]))
    st["codes"], st["packed"], st["dl"] = st["codes"][tok], st["packed"][tok], st["dl"][keep]
    bounds = su.delete_bounds(bounds, ids)
    check(h, "delete")
    rebalance(h, None, "rebalance after the delete")

    # rejected calls: every rank fails with PB_ERR_INVALID and nothing changes
    Dt = len(st["dl"])
    before = (h.num_documents(), h.export_ivf()[0].tobytes())
    for name, arg in (("bad bounds[0]", [1] + list(bounds[1:])), ("bad bounds[W]", list(bounds[:-1]) + [Dt + 1]),
                      ("ranks disagree", list(bounds) if rank else [0] * world + [Dt])):
        arr = np.ascontiguousarray(arg, np.int64)
        s = L.pb_index_rebalance_sharded(h._h, npb.index._ptr(arr), None)
        if s != 1 or (h.num_documents(), h.export_ivf()[0].tobytes()) != before:
            bad.append(f"rank {rank}: {name} gave status {s} or changed the handle")
    h.close()

    allbad = [None] * world
    dist.all_gather_object(allbad, bad)
    dist.destroy_process_group()
    if any(allbad):
        for x in allbad:
            for line in x or []:
                print(line, file=sys.stderr)
        sys.exit(1)
    if rank == 0:
        print(f"sharded rebalance check ok: world {world}")


if __name__ == "__main__":
    main()
