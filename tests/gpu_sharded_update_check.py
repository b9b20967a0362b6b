"""N-rank NCCL check of appends and deletes on a doc-sharded deployment (run under torchrun on N >= 2 GPUs of one box;
NCCL does not put two ranks on one device):
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 \\
        --master-port 29513 tests/gpu_sharded_update_check.py
Every rank opens its shard of one index, joins the communicator and runs the same sequence of
pb_index_delete_sharded / pb_index_append_encoded_sharded / pb_index_append_sharded calls.  After each one, every
rank's handle must equal a fresh open of its expected range (document and token counts, inverted file with its new
base), and the group's searches must equal, bit for bit, the CPU oracle on the changed index.  A rejected call (ranks
passing different ids) must fail on every rank and change nothing.  Rank 0 also writes an index directory, changes
it through a group of load_shard handles and checks it against the same changes made through one pb_index_load
handle on a copy, file for file.  Exit status 0 on every rank when all checks hold."""
import ctypes as C
import filecmp
import os
import shutil
import sys
import tempfile

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
    from ivf_slice import ivf_slice
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    L = npb.load_library()
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    bad = []

    # one index as arrays, every rank holding the same copy; rank r opens docs [bounds[r], bounds[r + 1])
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
    bounds = np.array([r * D // world for r in range(world)] + [D], np.int64)

    def open_range(b, e):
        off = np.concatenate([[0], np.cumsum(st["dl"])]).astype(np.int64)
        iv, ln = ivf_slice(st["ivf"], st["lens"], b, e)
        return npb.MmapIndex.from_arrays(art.centroids, art.bucket_weights, st["codes"][off[b]:off[e]],
                                         st["packed"][off[b]:off[e]], st["dl"][b:e], iv, ln, NBITS, device=local,
                                         doc_id_base=b)

    def join(h):
        uid = [npb.comm_unique_id() if rank == 0 else None]
        dist.broadcast_object_list(uid, src=0)
        h.comm_init(uid[0], rank, world)

    def check(h, what):
        fresh = open_range(int(bounds[rank]), int(bounds[rank + 1]))
        a, b = h.export_ivf(), fresh.export_ivf()
        if (h.num_documents(), h.num_embeddings()) != (fresh.num_documents(), fresh.num_embeddings()) or \
                not (np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])):
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

    h = open_range(int(bounds[rank]), int(bounds[rank + 1]))
    join(h)
    rng = np.random.default_rng(5)
    nxt = D
    for step in range(3):
        # delete: global ids, the same list on every rank
        ids = np.concatenate([rng.choice(len(st["dl"]), 80, replace=False), [-1, 10 ** 6]])
        cnt = C.c_int64()
        arr = np.ascontiguousarray(ids, np.int64)
        npb.index._check(L.pb_index_delete_sharded(h._h, npb.index._ptr(arr), len(arr), None, C.byref(cnt)))
        gone = su.deleted_set(ids, len(st["dl"]))
        if cnt.value != len(gone):
            bad.append(f"rank {rank}: delete reported {cnt.value}, expected {len(gone)}")
        keep = ~np.isin(np.arange(len(st["dl"])), gone)
        tok = np.repeat(keep, st["dl"])
        st["ivf"], st["lens"] = delete_ivf(st["ivf"], st["lens"], gone, len(st["dl"]))
        st["codes"], st["packed"], st["dl"] = st["codes"][tok], st["packed"][tok], st["dl"][keep]
        bounds = su.delete_bounds(bounds, ids)
        check(h, f"delete {step}")
        # append: encoded on even steps, on the device with the codec on odd ones; documents go to the last rank
        m = 40
        t0, t1 = int(off_all[nxt]), int(off_all[nxt + m])
        first = C.c_int64()
        last = rank == world - 1
        dl = np.ascontiguousarray(dl_all[nxt:nxt + m])
        if step % 2 == 0:
            c_, p_ = np.ascontiguousarray(codes_all[t0:t1]), np.ascontiguousarray(packed_all[t0:t1])
            npb.index._check(L.pb_index_append_encoded_sharded(h._h, npb.index._ptr(c_) if last else None,
                                                               npb.index._ptr(p_) if last else None,
                                                               npb.index._ptr(dl), m, 0, C.byref(first)))
        else:
            codec = npb.ResidualCodec(NBITS, art.centroids, art.bucket_cutoffs, device=local) if last else None
            x = np.ascontiguousarray(np.concatenate(docs[nxt:nxt + m], 0), np.float32)
            npb.index._check(L.pb_index_append_sharded(h._h, codec._h if last else None,
                                                       npb.index._ptr(x) if last else None, npb.index._ptr(dl), m, 0,
                                                       None, 0, C.byref(first)))
            if codec:
                codec.close()
        if first.value != len(st["dl"]):
            bad.append(f"rank {rank}: append returned first id {first.value}, expected {len(st['dl'])}")
        st["ivf"], st["lens"] = merge_ivf(st["ivf"], st["lens"], codes_all[t0:t1], dl, len(st["dl"]), K)
        st["codes"] = np.concatenate([st["codes"], codes_all[t0:t1]])
        st["packed"] = np.concatenate([st["packed"], packed_all[t0:t1]])
        st["dl"] = np.concatenate([st["dl"], dl])
        bounds = bounds.copy()
        bounds[-1] += m
        nxt += m
        check(h, f"append {step}")

    # a rejected call: rank 0 passes other ids than the rest; every rank fails, nothing changes
    before = (h.num_documents(), h.export_ivf()[0].tobytes())
    arr = np.array([1, 2] if rank == 0 else [1, 3], np.int64)
    s = L.pb_index_delete_sharded(h._h, npb.index._ptr(arr), len(arr), None, C.byref(cnt))
    if s != 1 or (h.num_documents(), h.export_ivf()[0].tobytes()) != before:
        bad.append(f"rank {rank}: mismatched ids gave status {s} or changed the handle")
    h.close()

    # the directory: written by rank 0, changed by a load_shard group; a copy changed by one handle on rank 0
    path = [tempfile.mkdtemp(prefix="pb_sharded_update_check_") if rank == 0 else None]
    dist.broadcast_object_list(path, src=0)
    a = os.path.join(path[0], "a")
    b = os.path.join(path[0], "b")
    if rank == 0:
        npb.create_index(docs[:1800], a, nbits=NBITS, num_partitions=K, batch_size=700, seed=7, device=local).close()
        shutil.copytree(a, b)
    dist.barrier()
    g = npb.MmapIndex.load_shard(a, rank, world, device=local)
    join(g)
    ids = np.random.default_rng(8).choice(1800, 150, replace=False).astype(np.int64)
    cnt = C.c_int64()
    npb.index._check(L.pb_index_delete_sharded(g._h, npb.index._ptr(ids), len(ids), os.fsencode(a), C.byref(cnt)))
    g.close()
    dist.barrier()
    if rank == 0:
        single = npb.MmapIndex.load(b, device=local)
        single.delete(ids, index_dir=b)
        single.close()
        for f in sorted(set(os.listdir(a)) | set(os.listdir(b))):
            if not (os.path.exists(os.path.join(a, f)) and os.path.exists(os.path.join(b, f)) and
                    filecmp.cmp(os.path.join(a, f), os.path.join(b, f), shallow=False)):
                bad.append(f"rank 0: directory file {f} differs from the single-handle change")
        shutil.rmtree(path[0], ignore_errors=True)

    allbad = [None] * world
    dist.all_gather_object(allbad, bad)
    dist.destroy_process_group()
    if any(allbad):
        for x in allbad:
            for line in x or []:
                print(line, file=sys.stderr)
        sys.exit(1)
    if rank == 0:
        print(f"sharded update check ok: world {world}")


if __name__ == "__main__":
    main()
