"""N-rank NCCL check of per-query subsets on the doc-sharded CUDA path (run under torchrun on N GPUs of one box):
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 \
        --master-port 29512 tests/gpu_sharded_subsets_check.py
The NCCL twin of tests/test_gpu_subsets.py's in-process groups: every rank searches the same queries with a subset
per query (and pb_search_batch with one subset) on both variants; every rank's result must be bit-identical to the
CPU oracle searching the UNSHARDED index.  Ranks then pass different subsets and must all refuse with
PB_ERR_INVALID, after which the deployment still searches correctly."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    import torch
    import torch.distributed as dist
    import next_plaid_b200 as npb
    from oracle import oracle
    import sharded_protocol as sp
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    docs = oracle.synthetic_corpus(4000, 40, dim=128, seed=31, ragged=True)
    ix = oracle.create_index(docs, nbits=4, seed=5, num_partitions=512)
    qs = [oracle.synthetic_queries(docs, 1, nq=n, seed=70 + i)[0][0] for i, n in enumerate((1, 32, 33, 64, 65, 32) * 3)]
    shard, base = sp.make_shard(oracle, ix, rank, world)
    gpu = npb.MmapIndex.from_arrays(shard.centroids, shard.bucket_weights, shard.codes, shard.residuals,
                                    shard.doc_lengths, shard.ivf, shard.ivf_lengths, shard.nbits, device=local,
                                    doc_id_base=base)
    uid = [npb.comm_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(uid, src=0)
    gpu.comm_init(uid[0], rank, world)
    D = ix.num_documents
    rng = np.random.default_rng(1)
    kinds = [None, [], [5, 5, 17, 10 ** 7, -3], sorted(rng.choice(D, 40, replace=False).tolist()),
             list(range(0, D, 2)), list(range(1, D, 20)), list(range(D)), [D, -1], list(range(0, D // world))]
    subs = (kinds * 2)[:len(qs)]
    bad = 0
    for cbs in (100_000, 128):
        kw = dict(top_k=10, n_ivf_probe=8, n_full_scores=256, centroid_batch_size=cbs)
        pg, po = npb.SearchParameters(**kw), oracle.SearchParameters(**kw)
        calls = [("per-query", subs, gpu.search_batch_subsets(qs, pg, subs))]
        for s in (list(range(0, D, 3)), list(range(1, D, 20))):
            calls.append(("single", [s] * len(qs), gpu.search_batch(qs, pg, subset=s)))
        for what, ss, res in calls:
            for q, s, r in zip(qs, ss, res):
                w = oracle.search_one(ix, q, po, subset=s)
                if r.passage_ids.tolist() != w.passage_ids.tolist() or not np.array_equal(r.scores, w.scores):
                    print(f"rank {rank}: {what} mismatch cbs={cbs}", file=sys.stderr)
                    bad += 1
    pg = npb.SearchParameters(top_k=10, n_ivf_probe=8, n_full_scores=256)
    try:
        gpu.search_batch_subsets(qs, pg, [list(range(rank, D, 3))] + subs[1:])
        print(f"rank {rank}: different subsets were not refused", file=sys.stderr)
        bad += 1
    except npb.PlaidError as e:
        if e.status != 1:
            print(f"rank {rank}: different subsets gave status {e.status}", file=sys.stderr)
            bad += 1
    po = oracle.SearchParameters(top_k=10, n_ivf_probe=8, n_full_scores=256)
    for q, s, r in zip(qs, subs, gpu.search_batch_subsets(qs, pg, subs)):
        w = oracle.search_one(ix, q, po, subset=s)
        if r.passage_ids.tolist() != w.passage_ids.tolist() or not np.array_equal(r.scores, w.scores):
            print(f"rank {rank}: mismatch after the refusal", file=sys.stderr)
            bad += 1
    t = torch.tensor([bad], device="cuda")
    dist.all_reduce(t)
    if rank == 0:
        print(f"sharded subsets check world={world}: {'OK' if t.item() == 0 else 'MISMATCH ' + str(t.item())}")
    gpu.close()
    dist.destroy_process_group()
    sys.exit(0 if t.item() == 0 else 1)


if __name__ == "__main__":
    main()
