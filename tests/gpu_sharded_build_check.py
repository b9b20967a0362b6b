"""N-rank NCCL check of pb_create_index_sharded (run under torchrun on N >= 2 GPUs of one box):
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 \
        --master-port 29517 tests/gpu_sharded_build_check.py
Every rank builds its part of one directory over NCCL (k-means off, so the result is pinned); rank 0 then builds the
same split through an in-process group on its own GPU, and the two directories must be identical file for file."""
import os
import shutil
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _files(path):
    return {f: open(os.path.join(path, f), "rb").read() for f in sorted(os.listdir(path))}


def main():
    import torch
    import torch.distributed as dist
    import next_plaid_b200 as npb
    from oracle import oracle
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    docs = oracle.synthetic_corpus(3000, 40, dim=128, seed=17, ragged=True)
    bounds = [len(docs) * r // world + (7 if 0 < r < world else 0) for r in range(world)] + [len(docs)]
    parts = [docs[bounds[r]:bounds[r + 1]] for r in range(world)]
    tmp = [tempfile.mkdtemp(prefix="pb_build_check_") if rank == 0 else None]
    dist.broadcast_object_list(tmp, src=0)
    uid = [npb.comm_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(uid, src=0)
    kw = dict(num_partitions=512, batch_size=400, kmeans_niters=0, seed=3)
    nccl_dir = os.path.join(tmp[0], "nccl")
    h = npb.create_index_sharded([parts[rank]], nccl_dir, device=local, nccl=(uid[0], rank, world), dim=128, **kw)
    ok = h.first_doc_id == bounds[rank]
    h.close()
    dist.barrier()
    if rank == 0:
        group_dir = os.path.join(tmp[0], "group")
        for s in npb.create_index_sharded(parts, group_dir, device=local, **kw):
            s.close()
        ok = ok and _files(nccl_dir) == _files(group_dir)
        shutil.rmtree(tmp[0], ignore_errors=True)
    flag = torch.tensor([int(ok)], device="cuda")
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    if rank == 0:
        print("gpu_sharded_build_check:", "OK" if int(flag[0]) else "MISMATCH")
    dist.destroy_process_group()
    sys.exit(0 if int(flag[0]) else 1)


if __name__ == "__main__":
    main()
