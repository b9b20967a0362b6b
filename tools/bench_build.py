"""Index-build benchmark (SURVEY 8 a12 / 8e build path, BASELINE config D shape): data-parallel k-means of K = 2^log2k
centroids over `--kmeans-points` sample vectors, then nearest-centroid + 4-bit residual encode of `--tokens` token
vectors, each rank on its own shard.

    python tools/bench_build.py --tokens 4194304 --kmeans-points 1048576                          # one GPU
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 --master-port 29544 \
        tools/bench_build.py --tokens 33554432 --kmeans-points 8388608                               # NCCL, 8 ranks

--tokens / --kmeans-points are whole-job totals, split evenly over the ranks.  Rank 0 prints one JSON line."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def clustered(rng, centers, n, dim):
    x = centers[rng.integers(0, len(centers), n)] + 0.35 * rng.standard_normal((n, dim), dtype=np.float32) / np.sqrt(dim)
    return x / np.linalg.norm(x, axis=1, keepdims=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", type=int, default=1 << 20)
    ap.add_argument("--kmeans-points", type=int, default=0, help="0 = skip k-means and encode against random unit centroids")
    ap.add_argument("--kmeans-iters", type=int, default=4)
    ap.add_argument("--log2k", type=int, default=18)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--nbits", type=int, default=4)
    ap.add_argument("--check", type=int, default=2048, help="tokens verified against the CPU oracle (rank 0)")
    a = ap.parse_args()
    import next_plaid_b200 as npb
    rank, world, local = (int(os.environ.get(k, d)) for k, d in (("RANK", 0), ("WORLD_SIZE", 1), ("LOCAL_RANK", 0)))
    dist = None
    if world > 1:
        import torch
        import torch.distributed as dist
        torch.cuda.set_device(local)
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    K = 1 << a.log2k
    grng = np.random.default_rng(42)                      # shared: latent topic centres
    centers = grng.standard_normal((4 * 4096, a.dim), dtype=np.float32)
    centers /= np.linalg.norm(centers, axis=1, keepdims=True)
    rng = np.random.default_rng(1000 + rank)              # per rank: its shard
    out = {"n_gpus": world, "num_centroids": K, "dim": a.dim, "nbits": a.nbits}
    if a.kmeans_points > 0:
        pts = clustered(rng, centers, a.kmeans_points // world, a.dim)
        nccl = None
        if world > 1:
            uid = [npb.comm_unique_id() if rank == 0 else None]
            dist.broadcast_object_list(uid, src=0)
            nccl = (uid[0], rank, world)
            dist.barrier()
        t0 = time.perf_counter()
        cent = npb.kmeans_fit_dp([pts], K, niters=a.kmeans_iters, seed=42, device=local, nccl=nccl) if world > 1 else \
            npb.kmeans_fit(pts, K, niters=a.kmeans_iters, seed=42, device=local)
        dt = time.perf_counter() - t0
        out["kmeans"] = {"points": a.kmeans_points, "iters": a.kmeans_iters, "seconds": dt,
                         "points_per_s_per_iter": a.kmeans_points * a.kmeans_iters / dt,
                         "fp32_tflops_equiv": 2.0 * a.kmeans_points * K * a.dim * a.kmeans_iters / dt / 1e12,
                         "allreduce_bytes_per_iter": K * (a.dim + 1) * 4 if world > 1 else 0}
    else:
        cent = grng.standard_normal((K, a.dim), dtype=np.float32)
        cent /= np.linalg.norm(cent, axis=1, keepdims=True)
    n_local = a.tokens // world
    emb = clustered(rng, centers, n_local, a.dim)
    codec = npb.ResidualCodec(a.nbits, cent, device=local)
    codec.train(emb[:min(n_local, 50_000)])       # bucket cutoffs from held-out residuals (index.rs:228-287)
    codec.encode_chunk(emb[:4096])                # warm-up (module load, allocations)
    if world > 1:
        dist.barrier()
    t0 = time.perf_counter()
    codes, packed = codec.encode_chunk(emb)
    dt = time.perf_counter() - t0
    if world > 1:
        import torch
        t = torch.tensor([dt], device="cuda", dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        dt = float(t[0])
    st = codec.last_assign_stats()
    out["encode"] = {"tokens": a.tokens, "seconds_e2e_host_buffers": dt, "tokens_per_s_e2e": a.tokens / dt,
                     "tflops_equiv_e2e": 2.0 * a.tokens * K * a.dim / dt / 1e12, "assign_stats_rank0": st}
    if a.check and rank == 0:
        from oracle import oracle
        idx = rng.choice(n_local, min(a.check, n_local), replace=False)
        want = oracle.compress_into_codes(emb[idx], cent)
        out["oracle_check"] = {"tokens": int(len(idx)), "codes_identical": bool(np.array_equal(want, codes[idx]))}
    if rank == 0:
        print(json.dumps(out))
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
