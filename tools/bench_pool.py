"""Token pooling on the device (pb_pool_embeddings, DESIGN.md §4p) at the size a build pipeline pools: 100 k documents of
300 tokens, dim 128, pool_factor 2 (colgrep's default), from oracle.synthetic_corpus.  Prints one JSON line:

  docs/s host -> host (input and output in host memory) and device -> device (CUDA tensors), best of --reps;
  device ms per phase of the last device call (CUDA events: distances, chain, cut + means);
  the FP64 rate the distance phase achieved, from n(n-1)/2 * dim f64 multiply-adds per document of n clustered tokens,
  beside the H100 SXM data sheet's 34 TFLOP/s FP64 vector figure (a bound, not a measurement);
  the CPU restatement (tests/pool_oracle.c, OpenMP over every host thread) on a --sample of the documents, and the
  device's parity with it on that sample, bit for bit;
  the card's name and power limit.

  python tools/bench_pool.py [--docs 100000] [--tokens 300] [--sample 2000] [--reps 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

FP64_DATASHEET_TFLOPS = 34.0   # H100 SXM, FP64 vector (not tensor core)


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=100_000)
    ap.add_argument("--tokens", type=int, default=300)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--pool-factor", type=int, default=2)
    ap.add_argument("--sample", type=int, default=2000)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()

    import torch
    import next_plaid_b200 as npb
    import pool_oracle
    from oracle import oracle
    npb.build_library()
    if npb.device_count() < 1:
        raise SystemExit("bench_pool needs an H100; the library has no CPU fallback")

    docs = oracle.synthetic_corpus(a.docs, a.tokens, dim=a.dim, seed=5)
    pf = a.pool_factor
    res = {"docs": a.docs, "tokens": a.tokens, "dim": a.dim, "pool_factor": pf, "card": card()}

    npb.pool_document_embeddings(docs[:256], pf)                     # warm-up: module load, shared-memory opt-ins
    best = float("inf")
    for _ in range(a.reps):
        t0 = time.perf_counter()
        npb.pool_document_embeddings(docs, pf)
        best = min(best, time.perf_counter() - t0)
    res["host_to_host_docs_per_s"] = a.docs / best

    L = npb.load_library()
    import ctypes as C
    d_in = torch.from_numpy(np.concatenate(docs, 0)).cuda()
    lens = np.array([d.shape[0] for d in docs], np.int64)
    olens = np.array([npb.pooled_doc_length(int(n), pf) for n in lens], np.int64)
    d_out = torch.empty((int(olens.sum()), a.dim), dtype=torch.float32, device="cuda")
    got = np.zeros(len(docs), np.int64)
    torch.cuda.synchronize()
    best = float("inf")
    for _ in range(a.reps):
        t0 = time.perf_counter()
        st = L.pb_pool_embeddings(0, d_in.data_ptr(), lens.ctypes.data_as(C.c_void_p), len(docs), a.dim, pf, 1,
                                  d_out.data_ptr(), got.ctypes.data_as(C.c_void_p))
        best = min(best, time.perf_counter() - t0)
        assert st == 0, L.pb_last_error()
    res["device_to_device_docs_per_s"] = a.docs / best
    ms = npb.last_pool_ms()
    res["phase_ms"] = ms
    t = lens - 1
    pooled = olens < lens
    dfma = float(np.sum((t * (t - 1) // 2)[pooled])) * a.dim
    res["distance_fp64_tflops"] = 2 * dfma / (ms["distances"] * 1e-3) / 1e12
    res["fp64_datasheet_tflops_bound"] = FP64_DATASHEET_TFLOPS

    sample = docs[:a.sample]
    t0 = time.perf_counter()
    want = pool_oracle.pool_embeddings(sample, pf)
    cpu_s = time.perf_counter() - t0
    res["cpu_oracle_docs_per_s"] = len(sample) / cpu_s
    res["cpu_threads"] = os.cpu_count()
    offs = np.concatenate([[0], np.cumsum(got)])
    dev = d_out[:int(offs[len(sample)])].cpu().numpy()
    ok = all(np.array_equal(dev[offs[i]:offs[i + 1]].view(np.uint32), w.view(np.uint32)) and got[i] == len(w)
             for i, w in enumerate(want))
    res["parity_sample_docs"] = len(sample)
    res["parity_bit_exact"] = bool(ok)
    print(json.dumps(res))
    if not ok:
        raise SystemExit(1)


if __name__ == "__main__":
    main()
