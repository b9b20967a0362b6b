#!/usr/bin/env python
"""profile_step.py -- per-kernel device time of one search step of the flagship workload, from torch.profiler.

    python tools/profile_step.py --out DIR [--steps S] [--warmup W] [bench.py workload options]

Builds bench.py's single-GPU corpus and queries (config B by default: 1M docs x 300 tokens, K = 2^18, 4-bit, batch
32 x 32 query tokens) with bench.py's own generators, runs W untimed steps and then S steps of search_batch_device
under torch.profiler (CUDA activities), and writes DIR/profile_step.json:
  gpu                  name, power limit and max SM clock of the card
  ms_per_step          device time of every kernel per step, and the total of them
  kernel_ms_per_step   per kernel (template arguments kept, parameter lists dropped), largest first
  work_per_step        the library's work counters per step
  a5_bound             k_a5_bound's device time per step and its achieved rate on the bytes the algorithm needs:
                       n_candidate_tokens x 4 (the distinct-code lists, from HBM) plus n_a5_live_rows x 2 QS (the live
                       rows of the 16-bit score table, from L2), QS = query tokens rounded up to 8
  scores_tc            k_scores16_tc's device time per step and its rates on what its shapes make it do, per
                       tensor-core pass (n_k1_tc of them per step; R = B QS rows padded to 128-row groups, T = ceil(K/128)
                       centroid tiles): issued fp16 FLOP 3 x 2 R (128 T) dim (three split products), table bytes
                       written B QS K 2 plus the slab maxima 8 T R 2, and operand bytes read from L2: every CTA reads
                       the hi and lo query tiles of every group, T R dim 4, plus its centroid tile, K dim 4
The profiler slows the host, so its step times are not bench.py's queries/s; use bench.py for that.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def short_name(name: str) -> str:
    """'void k_a5_bound<4>(unsigned short const*, ...)' -> 'k_a5_bound<4>'"""
    if name.startswith("void "):
        name = name[5:]
    depth = 0
    for i, ch in enumerate(name):
        if ch == "<":
            depth += 1
        elif ch == ">":
            depth -= 1
        elif ch == "(" and depth == 0:
            return name[:i]
    return name


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="output directory")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    own, rest = ap.parse_known_args()
    import bench
    sys.argv = [sys.argv[0], "--gpus", "1"] + rest
    args = bench.parse_args()
    args.steps, args.warmup = own.steps, own.warmup

    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile
    import next_plaid_b200 as npb
    if not torch.cuda.is_available():
        raise SystemExit("profile_step.py measures on a GPU; none is visible")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    bench.check_device_fits(args, 1, dev)
    G = bench.corpus_globals(args, dev)
    sh = bench.build_shard(args, G, 0, 1, dev)
    gpu = bench.open_shard(npb, args, G, sh, 0, 0)
    del sh["codes"]
    torch.cuda.empty_cache()
    params = npb.SearchParameters(top_k=args.top_k, n_ivf_probe=args.n_ivf_probe, n_full_scores=args.n_full_scores,
                                  centroid_score_threshold=args.threshold)
    n_batches = min(max(args.steps + args.warmup, 4), 24)
    queries = bench.make_queries(args, G, dev, n_batches * args.batch, seed=args.seed + 7)
    d_q = [torch.from_numpy(np.concatenate(queries[i * args.batch:(i + 1) * args.batch], 0)).to(dev)
           for i in range(n_batches)]
    offs = np.arange(args.batch + 1, dtype=np.int64) * args.nq
    d_ids = torch.empty((args.batch, args.top_k), dtype=torch.int64, device=dev)
    d_sc = torch.empty((args.batch, args.top_k), dtype=torch.float32, device=dev)
    d_cn = torch.empty((args.batch,), dtype=torch.int32, device=dev)

    def step(i):
        gpu.search_batch_device(d_q[i % n_batches].data_ptr(), offs, params, d_ids.data_ptr(), d_sc.data_ptr(),
                                d_cn.data_ptr())

    for i in range(args.warmup):
        step(i)
    torch.cuda.synchronize(dev)
    work = {}
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(args.steps):
            step(args.warmup + i)
            for k, v in gpu.last_work_counters().items():
                work[k] = work.get(k, 0) + v
        torch.cuda.synchronize(dev)

    kern = {}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        name = short_name(ev.name)
        if name.startswith("Memcpy") or name.startswith("Memset"):
            continue
        kern[name] = kern.get(name, 0.0) + ev.time_range.elapsed_us() / 1e3   # the kernel's span on the device
    S = args.steps
    kms = {k: v / S for k, v in sorted(kern.items(), key=lambda kv: -kv[1])}
    wps = {k: v / S for k, v in work.items()}
    QS = max(8, (args.nq + 7) & ~7) if args.nq <= 32 else (args.nq + 63) & ~63   # (query_row_tokens in engine.cu)
    bound_ms = sum(v for k, v in kms.items() if k.startswith("k_a5_bound"))
    hbm = wps.get("n_candidate_tokens", 0) * 4.0
    l2 = wps.get("n_a5_live_rows", 0) * 2.0 * QS
    K, dim, B = 1 << args.log2k, args.dim, args.batch
    passes = wps.get("n_k1_tc", 0)
    R, T = (B * QS + 127) // 128 * 128, (K + 127) // 128
    sc_ms = sum(v for k, v in kms.items() if k.startswith("k_scores16_tc"))
    flop = passes * 3 * 2 * R * 128 * T * dim
    wr = passes * (B * QS * K * 2 + 8 * T * R * 2)
    l2r = passes * (T * R * dim * 4 + K * dim * 4)

    def rate(x):
        return x / (sc_ms * 1e-3) if sc_ms > 0 else None
    out = {
        "gpu": bench.gpu_info(0),
        "workload": bench.workload_config(args, 1)["workload"],
        "steps": S, "warmup": args.warmup,
        "ms_per_step": {"kernels_total": sum(kms.values())},
        "kernel_ms_per_step": kms,
        "work_per_step": wps,
        "a5_bound": {"ms": bound_ms, "code_bytes_hbm": hbm, "live_row_bytes_l2": l2,
                     "gbs": (hbm + l2) / (bound_ms * 1e-3) / 1e9 if bound_ms > 0 else None,
                     "code_gbs": hbm / (bound_ms * 1e-3) / 1e9 if bound_ms > 0 else None},
        "scores_tc": {"ms": sc_ms, "passes": passes, "flop": flop, "table_write_bytes": wr, "operand_l2_bytes": l2r,
                      "tflops": rate(flop / 1e12), "table_write_gbs": rate(wr / 1e9),
                      "operand_l2_gbs": rate(l2r / 1e9)},
    }
    os.makedirs(own.out, exist_ok=True)
    with open(os.path.join(own.out, "profile_step.json"), "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps({"gpu": out["gpu"], "a5_bound": out["a5_bound"], "scores_tc": out["scores_tc"],
                      "top": dict(list(kms.items())[:8])}))
    gpu.close()


if __name__ == "__main__":
    main()
