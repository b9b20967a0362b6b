"""A deployment behind one handle (pb_index_load_devices, DESIGN.md 4o) against a plain pb_index_load handle of the same
directory.  Writes a synthetic index directory the card holds (default 200k docs x 300 tokens x 128-d, K = 2^16, 4-bit
residuals: uniform random codes and residual bytes, L2-normalised random centroids, queries of 32 tokens near random
centroids) to a temporary directory, then measures, the handles alternating inside each run:
  batch       search_batch queries/s at batch --batch (top_k 10, n_ivf_probe 8, n_full_scores 4096)
  coalesced   queries/s and p50 / p99 latency of single-query `search` calls from --threads threads, coalescing on
              (max_queries 32, max_wait_us 200, max_inflight 2)
for `load` on device 0, `load_devices([0])` (one rank: the cost of the fan-out alone) and, when the machine exposes two
or more GPUs, `load_devices` over all of them.  A deployment runs one merged batch at a time, so `load` is also measured
coalesced with max_inflight 1 (`load/inflight1`, its batch line repeats `load`'s work): the control that tells that
limit apart from the cost of the fan-out.  Every result is compared with the `load` handle's.  Prints one JSON line
with the card name and power limit.

--replicas measures a replica set instead (pb_index_load_replicas, DESIGN.md 4q): `load` against
`load_replicas([0, 0])` (two copies on device 0), alternating inside each run: search_batch queries/s at batch 32 and
256, coalesced queries/s with p50 / p99 from --threads threads (max_inflight 2 per handle or replica), the load time of
each (the set's minus the plain handle's is the cost of the copy), and the device and host bytes.  The set is also
measured coalesced with max_inflight 1 per replica, as many merged batches in flight as `load` runs.  Every result is
compared with the `load` handle's.  With several GPUs it adds `load_replicas` over all of them.

Run from the repository root on an H100: python tools/bench_multi_device.py"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402


def write_dir(path, D, T, K, dim, nbits, seed):
    from oracle import oracle
    rng = np.random.default_rng(seed)
    cent = rng.standard_normal((K, dim), dtype=np.float32)
    cent /= np.linalg.norm(cent, axis=1, keepdims=True)
    N = D * T
    codes = rng.integers(0, K, N, dtype=np.int64)
    res = rng.integers(0, 256, (N, dim * nbits // 8), dtype=np.uint8)
    dl = np.full(D, T, np.int64)
    ivf, lens = oracle.build_ivf(codes, dl, K)
    w = np.linspace(-0.05, 0.05, 1 << nbits, dtype=np.float32)
    ix = oracle.Index(cent, w, None, codes, res, dl, ivf, lens, nbits)
    oracle.write_index(ix, path, chunk_docs=25_000)
    qs = []
    for _ in range(256):
        q = cent[rng.integers(0, K, 32)] + 0.05 * rng.standard_normal((32, dim), dtype=np.float32)
        qs.append(np.ascontiguousarray(q / np.linalg.norm(q, axis=1, keepdims=True), np.float32))
    return qs


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
        return out[0], float(out[1])
    except Exception:  # noqa: BLE001 - reported as unknown
        return "unknown", None


def coalesced(h, qs, p, threads, seconds, inflight, ref_one):
    """queries/s, latencies and mismatches of single-query searches from `threads` threads, coalescing on"""
    h.set_coalescing(32, max_wait_us=200, max_inflight=inflight)
    lat, done, differ = [[] for _ in range(threads)], [0] * threads, [0] * threads
    gate = threading.Barrier(threads + 1)
    stop = [0.0]

    def body(t):
        gate.wait()
        i = t * 7
        while time.perf_counter() < stop[0]:
            j = i % len(qs)
            t1 = time.perf_counter()
            r = h.search(qs[j], p)
            lat[t].append(time.perf_counter() - t1)
            differ[t] += (r.passage_ids.tobytes(), r.scores.tobytes()) != ref_one[j]
            done[t] += 1
            i += 1
    ths = [threading.Thread(target=body, args=(t,)) for t in range(threads)]
    [t.start() for t in ths]
    stop[0] = time.perf_counter() + seconds
    t1 = time.perf_counter()
    gate.wait()
    [t.join() for t in ths]
    wall = time.perf_counter() - t1
    h.set_coalescing(1)
    return sum(done) / wall, [x for per in lat for x in per], sum(differ)


def replica_arm(a, npb, path, qs, p, write_s):
    n_gpu = npb.device_count()
    opens = {"load": lambda: npb.MmapIndex.load(path),
             "load_replicas[0,0]": lambda: npb.MmapIndex.load_replicas(path, [0, 0])}
    if n_gpu >= 2:
        opens[f"load_replicas[0..{n_gpu - 1}]"] = lambda: npb.MmapIndex.load_replicas(path, list(range(n_gpu)))
    res = lambda rs: [(r.passage_ids.tobytes(), r.scores.tobytes()) for r in rs]  # noqa: E731
    acc = {n: dict(b32=[], b256=[], coal=[], lat=[], load_s=[], differ=0) for n in opens}
    mem, ref, ref_one = {}, None, None
    for run in range(a.runs + 1):                         # run 0 warms every shape up
        for n, op in opens.items():
            t0 = time.perf_counter()
            h = op()
            load_s = time.perf_counter() - t0
            try:
                if ref is None:
                    ref = {bs: [res(h.search_batch(qs[i:i + bs], p)) for i in range(0, len(qs), bs)] for bs in (32, 256)}
                    ref_one = [res([h.search(q, p)])[0] for q in qs]
                mem[n] = h.memory_usage()
                rates = {}
                for bs in (32, 256):
                    batches = [qs[i:i + bs] for i in range(0, len(qs), bs)]
                    acc[n]["differ"] += sum(res(h.search_batch(b, p)) != r for b, r in zip(batches, ref[bs]))
                    k, t0 = 0, time.perf_counter()
                    while time.perf_counter() - t0 < a.seconds:
                        for b in batches:
                            h.search_batch(b, p)
                            k += len(b)
                    rates[bs] = k / (time.perf_counter() - t0)
                q, lat, differ = coalesced(h, qs, p, a.threads, a.seconds, 2, ref_one)
                acc[n]["differ"] += differ
                if n != "load":   # the control: one merged batch per replica, as many in flight as `load` runs
                    q1, lat1, differ1 = coalesced(h, qs, p, a.threads, a.seconds, 1, ref_one)
                    acc[n]["differ"] += differ1
                    if run:
                        acc[n].setdefault("coal1", []).append(q1)
                        acc[n].setdefault("lat1", []).extend(lat1)
                if run:
                    acc[n]["b32"].append(rates[32])
                    acc[n]["b256"].append(rates[256])
                    acc[n]["coal"].append(q)
                    acc[n]["lat"] += lat
                    acc[n]["load_s"].append(load_s)
            finally:
                h.close()
    out = {}
    for n, v in acc.items():
        lat = np.array(v["lat"]) * 1e3
        span = lambda xs: [round(min(xs), 1), round(max(xs), 1)]  # noqa: E731
        out[n] = dict(batch32_qps=round(float(np.median(v["b32"])), 1), batch32_qps_range=span(v["b32"]),
                      batch256_qps=round(float(np.median(v["b256"])), 1), batch256_qps_range=span(v["b256"]),
                      coalesced_qps=round(float(np.median(v["coal"])), 1), coalesced_qps_range=span(v["coal"]),
                      p50_ms=round(float(np.percentile(lat, 50)), 3), p99_ms=round(float(np.percentile(lat, 99)), 3),
                      load_s=round(float(np.median(v["load_s"])), 2), load_s_range=[round(min(v["load_s"]), 2),
                                                                                    round(max(v["load_s"]), 2)],
                      device_bytes=mem[n]["device_bytes"], host_bytes=mem[n]["host_bytes"],
                      same_as_load=v["differ"] == 0)
        if "coal1" in v:
            lat1 = np.array(v["lat1"]) * 1e3
            out[n].update(coalesced_inflight1_qps=round(float(np.median(v["coal1"])), 1),
                          coalesced_inflight1_qps_range=span(v["coal1"]),
                          inflight1_p50_ms=round(float(np.percentile(lat1, 50)), 3),
                          inflight1_p99_ms=round(float(np.percentile(lat1, 99)), 3))
    if n_gpu < 2:
        out["load_replicas[all GPUs]"] = "not measured: one GPU visible"
    name, power = gpu_info()
    print(json.dumps(dict(arm="replicas", docs=a.docs, doclen=a.doclen, K=1 << a.log2k, nbits=4, threads=a.threads,
                          runs=a.runs, seconds=a.seconds, write_s=round(write_s, 1), gpus=n_gpu, results=out,
                          gpu=name, power_limit_w=power)), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=200_000)
    ap.add_argument("--doclen", type=int, default=300)
    ap.add_argument("--log2k", type=int, default=16)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--threads", type=int, default=32)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--seconds", type=float, default=2.0)
    ap.add_argument("--replicas", action="store_true")
    a = ap.parse_args()
    import next_plaid_b200 as npb
    if npb.device_count() < 1:
        raise SystemExit("needs an H100: the library has no CPU fallback")
    tmp = tempfile.mkdtemp(prefix="pb_multi_device_")
    try:
        t0 = time.perf_counter()
        qs = write_dir(tmp, a.docs, a.doclen, 1 << a.log2k, 128, 4, 7)
        write_s = time.perf_counter() - t0
        p = npb.SearchParameters(top_k=10, n_ivf_probe=8, n_full_scores=4096)
        n_gpu = npb.device_count()
        if a.replicas:
            return replica_arm(a, npb, tmp, qs, p, write_s)
        handles = {"load": npb.MmapIndex.load(tmp), "load_devices[0]": npb.MmapIndex.load_devices(tmp, [0])}
        if n_gpu >= 2:
            handles[f"load_devices[0..{n_gpu - 1}]"] = npb.MmapIndex.load_devices(tmp, list(range(n_gpu)))
        batches = [qs[i:i + a.batch] for i in range(0, len(qs), a.batch)]
        res = lambda rs: [(r.passage_ids.tobytes(), r.scores.tobytes()) for r in rs]  # noqa: E731
        ref = [res(handles["load"].search_batch(b, p)) for b in batches]
        ref_one = [res([handles["load"].search(q, p)])[0] for q in qs]
        same = {n: all(res(h.search_batch(b, p)) == r for b, r in zip(batches, ref)) for n, h in handles.items()}

        def batch_run(h):
            n, t0 = 0, time.perf_counter()
            while time.perf_counter() - t0 < a.seconds:
                for b in batches:
                    h.search_batch(b, p)
                    n += len(b)
            return n / (time.perf_counter() - t0)

        def coalesced_run(h, inflight):
            return coalesced(h, qs, p, a.threads, a.seconds, inflight, ref_one)

        cells = [(n, h, 2) for n, h in handles.items()]
        cells.insert(1, ("load/inflight1", handles["load"], 1))
        acc = {n: dict(batch=[], coal=[], lat=[], differ=0) for n, _, _ in cells}
        for run in range(a.runs + 1):                     # run 0 warms every handle up
            for n, h, inflight in cells:
                q1 = batch_run(h)
                q2, lat, differ = coalesced_run(h, inflight)
                acc[n]["differ"] += differ
                if run:
                    acc[n]["batch"].append(q1)
                    acc[n]["coal"].append(q2)
                    acc[n]["lat"] += lat
        out = {}
        for n, v in acc.items():
            lat = np.array(v["lat"]) * 1e3
            out[n] = dict(batch_qps=round(float(np.median(v["batch"])), 1),
                          batch_qps_range=[round(min(v["batch"]), 1), round(max(v["batch"]), 1)],
                          coalesced_qps=round(float(np.median(v["coal"])), 1),
                          coalesced_qps_range=[round(min(v["coal"]), 1), round(max(v["coal"]), 1)],
                          p50_ms=round(float(np.percentile(lat, 50)), 3), p99_ms=round(float(np.percentile(lat, 99)), 3),
                          same_as_load=same[n.split("/")[0]] and v["differ"] == 0)
        if n_gpu < 2:
            out["load_devices[all GPUs]"] = "not measured: one GPU visible"
        for h in handles.values():
            h.close()
        name, power = gpu_info()
        print(json.dumps(dict(docs=a.docs, doclen=a.doclen, K=1 << a.log2k, nbits=4, batch=a.batch, threads=a.threads,
                              runs=a.runs, seconds=a.seconds, write_s=round(write_s, 1), gpus=n_gpu, results=out,
                              gpu=name, power_limit_w=power)), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
