"""Stand-in for the `next_plaid_b200` module backed by the CPU oracle, so bench.py's harness (corpus generator, query
decoding, recall / parity / roofline bookkeeping, JSON contract) runs end to end on a box without a GPU
(tests/test_bench_harness_cpu.py: PB_BENCH_LIB=fake_plaid PB_BENCH_DEVICE=cpu).  Test infrastructure only: nothing
here is the product, timings it reports are made up."""
import ctypes as C
import time

import numpy as np

from oracle import oracle

import next_plaid_b200 as _real

SearchParameters = _real.SearchParameters
QueryResult = _real.QueryResult
PlaidError = _real.PlaidError
STAGES = _real.STAGES


def _arr(ptr, n, ctype, dtype):
    if n == 0:
        return np.zeros(0, dtype)
    return np.ctypeslib.as_array((ctype * n).from_address(int(ptr))).view(dtype)


def _oparams(p):
    return oracle.SearchParameters(top_k=p.top_k, n_ivf_probe=p.n_ivf_probe, n_full_scores=p.n_full_scores,
                                   centroid_batch_size=p.centroid_batch_size,
                                   centroid_score_threshold=p.centroid_score_threshold)


class MmapIndex:
    def __init__(self, ix, base):
        self.ix, self.base, self._h = ix, base, self
        self.t_call = 0.0
        self.work = {}

    @classmethod
    def from_device_pointers(cls, dim, nbits, K, D, N, centroids, bucket_weights, codes, residuals, doc_lengths, ivf,
                             ivf_lengths, device=0, doc_id_base=0, adopt_residuals=False):
        assert ivf is None and ivf_lengths is None and adopt_residuals
        packed = dim * nbits // 8
        cen = _arr(centroids, K * dim, C.c_float, np.float32).reshape(K, dim).copy()
        w = _arr(bucket_weights, 1 << nbits, C.c_float, np.float32).copy()
        cd = _arr(codes, N, C.c_int64, np.int64).copy()
        rs = _arr(residuals, N * packed, C.c_uint8, np.uint8).reshape(N, packed).copy()
        dl = _arr(doc_lengths, D, C.c_int64, np.int64).copy()
        iv, il = oracle.build_ivf(cd, dl, K)
        return cls(oracle.Index(cen, w, None, cd, rs, dl, iv, il, nbits), doc_id_base)

    def num_documents(self):
        return self.ix.num_documents

    def comm_init(self, *a):
        raise NotImplementedError("the CPU dry-run is single-rank")

    def search_batch(self, queries, params, subset=None):
        t0 = time.perf_counter()
        po = _oparams(params)
        out = []
        for i, q in enumerate(queries):
            r = oracle.search_one(self.ix, q, po)
            out.append(QueryResult(i, r.passage_ids + self.base, r.scores))
        self.t_call = 1e3 * (time.perf_counter() - t0)
        nq = sum(len(q) for q in queries)
        self.work = dict(n_queries=len(queries), n_query_tokens=nq, n_cells=0, n_candidates=0,
                         n_candidate_tokens=1000 * len(queries), n_exact_docs=10 * len(queries),
                         n_exact_tokens=300 * len(queries), n_filter_docs=50 * len(queries),
                         n_filter_tokens=1500 * len(queries), k1_tc_max_code_diff=0, k1_rows_mismatch=0,
                         n_probe_threshold=0, n_probe_list=0, n_k1_tc=1, n_recheck_docs=0, n_k1_tc_redo=0, n_exact_pairs=0,
                         n_pair_fallback_queries=0, filter_err_ratio_e6=0, filter_diag_pairs=0)
        return out

    def _raw(self, qptr, offs, params, ids_ptr, sc_ptr, cn_ptr):
        offs = np.asarray(offs, np.int64)
        B, k, dim = len(offs) - 1, params.top_k, self.ix.dim
        flat = _arr(qptr, int(offs[-1]) * dim, C.c_float, np.float32).reshape(-1, dim)
        res = self.search_batch([flat[offs[i]:offs[i + 1]] for i in range(B)], params)
        ids = _arr(ids_ptr, B * k, C.c_int64, np.int64).reshape(B, k)
        sc = _arr(sc_ptr, B * k, C.c_float, np.float32).reshape(B, k)
        cn = _arr(cn_ptr, B, C.c_int32, np.int32)
        for i, r in enumerate(res):
            n = len(r.passage_ids)
            ids[i, :n], sc[i, :n], cn[i] = r.passage_ids, r.scores, n

    def search_batch_device(self, d_q, offs, params, d_ids, d_sc, d_cn):
        self._raw(d_q, offs, params, d_ids, d_sc, d_cn)

    def exhaustive_scores(self, queries):
        return np.stack([oracle.exhaustive_scores(self.ix, q) for q in queries])

    def set_lanes(self, lanes):
        pass

    def set_profiling(self, on):
        pass

    def set_scores_tc(self, on):
        pass

    def set_fast_exact(self, on):
        pass

    def last_call_ms(self):
        return self.t_call

    def last_stage_stats(self):
        return {s: self.t_call / len(STAGES) for s in STAGES}, {s: 2 for s in STAGES}

    def last_kernel_ms(self):
        return dict(scores=0.1 * self.t_call, approx16=0.4 * self.t_call, filter=0.2 * self.t_call, exact=0.1 * self.t_call)

    def last_work_counters(self):
        return dict(self.work)

    def close(self):
        pass


class _Lib:
    def pb_search_batch(self, h, qptr, offptr, n, pref, subset, n_subset, ids, sc, cn):
        pc = pref._obj
        thr = pc.centroid_score_threshold if pc.has_centroid_score_threshold else None
        p = SearchParameters(top_k=pc.top_k, n_ivf_probe=pc.n_ivf_probe, n_full_scores=pc.n_full_scores,
                             centroid_batch_size=pc.centroid_batch_size, centroid_score_threshold=thr)
        offs = _arr(offptr.value, n + 1, C.c_int64, np.int64)
        h._raw(qptr.value, offs, p, ids.value, sc.value, cn.value)
        return 0

    def pb_last_error(self):
        return b""


def load_library():
    return _Lib()


def comm_unique_id():
    raise NotImplementedError
