"""Host-side mirror of the reference's index/search interface over the C-ABI of libplaid_b200.

Names, argument meaning and error behaviour follow next-plaid/src (paths relative to it):
  MmapIndex.load / search / search_batch / accessors ... index.rs:1026, :1258, :1279, :1290-1312
  SearchParameters, QueryResult ........................ search.rs:27-80
  Error kinds .......................................... error.rs:10-66

This module is a thin ctypes binding: all work happens in hand-written sm_90a kernels behind
include/plaid_b200.h.  There is no CPU path: if the shared library or an H100 is missing every call
raises.
"""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass
from typing import List, Optional, Sequence

import numpy as np

_PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_PKG, "libplaid_b200.so")

PB_OK, PB_ERR_INVALID, PB_ERR_CUDA, PB_ERR_IO, PB_ERR_UNSUPPORTED, PB_ERR_NOMEM, PB_ERR_COMM = range(7)
STAGES = ["h2d", "centroid_scores", "probe", "candidates", "approx", "cut", "exact", "topk", "d2h"]


class PlaidError(RuntimeError):
    """next_plaid::Error (error.rs:10-66); `.status` is the pb_status code."""

    def __init__(self, status: int, message: str):
        super().__init__(f"[pb_status {status}] {message}")
        self.status = status


class _Desc(C.Structure):
    _fields_ = [
        ("dim", C.c_int32), ("nbits", C.c_int32), ("num_centroids", C.c_int64),
        ("num_documents", C.c_int64), ("num_embeddings", C.c_int64),
        ("centroids", C.c_void_p), ("bucket_weights", C.c_void_p), ("codes", C.c_void_p),
        ("residuals", C.c_void_p), ("doc_lengths", C.c_void_p), ("ivf", C.c_void_p),
        ("ivf_lengths", C.c_void_p), ("device", C.c_int32), ("memory_space", C.c_int32),
        ("doc_id_base", C.c_int64), ("flags", C.c_int32),
    ]


class _Params(C.Structure):
    _fields_ = [
        ("batch_size", C.c_int64), ("n_full_scores", C.c_int64), ("top_k", C.c_int64),
        ("n_ivf_probe", C.c_int64), ("centroid_batch_size", C.c_int64),
        ("has_centroid_score_threshold", C.c_int32), ("centroid_score_threshold", C.c_float),
    ]


class _Trace(C.Structure):
    _fields_ = [
        ("cells", C.c_void_p), ("n_cells", C.c_void_p), ("cells_cap", C.c_int64),
        ("candidates", C.c_void_p), ("approx", C.c_void_p), ("n_candidates", C.c_void_p),
        ("cand_cap", C.c_int64),
        ("kept", C.c_void_p), ("kept_exact", C.c_void_p), ("n_kept", C.c_void_p),
        ("kept_cap", C.c_int64),
    ]


class _Work(C.Structure):
    _fields_ = [(n, C.c_int64) for n in ("n_queries", "n_query_tokens", "n_cells", "n_candidates",
                                         "n_candidate_tokens", "n_exact_docs", "n_exact_tokens",
                                         "n_filter_docs", "n_filter_tokens", "k1_tc_max_code_diff",
                                         "k1_rows_mismatch", "n_probe_threshold", "n_probe_list", "n_k1_tc",
                                         "n_recheck_docs", "n_k1_tc_redo", "n_exact_pairs",
                                         "n_pair_fallback_queries", "filter_err_ratio_e6", "filter_diag_pairs",
                                         "n_a5_live_rows", "n_a5_dense_docs")]


class _CoalesceConfig(C.Structure):
    _fields_ = [("max_queries", C.c_int32), ("max_wait_us", C.c_int32), ("max_inflight", C.c_int32)]


class _CoalesceStats(C.Structure):
    _fields_ = [("n_requests", C.c_int64), ("n_batches", C.c_int64), ("n_bypassed", C.c_int64),
                ("n_refused", C.c_int64), ("n_rerun_alone", C.c_int64), ("max_batch", C.c_int64),
                ("batch_hist", C.c_int64 * 8), ("queue_wait_us", C.c_int64)]


EXPORTS = [
    "pb_search_params_default", "pb_index_load", "pb_index_open", "pb_index_close",
    "pb_index_num_documents", "pb_index_num_embeddings", "pb_index_num_partitions",
    "pb_index_avg_doclen", "pb_index_embedding_dim", "pb_index_nbits", "pb_index_device",
    "pb_search_batch", "pb_search_batch_traced", "pb_search_batch_subsets", "pb_search_batch_params", "pb_centroid_scores", "pb_decompress_documents",
    "pb_maxsim_scores", "pb_exhaustive_scores", "pb_set_profiling", "pb_last_stage_stats",
    "pb_last_work_counters", "pb_search_batch_device", "pb_last_error", "pb_version",
    "pb_device_count", "pb_comm_unique_id", "pb_index_comm_init", "pb_shard_group_create", "pb_shard_group_destroy",
    "pb_index_group_join", "pb_index_export_ivf", "pb_last_call_ms", "pb_last_kernel_ms", "pb_set_fast_approx", "pb_set_fast_exact", "pb_set_scores_tc", "pb_set_lanes",
    "pb_codec_open", "pb_codec_close", "pb_codec_compress_into_codes", "pb_codec_compress_and_residuals",
    "pb_codec_encode_chunk", "pb_kmeans_fit", "pb_codec_train", "pb_kmeans_num_sample_docs",
    "pb_kmeans_num_partitions", "pb_codec_num_sample_docs", "pb_codec_heldout_tokens", "pb_create_index",
    "pb_create_params_default", "pb_build_comm_init", "pb_build_comm_group", "pb_build_comm_destroy", "pb_kmeans_fit_dp", "pb_codec_last_assign_stats", "pb_codec_find_outliers",
    "pb_index_append", "pb_index_append_encoded", "pb_index_reserve",
    "pb_index_delete", "pb_last_delete_ms", "pb_index_load_range", "pb_index_dir_shard_bounds",
    "pb_index_delete_sharded", "pb_index_append_sharded", "pb_index_append_encoded_sharded",
    "pb_index_rebalance_sharded", "pb_index_load_range_flags", "pb_index_memory", "pb_last_staging_stats",
    "pb_search", "pb_index_set_coalescing", "pb_index_coalesce_stats",
]

PB_OPEN_ADOPT_RESIDUALS, PB_OPEN_HOST_RESIDUALS = 1, 2

_lib = None


def load_library():
    """dlopen libplaid_b200.so; raise (never fall back) when it is missing."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise PlaidError(PB_ERR_CUDA, f"{LIB_PATH} is not built (run __graft_entry__.build()); "
                                          "there is no CPU fallback for the search path")
        L = C.CDLL(LIB_PATH)
        L.pb_last_error.restype = C.c_char_p
        L.pb_version.restype = C.c_char_p
        for f in ("pb_index_num_documents", "pb_index_num_embeddings", "pb_index_num_partitions"):
            getattr(L, f).restype = C.c_int64
            getattr(L, f).argtypes = [C.c_void_p]
        L.pb_index_avg_doclen.restype = C.c_double
        L.pb_index_avg_doclen.argtypes = [C.c_void_p]
        for f in ("pb_index_embedding_dim", "pb_index_nbits", "pb_index_device"):
            getattr(L, f).restype = C.c_int32
            getattr(L, f).argtypes = [C.c_void_p]
        L.pb_index_close.argtypes = [C.c_void_p]
        L.pb_index_close.restype = None
        L.pb_set_profiling.argtypes = [C.c_void_p, C.c_int32]
        L.pb_set_profiling.restype = None
        L.pb_set_fast_approx.argtypes = [C.c_void_p, C.c_int32]
        L.pb_set_fast_approx.restype = None
        L.pb_set_fast_exact.argtypes = [C.c_void_p, C.c_int32]
        L.pb_set_fast_exact.restype = None
        L.pb_set_scores_tc.argtypes = [C.c_void_p, C.c_int32]
        L.pb_set_scores_tc.restype = None
        L.pb_set_lanes.argtypes = [C.c_void_p, C.c_int32]
        L.pb_set_lanes.restype = None
        L.pb_index_load.argtypes = [C.c_char_p, C.c_int32, C.POINTER(C.c_void_p)]
        L.pb_index_load_range.argtypes = [C.c_char_p, C.c_int32, C.c_int64, C.c_int64, C.POINTER(C.c_void_p)]
        L.pb_index_load_range_flags.argtypes = [C.c_char_p, C.c_int32, C.c_int64, C.c_int64, C.c_int32,
                                                C.POINTER(C.c_void_p)]
        L.pb_index_memory.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.pb_last_staging_stats.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.pb_index_dir_shard_bounds.argtypes = [C.c_char_p, C.c_int32, C.c_void_p]
        L.pb_index_open.argtypes = [C.POINTER(_Desc), C.POINTER(C.c_void_p)]
        L.pb_search_batch_traced.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                             C.POINTER(_Params), C.c_void_p, C.c_int64, C.c_void_p,
                                             C.c_void_p, C.c_void_p, C.c_void_p]
        L.pb_search_batch.argtypes = L.pb_search_batch_traced.argtypes[:-1]
        L.pb_search_batch_subsets.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.POINTER(_Params),
                                              C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                              C.c_void_p]
        L.pb_search_batch_params.argtypes = list(L.pb_search_batch_subsets.argtypes)
        L.pb_search.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.POINTER(_Params), C.c_void_p, C.c_int64,
                                C.c_void_p, C.c_void_p, C.c_void_p]
        L.pb_index_set_coalescing.argtypes = [C.c_void_p, C.POINTER(_CoalesceConfig)]
        L.pb_index_coalesce_stats.argtypes = [C.c_void_p, C.POINTER(_CoalesceStats), C.c_int32]
        L.pb_search_batch_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                             C.POINTER(_Params), C.c_void_p, C.c_void_p, C.c_void_p]
        L.pb_centroid_scores.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
        L.pb_decompress_documents.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
        L.pb_maxsim_scores.argtypes = [C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p,
                                       C.c_void_p, C.c_int64, C.c_void_p]
        L.pb_exhaustive_scores.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
        L.pb_last_stage_stats.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.pb_last_work_counters.argtypes = [C.c_void_p, C.POINTER(_Work)]
        L.pb_last_call_ms.argtypes = [C.c_void_p, C.c_void_p]
        L.pb_last_kernel_ms.argtypes = [C.c_void_p, C.c_void_p]
        L.pb_index_export_ivf.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.pb_codec_open.argtypes = [C.c_int32, C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_void_p,
                                    C.POINTER(C.c_void_p)]
        L.pb_codec_close.argtypes = [C.c_void_p]
        L.pb_codec_close.restype = None
        L.pb_codec_find_outliers.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_float, C.c_void_p, C.c_void_p]
        L.pb_codec_last_assign_stats.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.pb_codec_compress_into_codes.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
        L.pb_codec_compress_and_residuals.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
        L.pb_codec_encode_chunk.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
        L.pb_kmeans_fit.argtypes = [C.c_int32, C.c_void_p, C.c_int64, C.c_int32, C.c_int64, C.c_int32, C.c_uint64,
                                    C.c_void_p]
        L.pb_codec_train.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        for f in ("pb_kmeans_num_sample_docs", "pb_codec_num_sample_docs", "pb_codec_heldout_tokens"):
            getattr(L, f).restype = C.c_int64
            getattr(L, f).argtypes = [C.c_int64]
        L.pb_kmeans_num_partitions.restype = C.c_int64
        L.pb_kmeans_num_partitions.argtypes = [C.c_int64, C.c_double, C.c_int64]
        L.pb_create_index.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_char_p, C.c_void_p]
        L.pb_create_params_default.argtypes = [C.c_void_p]
        L.pb_create_params_default.restype = None
        L.pb_build_comm_init.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]
        L.pb_build_comm_group.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p]
        L.pb_build_comm_destroy.argtypes = [C.c_void_p]
        L.pb_build_comm_destroy.restype = None
        L.pb_kmeans_fit_dp.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int64, C.c_int32, C.c_uint64, C.c_void_p]
        L.pb_comm_unique_id.argtypes = [C.c_void_p]
        L.pb_index_comm_init.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32]
        L.pb_shard_group_create.argtypes = [C.c_int32, C.c_void_p]
        L.pb_shard_group_destroy.argtypes = [C.c_void_p]
        L.pb_shard_group_destroy.restype = None
        L.pb_index_group_join.argtypes = [C.c_void_p, C.c_void_p, C.c_int32]
        L.pb_index_append.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_char_p,
                                      C.c_int64, C.c_void_p]
        L.pb_index_append_encoded.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32,
                                              C.c_void_p]
        L.pb_index_reserve.argtypes = [C.c_void_p, C.c_int64, C.c_int64]
        L.pb_index_delete.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_char_p, C.c_void_p]
        L.pb_last_delete_ms.argtypes = [C.c_void_p, C.c_void_p]
        L.pb_index_delete_sharded.argtypes = L.pb_index_delete.argtypes
        L.pb_index_append_sharded.argtypes = L.pb_index_append.argtypes
        L.pb_index_append_encoded_sharded.argtypes = L.pb_index_append_encoded.argtypes
        L.pb_index_rebalance_sharded.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        _lib = L
    return _lib


def _check(status: int):
    if status != PB_OK:
        raise PlaidError(status, load_library().pb_last_error().decode("utf-8", "replace"))


def _ptr(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _per_rank(n: int, call) -> list:
    """call(r) for r in range(n), one host thread per rank (the ranks of an in-process shard group); the results in
    rank order, or the first rank's exception once every thread has finished"""
    import threading
    out, err = [None] * n, [None] * n

    def run(r):
        try:
            out[r] = call(r)
        except Exception as e:      # noqa: BLE001 - re-raised below
            err[r] = e
    ths = [threading.Thread(target=run, args=(r,)) for r in range(n)]
    [t.start() for t in ths]
    [t.join() for t in ths]
    for e in err:
        if e is not None:
            raise e
    return out


class ShardGroup:
    """pb_shard_group: several shard handles of ONE process searched and changed together (one host thread per shard).

    `search_batch`, `delete`, `append` and `append_encoded` run the collective from len(shards) threads and return
    rank 0's result (every rank's result is identical; `all_results` keeps them for the tests)."""

    def __init__(self, shards: Sequence["MmapIndex"]):
        self.shards = list(shards)
        h = C.c_void_p()
        _check(load_library().pb_shard_group_create(len(self.shards), C.byref(h)))
        self._g = h
        for r, s in enumerate(self.shards):
            _check(load_library().pb_index_group_join(s._h, self._g, r))
            s._world = len(self.shards)
        self.all_results = None

    def _collective(self, call):
        """call(r, shard) from one thread per rank; the per-rank results, or the first rank's exception"""
        self.all_results = _per_rank(len(self.shards), lambda r: call(r, self.shards[r]))
        return self.all_results

    def search_batch(self, queries, params=None, subset=None):
        return self._collective(lambda r, s: s.search_batch(queries, params, subset=subset))[0]

    def search_batch_subsets(self, queries, params, subsets, trace=False):
        """MmapIndex.search_batch_subsets on the whole deployment (global ids; every rank gets the same subsets)."""
        return self._collective(lambda r, s: s.search_batch_subsets(queries, params, subsets, trace=trace))[0]

    def search_batch_params(self, queries, params, subsets=None, trace=False):
        """MmapIndex.search_batch_params on the whole deployment (every rank gets the same parameters and subsets)."""
        return self._collective(lambda r, s: s.search_batch_params(queries, params, subsets, trace=trace))[0]

    def delete(self, doc_ids: Sequence[int], index_dir: Optional[str] = None) -> int:
        """pb_index_delete_sharded: MmapIndex.delete on the whole deployment (global ids); each rank renumbers its
        survivors and shifts its doc_id_base, and with `index_dir` the last rank applies delete_from_index's file
        changes.  Returns the number of documents removed over all ranks."""
        ids = np.ascontiguousarray(doc_ids, np.int64).reshape(-1)
        d = None if index_dir is None else os.fsencode(index_dir)

        def call(r, s):
            n = C.c_int64()
            _check(load_library().pb_index_delete_sharded(s._h, _ptr(ids), len(ids), d, C.byref(n)))
            return int(n.value)
        return self._collective(call)[0]

    def append(self, embeddings: Sequence[np.ndarray], codec: "ResidualCodec", index_dir: Optional[str] = None,
               batch_size: int = 50_000) -> List[int]:
        """pb_index_append_sharded: MmapIndex.append on the whole deployment.  The documents go to the last rank as
        ids D_total ..; with `index_dir` the last rank applies update_index's file changes.  Returns the new ids."""
        dl = np.array([e.shape[0] for e in embeddings], np.int64)
        dim = self.shards[-1].embedding_dim()
        flat = (np.ascontiguousarray(np.concatenate(embeddings, 0), np.float32) if len(embeddings)
                else np.zeros((0, dim), np.float32))
        d = None if index_dir is None else os.fsencode(index_dir)
        W = len(self.shards)

        def call(r, s):
            first = C.c_int64()
            last = r == W - 1
            _check(load_library().pb_index_append_sharded(s._h, codec._h if last else None, _ptr(flat) if last else None,
                                                          _ptr(dl), len(dl), 0, d, batch_size, C.byref(first)))
            return first.value
        first = self._collective(call)[0]
        return list(range(first, first + len(dl)))

    def append_encoded(self, codes: np.ndarray, residuals: np.ndarray, doc_lengths: Sequence[int]) -> List[int]:
        """pb_index_append_encoded_sharded: MmapIndex.append_encoded on the whole deployment (to the last rank)."""
        cd = np.ascontiguousarray(codes, np.int64)
        rs = np.ascontiguousarray(residuals, np.uint8)
        dl = np.ascontiguousarray(doc_lengths, np.int64)
        last = self.shards[-1]
        if rs.size != len(cd) * last.embedding_dim() * last.nbits() // 8 or int(dl.sum()) != len(cd):
            raise PlaidError(PB_ERR_INVALID, f"codes {cd.shape}, residuals {rs.shape} and doc_lengths (sum "
                                             f"{int(dl.sum())}) do not describe the same tokens")
        W = len(self.shards)

        def call(r, s):
            first = C.c_int64()
            mine = r == W - 1
            _check(load_library().pb_index_append_encoded_sharded(s._h, _ptr(cd) if mine else None,
                                                                  _ptr(rs) if mine else None, _ptr(dl), len(dl), 0,
                                                                  C.byref(first)))
            return first.value
        first = self._collective(call)[0]
        return list(range(first, first + len(dl)))

    def rebalance(self, bounds: Optional[Sequence[int]] = None) -> np.ndarray:
        """pb_index_rebalance_sharded: rank r takes documents [bounds[r], bounds[r + 1]) of the deployment (None: the
        token-balanced split), moving them between the ranks on the device; global ids and search results do not
        change.  Returns the bounds applied."""
        return self._collective(lambda r, s: s.rebalance_sharded(bounds))[0]

    def close(self):
        for s in self.shards:
            s.close()
        self.shards = []
        if self._g:
            load_library().pb_shard_group_destroy(self._g)
            self._g = None


def comm_unique_id() -> bytes:
    """pb_comm_unique_id (rank 0); ship the 128 bytes to the other ranks."""
    buf = np.zeros(128, np.uint8)
    _check(load_library().pb_comm_unique_id(_ptr(buf)))
    return buf.tobytes()


def device_count() -> int:
    return int(load_library().pb_device_count())


def shard_bounds(index_path: str, world: int) -> np.ndarray:
    """pb_index_dir_shard_bounds: the token-balanced split of the directory's documents over `world` ranks, <i8
    [world + 1]; rank r holds documents [bounds[r], bounds[r + 1]).  Host only."""
    out = np.zeros(max(int(world), 0) + 1, np.int64)
    _check(load_library().pb_index_dir_shard_bounds(os.fsencode(index_path), world, _ptr(out)))
    return out


@dataclass
class SearchParameters:
    """search.rs:27-69; defaults are SearchParameters::default() (search.rs:58-69)."""
    batch_size: int = 2000
    n_full_scores: int = 4096
    top_k: int = 10
    n_ivf_probe: int = 8
    centroid_batch_size: int = 100_000
    centroid_score_threshold: Optional[float] = 0.4

    def _c(self) -> _Params:
        t = self.centroid_score_threshold
        return _Params(self.batch_size, self.n_full_scores, self.top_k, self.n_ivf_probe,
                       self.centroid_batch_size, 0 if t is None else 1, 0.0 if t is None else float(t))


@dataclass
class QueryResult:
    """search.rs:72-80."""
    query_id: int
    passage_ids: np.ndarray
    scores: np.ndarray


@dataclass
class SearchTrace:
    cells: List[np.ndarray]
    candidates: List[np.ndarray]
    approx: List[np.ndarray]
    kept: List[np.ndarray]
    kept_exact: List[np.ndarray]


def _subset_args(subsets, n_queries):
    """(offsets, ids, has) of pb_search_batch_subsets for a list of Option<&[i64]> subsets (None: no query has one)"""
    if subsets is None:
        subsets = [None] * n_queries
    if len(subsets) != n_queries:
        raise PlaidError(PB_ERR_INVALID, f"{len(subsets)} subsets for {n_queries} queries")
    has = np.array([s is not None for s in subsets], np.uint8)
    lists = [np.ascontiguousarray(s, np.int64).reshape(-1) if s is not None else np.zeros(0, np.int64)
             for s in subsets]
    so = np.zeros(len(lists) + 1, np.int64)
    so[1:] = np.cumsum([len(x) for x in lists])
    si = np.ascontiguousarray(np.concatenate(lists) if lists else np.zeros(0, np.int64), np.int64)
    return so, si, has


def _pack_queries(queries: Sequence[np.ndarray], dim: int):
    offs = np.zeros(len(queries) + 1, np.int64)
    for i, q in enumerate(queries):
        q = np.asarray(q)
        if q.ndim != 2 or q.shape[1] != dim:
            raise PlaidError(PB_ERR_INVALID, f"query {i} has shape {q.shape}, expected [tokens, {dim}]")
        offs[i + 1] = offs[i] + q.shape[0]
    flat = np.zeros((int(offs[-1]), dim), np.float32)
    for i, q in enumerate(queries):
        flat[offs[i]:offs[i + 1]] = q
    return flat, offs


class MmapIndex:
    """GPU-resident stand-in for next_plaid::MmapIndex (index.rs:995-1016)."""

    def __init__(self, handle: int, path: str = ""):
        self._h = C.c_void_p(handle)
        self.path = path
        self._world = 1           # ranks of the doc-sharded deployment it joined (comm_init / ShardGroup)

    # -- construction ----------------------------------------------------------------------
    @classmethod
    def load(cls, index_path: str, device: int = 0, host_residuals: bool = False) -> "MmapIndex":
        """MmapIndex::load (index.rs:1026): reads the reference's index directory.  host_residuals: the packed
        residuals go to pinned host memory instead of the device (PB_OPEN_HOST_RESIDUALS; same results, slower search,
        no appends or deletes)."""
        L = load_library()
        h = C.c_void_p()
        if host_residuals:
            _check(L.pb_index_load_range_flags(os.fsencode(index_path), device, 0, -1, PB_OPEN_HOST_RESIDUALS,
                                               C.byref(h)))
        else:
            _check(L.pb_index_load(os.fsencode(index_path), device, C.byref(h)))
        return cls(h.value, index_path)

    @classmethod
    def load_range(cls, index_path: str, doc_begin: int, doc_end: int, device: int = 0,
                   host_residuals: bool = False) -> "MmapIndex":
        """pb_index_load_range: documents [doc_begin, doc_end) of the directory as one shard of a doc-sharded
        deployment (doc_id_base = doc_begin, so search returns global ids).  Reads only that range's chunk rows.
        host_residuals: as for load."""
        h = C.c_void_p()
        L = load_library()
        if host_residuals:
            _check(L.pb_index_load_range_flags(os.fsencode(index_path), device, doc_begin, doc_end,
                                               PB_OPEN_HOST_RESIDUALS, C.byref(h)))
        else:
            _check(L.pb_index_load_range(os.fsencode(index_path), device, doc_begin, doc_end, C.byref(h)))
        return cls(h.value, index_path)

    @classmethod
    def load_shard(cls, index_path: str, rank: int, world: int, device: int = 0,
                   host_residuals: bool = False) -> "MmapIndex":
        """Shard `rank` of `world` of the directory: load_range over shard_bounds(index_path, world)."""
        if not 0 <= rank < world:
            raise PlaidError(PB_ERR_INVALID, f"rank {rank} outside [0, {world})")
        b = shard_bounds(index_path, world)
        return cls.load_range(index_path, int(b[rank]), int(b[rank + 1]), device, host_residuals)

    @classmethod
    def from_arrays(cls, centroids, bucket_weights, codes, residuals, doc_lengths, ivf, ivf_lengths,
                    nbits: int, device: int = 0, doc_id_base: int = 0, host_residuals: bool = False) -> "MmapIndex":
        """pb_index_open from host arrays in the reference's dtypes.  host_residuals: as for load."""
        L = load_library()
        cen = np.ascontiguousarray(centroids, np.float32)
        w = np.ascontiguousarray(bucket_weights, np.float32)
        cd = np.ascontiguousarray(codes, np.int64)
        rs = np.ascontiguousarray(residuals, np.uint8)
        dl = np.ascontiguousarray(doc_lengths, np.int64)
        # ivf = ivf_lengths = None: the inverted file is built on the device from the codes (index.rs:850-873)
        iv = None if ivf is None else np.ascontiguousarray(ivf, np.int64)
        il = None if ivf_lengths is None else np.ascontiguousarray(ivf_lengths, np.int32)
        d = _Desc(cen.shape[1], nbits, cen.shape[0], len(dl), len(cd), _ptr(cen), _ptr(w), _ptr(cd),
                  _ptr(rs), _ptr(dl), _ptr(iv), _ptr(il), device, 0, doc_id_base,
                  PB_OPEN_HOST_RESIDUALS if host_residuals else 0)
        h = C.c_void_p()
        _check(L.pb_index_open(C.byref(d), C.byref(h)))
        return cls(h.value)

    @classmethod
    def from_device_pointers(cls, dim, nbits, K, D, N, centroids, bucket_weights, codes, residuals,
                             doc_lengths, ivf, ivf_lengths, device: int = 0, doc_id_base: int = 0,
                             adopt_residuals: bool = False, host_residuals: bool = False):
        """pb_index_open with PB_MEM_DEVICE pointers (integers), e.g. torch tensors' data_ptr().  ivf = ivf_lengths
        = None: the inverted file is built on the device (index.rs:850-873).  adopt_residuals: the packed residuals
        are used in place (keep the array alive until close()).  host_residuals: they are copied to pinned host
        memory, as for load."""
        L = load_library()
        flags = (PB_OPEN_ADOPT_RESIDUALS if adopt_residuals else 0) | (PB_OPEN_HOST_RESIDUALS if host_residuals else 0)
        d = _Desc(dim, nbits, K, D, N, centroids, bucket_weights, codes, residuals, doc_lengths, ivf,
                  ivf_lengths, device, 1, doc_id_base, flags)
        h = C.c_void_p()
        _check(L.pb_index_open(C.byref(d), C.byref(h)))
        return cls(h.value)

    def close(self):
        if self._h:
            load_library().pb_index_close(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- accessors (index.rs:1290-1312) ----------------------------------------------------------
    def num_documents(self) -> int:
        return int(load_library().pb_index_num_documents(self._h))

    def num_embeddings(self) -> int:
        return int(load_library().pb_index_num_embeddings(self._h))

    def num_partitions(self) -> int:
        return int(load_library().pb_index_num_partitions(self._h))

    def avg_doclen(self) -> float:
        return float(load_library().pb_index_avg_doclen(self._h))

    def embedding_dim(self) -> int:
        return int(load_library().pb_index_embedding_dim(self._h))

    def nbits(self) -> int:
        return int(load_library().pb_index_nbits(self._h))

    def memory_usage(self) -> dict:
        """pb_index_memory: bytes the index arrays hold on the device and in pinned host memory (workspaces excluded)."""
        dev, host = C.c_int64(), C.c_int64()
        _check(load_library().pb_index_memory(self._h, C.byref(dev), C.byref(host)))
        return dict(device_bytes=int(dev.value), host_bytes=int(host.value))

    # -- incremental append (index.rs:1675 update_append + reload) ------------------------------------
    def append(self, embeddings: Sequence[np.ndarray], codec: "ResidualCodec", index_dir: Optional[str] = None,
               batch_size: int = 50_000) -> List[int]:
        """MmapIndex::update_append + reload (pb_index_append): encodes the documents on the device with `codec` (the
        index's centroids and bucket cutoffs) and appends them; with `index_dir` also applies update_index's file
        changes to that directory (chunks of `batch_size` docs).  Returns the assigned doc ids."""
        dl = np.array([e.shape[0] for e in embeddings], np.int64)
        dim = self.embedding_dim()
        flat = (np.ascontiguousarray(np.concatenate(embeddings, 0), np.float32) if len(embeddings)
                else np.zeros((0, dim), np.float32))
        first = C.c_int64()
        _check(load_library().pb_index_append(self._h, codec._h, _ptr(flat), _ptr(dl), len(dl), 0,
                                              None if index_dir is None else os.fsencode(index_dir), batch_size,
                                              C.byref(first)))
        return list(range(first.value, first.value + len(dl)))

    def append_encoded(self, codes: np.ndarray, residuals: np.ndarray, doc_lengths: Sequence[int]) -> List[int]:
        """pb_index_append_encoded: documents already encoded (codes i64 [n], packed residuals u8 [n, dim*nbits/8])."""
        cd = np.ascontiguousarray(codes, np.int64)
        rs = np.ascontiguousarray(residuals, np.uint8)
        dl = np.ascontiguousarray(doc_lengths, np.int64)
        if rs.size != len(cd) * self.embedding_dim() * self.nbits() // 8 or int(dl.sum()) != len(cd):
            raise PlaidError(PB_ERR_INVALID, f"codes {cd.shape}, residuals {rs.shape} and doc_lengths (sum "
                                             f"{int(dl.sum())}) do not describe the same tokens")
        first = C.c_int64()
        _check(load_library().pb_index_append_encoded(self._h, _ptr(cd), _ptr(rs), _ptr(dl), len(dl), 0, C.byref(first)))
        return list(range(first.value, first.value + len(dl)))

    def reserve(self, num_documents: int, num_embeddings: int):
        """pb_index_reserve: capacity for appends up to these totals without reallocation."""
        _check(load_library().pb_index_reserve(self._h, num_documents, num_embeddings))

    # -- incremental delete (index.rs:1805 delete_with_options + reload) --------------------------------
    def delete(self, doc_ids: Sequence[int], index_dir: Optional[str] = None) -> int:
        """MmapIndex::delete + reload (pb_index_delete): removes these documents (the ids search returns; ids outside
        the index, negative and repeated ids are ignored) and renumbers the rest in order; with `index_dir` also
        applies delete_from_index's file changes to that directory.  Returns the number of documents removed."""
        ids = np.ascontiguousarray(doc_ids, np.int64).reshape(-1)
        n = C.c_int64()
        _check(load_library().pb_index_delete(self._h, _ptr(ids), len(ids),
                                              None if index_dir is None else os.fsencode(index_dir), C.byref(n)))
        return int(n.value)

    def last_delete_ms(self) -> dict:
        """Device time of the last delete, with set_profiling(True): compaction, inverted file, norm pass (ms)."""
        v = np.zeros(3, np.float32)
        _check(load_library().pb_last_delete_ms(self._h, _ptr(v)))
        return dict(compact_ms=float(v[0]), ivf_ms=float(v[1]), norms_ms=float(v[2]))

    # -- search ------------------------------------------------------------------------------
    def search(self, query: np.ndarray, params: SearchParameters,
               subset: Optional[Sequence[int]] = None) -> QueryResult:
        """MmapIndex::search (index.rs:1258), pb_search: one query per call.  The call releases the GIL, so with
        set_coalescing the searches of concurrent Python threads share batches."""
        q = np.asarray(query)
        if q.ndim != 2 or q.shape[1] != self.embedding_dim():
            raise PlaidError(PB_ERR_INVALID, f"query has shape {q.shape}, expected [tokens, {self.embedding_dim()}]")
        q = np.ascontiguousarray(q, np.float32)
        ss = None if subset is None else np.ascontiguousarray(subset, np.int64).reshape(-1)
        k = max(int(params.top_k), 1)
        ids, sc, cn = np.zeros(k, np.int64), np.zeros(k, np.float32), C.c_int32()
        p = params._c()
        _check(load_library().pb_search(self._h, _ptr(q), q.shape[0], C.byref(p), _ptr(ss),
                                        0 if ss is None else len(ss), _ptr(ids), _ptr(sc), C.byref(cn)))
        return QueryResult(0, ids[:cn.value].copy(), sc[:cn.value].copy())

    def set_coalescing(self, max_queries: int, max_wait_us: int = 0, max_inflight: int = 2):
        """pb_index_set_coalescing: merge the `search` calls of concurrent threads into batches of up to max_queries
        (1 = off), with at most max_inflight batches running at once; a leader whose batch is short waits up to
        max_wait_us for more requests (0 = never)."""
        c = _CoalesceConfig(int(max_queries), int(max_wait_us), int(max_inflight))
        _check(load_library().pb_index_set_coalescing(self._h, C.byref(c)))

    def coalesce_stats(self, reset: bool = False) -> dict:
        """pb_index_coalesce_stats: the counters of the handle's request queue (batch_hist: merged batches of size
        1, 2, 3-4, 5-8, 9-16, 17-32, 33-64, > 64)."""
        st = _CoalesceStats()
        _check(load_library().pb_index_coalesce_stats(self._h, C.byref(st), 1 if reset else 0))
        out = {n: int(getattr(st, n)) for n, _ in _CoalesceStats._fields_ if n != "batch_hist"}
        out["batch_hist"] = [int(v) for v in st.batch_hist]
        return out

    def search_batch(self, queries: Sequence[np.ndarray], params: SearchParameters,
                     parallel: bool = True, subset: Optional[Sequence[int]] = None,
                     trace: bool = False):
        """MmapIndex::search_batch (index.rs:1279).  `parallel` is accepted for signature parity;
        the GPU always processes the batch together."""
        L = load_library()
        ss = None if subset is None else np.ascontiguousarray(subset, np.int64)
        return self._search(queries, params, trace, ss is not None,
                            lambda flat, offs, B, p, ids, sc, cn, tr: L.pb_search_batch_traced(
                                self._h, _ptr(flat), _ptr(offs), B, p, _ptr(ss), 0 if ss is None else len(ss),
                                _ptr(ids), _ptr(sc), _ptr(cn), tr))

    def search_batch_subsets(self, queries: Sequence[np.ndarray], params: SearchParameters,
                             subsets: Sequence[Optional[Sequence[int]]], trace: bool = False):
        """pb_search_batch_subsets: search_batch with its own Option<&[i64]> subset per query (None: no filter, []:
        nothing eligible).  Result i equals search_batch([queries[i]], params, subset=subsets[i])[0]."""
        L = load_library()
        so, si, has = _subset_args(subsets, len(queries))
        return self._search(queries, params, trace, bool(has.any()),
                            lambda flat, offs, B, p, ids, sc, cn, tr: L.pb_search_batch_subsets(
                                self._h, _ptr(flat), _ptr(offs), B, p, _ptr(so), _ptr(si), _ptr(has),
                                _ptr(ids), _ptr(sc), _ptr(cn), tr))

    def search_batch_params(self, queries: Sequence[np.ndarray], params: Sequence[SearchParameters],
                            subsets: Optional[Sequence[Optional[Sequence[int]]]] = None, trace: bool = False):
        """pb_search_batch_params: search_batch_subsets with its own SearchParameters per query.  Result i equals
        search_batch([queries[i]], params[i], subset=subsets[i])[0], cut to its own count."""
        L = load_library()
        params = list(params)
        if len(params) != len(queries):
            raise PlaidError(PB_ERR_INVALID, f"{len(params)} parameter sets for {len(queries)} queries")
        so, si, has = _subset_args(subsets, len(queries))
        return self._search(queries, params, trace, bool(has.any()),
                            lambda flat, offs, B, p, ids, sc, cn, tr: L.pb_search_batch_params(
                                self._h, _ptr(flat), _ptr(offs), B, p, None if subsets is None else _ptr(so),
                                _ptr(si), _ptr(has), _ptr(ids), _ptr(sc), _ptr(cn), tr))

    def _search(self, queries, params, trace, any_subset, invoke):
        """the outputs (and trace buffers) of one search call; invoke(flat, offs, B, params, ids, scores, counts,
        trace pointer) makes the call.  params: one SearchParameters, or a list of one per query"""
        flat, offs = _pack_queries(queries, self.embedding_dim())
        plist = params if isinstance(params, list) else [params]
        B, k = len(queries), max([int(q.top_k) for q in plist] + [0])
        ids = np.zeros((B, max(k, 1)), np.int64)
        sc = np.zeros((B, max(k, 1)), np.float32)
        cn = np.zeros(B, np.int32)
        if isinstance(params, list):
            p = (_Params * max(B, 1))(*[q._c() for q in params])
            p_arg = C.cast(p, C.POINTER(_Params)) if B else None
        else:
            p = params._c()
            p_arg = C.byref(p)
        tr, bufs = None, None
        if trace:
            D, K = self.num_documents(), self.num_partitions()
            M = max([min(q.n_full_scores, max(q.n_full_scores // 4, q.top_k)) for q in plist] + [1])
            n_probe = max([max(q.n_ivf_probe, 1) for q in plist] + [1])
            cc = min(K, max(int(offs[-1]) * n_probe, 1)) if not any_subset else K
            bufs = dict(cells=np.zeros((B, cc), np.int64), n_cells=np.zeros(B, np.int32),
                        cand=np.zeros((B, max(D, 1)), np.int64), approx=np.zeros((B, max(D, 1)), np.float32),
                        n_cand=np.zeros(B, np.int32), kept=np.zeros((B, M), np.int64),
                        kex=np.zeros((B, M), np.float32), n_kept=np.zeros(B, np.int32))
            tr = _Trace(_ptr(bufs["cells"]), _ptr(bufs["n_cells"]), cc, _ptr(bufs["cand"]),
                        _ptr(bufs["approx"]), _ptr(bufs["n_cand"]), max(D, 1), _ptr(bufs["kept"]),
                        _ptr(bufs["kex"]), _ptr(bufs["n_kept"]), M)
        _check(invoke(flat, offs, B, p_arg, ids, sc, cn, None if tr is None else C.cast(C.pointer(tr), C.c_void_p)))
        res = [QueryResult(i, ids[i, :cn[i]].copy(), sc[i, :cn[i]].copy()) for i in range(B)]
        if trace:
            t = SearchTrace(
                [bufs["cells"][i, :bufs["n_cells"][i]].copy() for i in range(B)],
                [bufs["cand"][i, :bufs["n_cand"][i]].copy() for i in range(B)],
                [bufs["approx"][i, :bufs["n_cand"][i]].copy() for i in range(B)],
                [bufs["kept"][i, :bufs["n_kept"][i]].copy() for i in range(B)],
                [bufs["kex"][i, :bufs["n_kept"][i]].copy() for i in range(B)])
            return res, t
        return res

    # -- stage entry points --------------------------------------------------------------------
    def centroid_scores(self, query_tokens: np.ndarray) -> np.ndarray:
        """Stage 1, S = Q.C^T (search.rs:345), [n_tokens, K]."""
        q = np.ascontiguousarray(query_tokens, np.float32)
        out = np.zeros((q.shape[0], self.num_partitions()), np.float32)
        _check(load_library().pb_centroid_scores(self._h, _ptr(q), q.shape[0], _ptr(out)))
        return out

    def decompress_documents(self, doc_ids: Sequence[int]):
        """MmapIndex::decompress_documents (index.rs:1197): (embeddings [sum len, dim], lengths)."""
        L = load_library()
        ids = np.ascontiguousarray(doc_ids, np.int64)
        lens = np.zeros(len(ids), np.int64)
        _check(L.pb_decompress_documents(self._h, _ptr(ids), len(ids), None, _ptr(lens)))
        emb = np.zeros((int(lens.sum()), self.embedding_dim()), np.float32)
        if emb.shape[0]:
            _check(L.pb_decompress_documents(self._h, _ptr(ids), len(ids), _ptr(emb), _ptr(lens)))
        return emb, lens

    def get_document_embeddings(self, doc_id: int) -> np.ndarray:
        """MmapIndex::get_document_embeddings (index.rs:1159)."""
        if not (0 <= doc_id < self.num_documents()):
            raise PlaidError(PB_ERR_INVALID, f"Invalid document ID: {doc_id}")
        return self.decompress_documents([doc_id])[0]

    def exhaustive_scores(self, queries: Sequence[np.ndarray]) -> np.ndarray:
        """Exact MaxSim of each query against every document (recall ground truth)."""
        flat, offs = _pack_queries(queries, self.embedding_dim())
        out = np.zeros((len(queries), self.num_documents()), np.float32)
        _check(load_library().pb_exhaustive_scores(self._h, _ptr(flat), _ptr(offs), len(queries), _ptr(out)))
        return out

    # -- doc-sharded deployment ------------------------------------------------------------------
    def comm_init(self, unique_id: bytes, rank: int, world: int):
        """pb_index_comm_init: after this, search_batch is a collective over `world` ranks."""
        buf = np.frombuffer(bytes(unique_id), np.uint8).copy()
        assert buf.size == 128
        _check(load_library().pb_index_comm_init(self._h, _ptr(buf), rank, world))
        self._world = world

    def rebalance_sharded(self, bounds: Optional[Sequence[int]] = None) -> np.ndarray:
        """pb_index_rebalance_sharded, this rank's part of the collective: every rank calls it with the same `bounds`
        ([world + 1] document bounds, or None for the token-balanced split).  Returns the bounds applied."""
        W = self._world
        b = None
        if bounds is not None:
            b = np.ascontiguousarray(bounds, np.int64).reshape(-1)
            if b.size != W + 1:
                raise PlaidError(PB_ERR_INVALID, f"bounds has {b.size} entries, the deployment needs {W + 1}")
        out = np.zeros(W + 1, np.int64)
        _check(load_library().pb_index_rebalance_sharded(self._h, _ptr(b), _ptr(out)))
        return out

    # -- measurement hooks -------------------------------------------------------------------------
    def set_fast_approx(self, mode):
        """0/False = single exact pass over every candidate, 1/True = two-pass (default)."""
        load_library().pb_set_fast_approx(self._h, int(mode))

    def set_scores_tc(self, on: bool):
        """a2 on the tensor cores (default on) vs the dense fp32 kernel; same results either way."""
        load_library().pb_set_scores_tc(self._h, 1 if on else 0)

    def set_fast_exact(self, on: bool):
        """wgmma certified filter in front of the exact stage (default on); same results either way."""
        load_library().pb_set_fast_exact(self._h, 1 if on else 0)

    def set_profiling(self, on: bool):
        load_library().pb_set_profiling(self._h, 1 if on else 0)

    def set_lanes(self, lanes: int):
        """Slices of a batch searched concurrently inside one call (pb_set_lanes); 1 = off."""
        load_library().pb_set_lanes(self._h, int(lanes))

    def last_stage_stats(self):
        ms = np.zeros(len(STAGES), np.float32)
        ln = np.zeros(len(STAGES), np.int32)
        _check(load_library().pb_last_stage_stats(self._h, _ptr(ms), _ptr(ln)))
        return dict(zip(STAGES, ms.tolist())), dict(zip(STAGES, ln.tolist()))

    def export_ivf(self):
        """pb_index_export_ivf: (ivf <i8 global doc ids, ivf_lengths <i4), what create_index writes to ivf.npy /
        ivf_lengths.npy (index.rs:501-508)."""
        L = load_library()
        tot = C.c_int64()
        _check(L.pb_index_export_ivf(self._h, None, None, C.byref(tot)))
        ivf = np.zeros(max(tot.value, 1), np.int64)
        lens = np.zeros(self.num_partitions(), np.int32)
        _check(L.pb_index_export_ivf(self._h, _ptr(ivf), _ptr(lens), C.byref(tot)))
        return ivf[:tot.value], lens

    def last_call_ms(self) -> float:
        v = np.zeros(1, np.float32)
        _check(load_library().pb_last_call_ms(self._h, _ptr(v)))
        return float(v[0])

    def last_kernel_ms(self) -> dict:
        v = np.zeros(4, np.float32)
        _check(load_library().pb_last_kernel_ms(self._h, _ptr(v)))
        return dict(zip(("scores", "approx16", "filter", "exact"), v.tolist()))

    def last_work_counters(self) -> dict:
        w = _Work()
        _check(load_library().pb_last_work_counters(self._h, C.byref(w)))
        return {n: int(getattr(w, n)) for n, _ in _Work._fields_}

    def last_staging_stats(self) -> dict:
        """pb_last_staging_stats: docs and residual bytes the calling thread's last search staged from host memory (0 on
        a resident handle), and their staging time in ms (with set_profiling(True))."""
        docs, nbytes, ms = C.c_int64(), C.c_int64(), C.c_float()
        _check(load_library().pb_last_staging_stats(self._h, C.byref(docs), C.byref(nbytes), C.byref(ms)))
        return dict(docs=int(docs.value), bytes=int(nbytes.value), ms=float(ms.value))

    def search_batch_device(self, d_queries_ptr: int, q_tok_offsets: np.ndarray, params: SearchParameters,
                            d_ids_ptr: int, d_scores_ptr: int, d_counts_ptr: int):
        """pb_search_batch_device: queries and results stay on the device (kernel-only timing)."""
        offs = np.ascontiguousarray(q_tok_offsets, np.int64)
        p = params._c()
        _check(load_library().pb_search_batch_device(self._h, d_queries_ptr, _ptr(offs), len(offs) - 1,
                                                     C.byref(p), d_ids_ptr, d_scores_ptr, d_counts_ptr))


def maxsim_scores(query: np.ndarray, docs: Sequence[np.ndarray], device: int = 0) -> np.ndarray:
    """maxsim::maxsim_score (maxsim.rs:270) for a list of already-decompressed documents."""
    q = np.ascontiguousarray(query, np.float32)
    offs = np.zeros(len(docs) + 1, np.int64)
    for i, d in enumerate(docs):
        offs[i + 1] = offs[i] + d.shape[0]
    flat = np.zeros((int(offs[-1]), q.shape[1]), np.float32)
    for i, d in enumerate(docs):
        flat[offs[i]:offs[i + 1]] = d
    out = np.zeros(len(docs), np.float32)
    _check(load_library().pb_maxsim_scores(device, _ptr(q), q.shape[0], q.shape[1], _ptr(flat), _ptr(offs),
                                           len(docs), _ptr(out)))
    return out


class _CreateParams(C.Structure):
    _fields_ = [("nbits", C.c_int32), ("kmeans_niters", C.c_int32), ("max_points_per_centroid", C.c_int32),
                ("device", C.c_int32), ("num_partitions", C.c_int64), ("batch_size", C.c_int64), ("seed", C.c_uint64)]


def create_index(embeddings: Sequence[np.ndarray], index_dir: str, nbits: int = 4, kmeans_niters: int = 4,
                 num_partitions: int = 0, batch_size: int = 50_000, seed: int = 42, device: int = 0,
                 max_points_per_centroid: int = 256) -> "MmapIndex":
    """MmapIndex::create_with_kmeans (index.rs:1392): builds the reference's index directory from document embeddings
    on the GPU (pb_create_index) and returns the open index."""
    L = load_library()
    dl = np.array([e.shape[0] for e in embeddings], np.int64)
    flat = np.ascontiguousarray(np.concatenate(embeddings, 0), np.float32)
    p = _CreateParams(nbits, kmeans_niters, max_points_per_centroid, device, num_partitions, batch_size, seed)
    h = C.c_void_p()
    _check(L.pb_create_index(_ptr(flat), _ptr(dl), len(dl), flat.shape[1], C.byref(p), index_dir.encode(), C.byref(h)))
    return MmapIndex(h.value)


def kmeans_fit_dp(shards: Sequence[np.ndarray], K: int, niters: int = 4, seed: int = 42, device: int = 0,
                  nccl: Optional[tuple] = None) -> np.ndarray:
    """pb_kmeans_fit_dp.  Without `nccl`: the shards are fitted by len(shards) host threads of this process through an
    in-process shard group (all on `device`); with nccl = (unique_id, rank, world) the single shard shards[0] is this
    rank's part of an NCCL job.  Returns the centroids (identical on every rank)."""
    L = load_library()
    dim = shards[0].shape[1]
    if nccl is not None:
        uid, rank, world = nccl
        buf = np.frombuffer(bytes(uid), np.uint8).copy()
        h = C.c_void_p()
        _check(L.pb_build_comm_init(_ptr(buf), rank, world, device, C.byref(h)))
        x = np.ascontiguousarray(shards[0], np.float32)
        out = np.zeros((K, dim), np.float32)
        try:
            _check(L.pb_kmeans_fit_dp(h, _ptr(x), x.shape[0], dim, K, niters, seed, _ptr(out)))
        finally:
            L.pb_build_comm_destroy(h)
        return out
    G = len(shards)
    g = C.c_void_p()
    _check(L.pb_shard_group_create(G, C.byref(g)))

    def run(r):
        h = C.c_void_p()
        _check(L.pb_build_comm_group(g, r, device, C.byref(h)))
        x = np.ascontiguousarray(shards[r], np.float32)
        out = np.zeros((K, dim), np.float32)
        try:
            _check(L.pb_kmeans_fit_dp(h, _ptr(x), x.shape[0], dim, K, niters, seed, _ptr(out)))
        finally:
            L.pb_build_comm_destroy(h)
        return out
    try:
        outs = _per_rank(G, run)
    finally:
        L.pb_shard_group_destroy(g)
    for o in outs[1:]:
        assert np.array_equal(o, outs[0]), "ranks disagree on the centroids"
    return outs[0]


def kmeans_sizing(num_documents: int, avg_sample_doclen: float, num_sample_tokens: int, num_embeddings: int) -> dict:
    """The sizing rules of compute_kmeans (kmeans.rs:273-312) and prepare_codec_artifacts (index.rs:195-212)."""
    L = load_library()
    return {"kmeans_sample_docs": int(L.pb_kmeans_num_sample_docs(num_documents)),
            "num_partitions": int(L.pb_kmeans_num_partitions(num_documents, float(avg_sample_doclen), num_sample_tokens)),
            "codec_sample_docs": int(L.pb_codec_num_sample_docs(num_documents)),
            "heldout_tokens": int(L.pb_codec_heldout_tokens(num_embeddings))}


class ResidualCodec:
    """Device-resident next_plaid::ResidualCodec (codec.rs:107-123) for the index-build path."""

    def __init__(self, nbits: int, centroids: np.ndarray, bucket_cutoffs: Optional[np.ndarray] = None,
                 device: int = 0):
        cen = np.ascontiguousarray(centroids, np.float32)
        cut = None if bucket_cutoffs is None else np.ascontiguousarray(bucket_cutoffs, np.float32)
        h = C.c_void_p()
        _check(load_library().pb_codec_open(device, _ptr(cen), cen.shape[0], cen.shape[1], nbits, _ptr(cut),
                                            C.byref(h)))
        self._h, self.nbits, self.dim = h, nbits, cen.shape[1]

    def close(self):
        if self._h:
            load_library().pb_codec_close(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def last_assign_stats(self) -> dict:
        n, f, tc = C.c_int64(), C.c_int64(), C.c_int32()
        _check(load_library().pb_codec_last_assign_stats(self._h, C.byref(n), C.byref(f), C.byref(tc)))
        return {"tokens": n.value, "exact_fallback": f.value, "tensor_cores": bool(tc.value)}

    def compress_into_codes(self, embeddings: np.ndarray) -> np.ndarray:
        """codec.rs:260."""
        e = np.ascontiguousarray(embeddings, np.float32)
        out = np.zeros(e.shape[0], np.int64)
        _check(load_library().pb_codec_compress_into_codes(self._h, _ptr(e), e.shape[0], _ptr(out)))
        return out

    def compress_and_residuals(self, embeddings: np.ndarray):
        """index.rs:17-40."""
        e = np.ascontiguousarray(embeddings, np.float32)
        codes = np.zeros(e.shape[0], np.int64)
        res = np.zeros_like(e)
        _check(load_library().pb_codec_compress_and_residuals(self._h, _ptr(e), e.shape[0], _ptr(codes), _ptr(res)))
        return codes, res

    def find_outliers(self, embeddings: np.ndarray, threshold_sq: float) -> np.ndarray:
        """update.rs:490: row indices farther than sqrt(threshold_sq) from every centroid."""
        e = np.ascontiguousarray(embeddings, np.float32)
        out = np.zeros(max(e.shape[0], 1), np.int64)
        cnt = C.c_int64()
        _check(load_library().pb_codec_find_outliers(self._h, _ptr(e), e.shape[0], float(threshold_sq), _ptr(out),
                                                     C.byref(cnt)))
        return out[:cnt.value].copy()

    def train(self, heldout: np.ndarray):
        """pb_codec_train (prepare_codec_artifacts, index.rs:228-287, on held-out rows the caller sampled):
        (bucket_cutoffs, bucket_weights, avg_residual, cluster_threshold); the codec keeps the cutoffs."""
        e = np.ascontiguousarray(heldout, np.float32).reshape(-1, self.dim)
        nopt = 1 << self.nbits
        cut, wts, avg = np.zeros(max(nopt - 1, 1), np.float32), np.zeros(nopt, np.float32), np.zeros(self.dim, np.float32)
        thr = C.c_float()
        _check(load_library().pb_codec_train(self._h, _ptr(e), e.shape[0], _ptr(cut), _ptr(wts), _ptr(avg), C.byref(thr)))
        return cut[:nopt - 1], wts, avg, float(thr.value)

    def encode_chunk(self, embeddings: np.ndarray):
        """encode_index_chunk (index.rs:289): (codes i64 [n], packed residuals u8 [n, dim*nbits/8])."""
        e = np.ascontiguousarray(embeddings, np.float32)
        codes = np.zeros(e.shape[0], np.int64)
        packed = np.zeros((e.shape[0], self.dim * self.nbits // 8), np.uint8)
        _check(load_library().pb_codec_encode_chunk(self._h, _ptr(e), e.shape[0], _ptr(codes), _ptr(packed)))
        return codes, packed


def kmeans_fit(samples: np.ndarray, num_centroids: int, niters: int = 4, seed: int = 42, device: int = 0) -> np.ndarray:
    """The fit inside compute_kmeans (kmeans.rs:319-419): Lloyd iterations + L2 normalisation."""
    x = np.ascontiguousarray(samples, np.float32)
    out = np.zeros((num_centroids, x.shape[1]), np.float32)
    _check(load_library().pb_kmeans_fit(device, _ptr(x), x.shape[0], x.shape[1], num_centroids, niters, seed, _ptr(out)))
    return out
