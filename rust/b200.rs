//! next-plaid/src/b200.rs -- binding of libplaid_b200 (include/plaid_b200.h) for the `b200` cargo
//! feature.  NOT COMPILED IN THIS REPOSITORY'S CI: the build image has no cargo/rustc.  It is the
//! shim a next-plaid maintainer adds so that `MmapIndex::{load, search, search_batch}` keep their
//! signatures (index.rs:1026, :1258, :1279) while the work runs on an H100; `colgrep` and
//! `next-plaid-api` link unchanged because they only see `MmapIndex`.
#![cfg(feature = "b200")]

use std::ffi::{c_char, c_void, CStr, CString};
use std::os::raw::c_int;

use ndarray::Array2;

use crate::error::{Error, Result};
use crate::search::{QueryResult, SearchParameters};

#[repr(C)]
pub struct PbSearchParams {
    pub batch_size: i64,
    pub n_full_scores: i64,
    pub top_k: i64,
    pub n_ivf_probe: i64,
    pub centroid_batch_size: i64,
    pub has_centroid_score_threshold: i32,
    pub centroid_score_threshold: f32,
}

impl From<&SearchParameters> for PbSearchParams {
    fn from(p: &SearchParameters) -> Self {
        PbSearchParams {
            batch_size: p.batch_size as i64,
            n_full_scores: p.n_full_scores as i64,
            top_k: p.top_k as i64,
            n_ivf_probe: p.n_ivf_probe as i64,
            centroid_batch_size: p.centroid_batch_size as i64,
            has_centroid_score_threshold: p.centroid_score_threshold.is_some() as i32,
            centroid_score_threshold: p.centroid_score_threshold.unwrap_or(0.0),
        }
    }
}

/// `pb_coalesce_config`
/// `pb_row_cache_stats`: a host-tier handle's device row cache (DESIGN §4s)
#[repr(C)]
#[derive(Default, Debug, Clone, Copy)]
pub struct PbRowCacheStats {
    pub budget_bytes: i64,
    pub cached_docs: i64,
    pub cached_bytes: i64,
    /// rows of docs deleted since the fill
    pub dead_bytes: i64,
    /// search staging since the last reset
    pub staged_docs: i64,
    pub hit_docs: i64,
    pub hit_bytes: i64,
    pub last_fill_ms: f32,
}

#[repr(C)]
struct PbCoalesceConfig {
    max_queries: i32,
    max_wait_us: i32,
    max_inflight: i32,
}

#[link(name = "plaid_b200")]
extern "C" {
    fn pb_pooled_doc_length(n_tokens: i64, pool_factor: i64) -> i64;
    fn pb_pool_embeddings(device: i32, embeddings: *const f32, doc_lengths: *const i64, n_docs: i64, dim: i32,
                          pool_factor: i64, memory_space: i32, out_embeddings: *mut f32, out_doc_lengths: *mut i64)
                          -> c_int;
    fn pb_index_load(index_dir: *const c_char, device: i32, out: *mut *mut c_void) -> c_int;
    fn pb_index_close(ix: *mut c_void);
    fn pb_index_embedding_dim(ix: *const c_void) -> i32;
    fn pb_index_device(ix: *const c_void) -> i32;
    fn pb_search_batch(
        ix: *mut c_void,
        queries: *const f32,
        q_tok_offsets: *const i64,
        n_queries: i64,
        params: *const PbSearchParams,
        subset: *const i64,
        n_subset: i64,
        out_ids: *mut i64,
        out_scores: *mut f32,
        out_counts: *mut i32,
    ) -> c_int;
    fn pb_search_batch_subsets(
        ix: *mut c_void,
        queries: *const f32,
        q_tok_offsets: *const i64,
        n_queries: i64,
        params: *const PbSearchParams,
        subset_offsets: *const i64,
        subset_ids: *const i64,
        has_subset: *const u8,
        out_ids: *mut i64,
        out_scores: *mut f32,
        out_counts: *mut i32,
        trace: *mut c_void,
    ) -> c_int;
    fn pb_search_batch_params(
        ix: *mut c_void,
        queries: *const f32,
        q_tok_offsets: *const i64,
        n_queries: i64,
        params: *const PbSearchParams, // [n_queries]
        subset_offsets: *const i64,
        subset_ids: *const i64,
        has_subset: *const u8,
        out_ids: *mut i64, // row i at i * max top_k
        out_scores: *mut f32,
        out_counts: *mut i32,
        trace: *mut c_void,
    ) -> c_int;
    fn pb_search(
        ix: *mut c_void,
        query: *const f32,
        n_query_tokens: i64,
        params: *const PbSearchParams,
        subset: *const i64,
        n_subset: i64,
        out_ids: *mut i64, // [top_k]
        out_scores: *mut f32,
        out_count: *mut i32,
    ) -> c_int;
    fn pb_index_set_coalescing(ix: *mut c_void, cfg: *const PbCoalesceConfig) -> c_int;
    fn pb_last_error() -> *const c_char;
    fn pb_codec_open(device: i32, centroids: *const f32, k: i64, dim: i32, nbits: i32, cutoffs: *const f32,
                     out: *mut *mut c_void) -> c_int;
    fn pb_codec_close(c: *mut c_void);
    fn pb_index_append(ix: *mut c_void, codec: *mut c_void, embeddings: *const f32, doc_lengths: *const i64,
                       n_docs: i64, memory_space: i32, index_dir: *const c_char, batch_size: i64,
                       out_first_doc_id: *mut i64) -> c_int;
    fn pb_index_append_encoded(ix: *mut c_void, codes: *const i64, residuals: *const u8, doc_lengths: *const i64,
                               n_docs: i64, memory_space: i32, out_first_doc_id: *mut i64) -> c_int;
    fn pb_index_reserve(ix: *mut c_void, num_documents: i64, num_embeddings: i64) -> c_int;
    fn pb_index_delete(ix: *mut c_void, doc_ids: *const i64, n_ids: i64, index_dir: *const c_char,
                       out_deleted: *mut i64) -> c_int;
    fn pb_index_load_range(index_dir: *const c_char, device: i32, doc_begin: i64, doc_end: i64,
                           out: *mut *mut c_void) -> c_int;
    fn pb_index_dir_shard_bounds(index_dir: *const c_char, world: i32, out_bounds: *mut i64) -> c_int;
    fn pb_index_delete_sharded(ix: *mut c_void, doc_ids: *const i64, n_ids: i64, index_dir: *const c_char,
                               out_deleted: *mut i64) -> c_int;
    fn pb_index_append_sharded(ix: *mut c_void, codec: *mut c_void, embeddings: *const f32, doc_lengths: *const i64,
                               n_docs: i64, memory_space: i32, index_dir: *const c_char, batch_size: i64,
                               out_first_doc_id: *mut i64) -> c_int;
    fn pb_index_append_encoded_sharded(ix: *mut c_void, codes: *const i64, residuals: *const u8,
                                       doc_lengths: *const i64, n_docs: i64, memory_space: i32,
                                       out_first_doc_id: *mut i64) -> c_int;
    fn pb_index_rebalance_sharded(ix: *mut c_void, bounds: *const i64, out_bounds: *mut i64) -> c_int;
    fn pb_index_load_range_flags(index_dir: *const c_char, device: i32, doc_begin: i64, doc_end: i64, flags: i32,
                                 out: *mut *mut c_void) -> c_int;
    fn pb_index_load_devices(index_dir: *const c_char, devices: *const i32, n_devices: i32, flags: i32,
                             out: *mut *mut c_void) -> c_int;
    fn pb_index_shard_layout(ix: *const c_void, out_world: *mut i32, out_bounds: *mut i64, out_devices: *mut i32) -> c_int;
    fn pb_index_add_devices(ix: *mut c_void, devices: *const i32, n_devices: i32, bounds: *const i64,
                            out_bounds: *mut i64) -> c_int;
    fn pb_index_remove_ranks(ix: *mut c_void, ranks: *const i32, n_ranks: i32, bounds: *const i64,
                             out_bounds: *mut i64) -> c_int;
    fn pb_index_load_replicas(index_dir: *const c_char, devices: *const i32, n_devices: i32, n_shards: i32, flags: i32,
                              out: *mut *mut c_void) -> c_int;
    fn pb_index_add_replicas(ix: *mut c_void, devices: *const i32, n_devices: i32) -> c_int;
    fn pb_index_remove_replicas(ix: *mut c_void, replicas: *const i32, n_replicas: i32) -> c_int;
    fn pb_index_memory(ix: *const c_void, device_bytes: *mut i64, host_bytes: *mut i64) -> c_int;
    fn pb_last_staging_stats(ix: *mut c_void, docs: *mut i64, bytes: *mut i64, ms: *mut f32) -> c_int;
    fn pb_index_set_row_cache(ix: *mut c_void, max_bytes: i64) -> c_int;
    fn pb_index_fill_row_cache(ix: *mut c_void, doc_ids: *const i64, n_ids: i64, out_ids: *mut i64, out_cap: i64,
                               out_n: *mut i64) -> c_int;
    fn pb_index_row_cache_stats(ix: *mut c_void, out: *mut PbRowCacheStats, reset: i32) -> c_int;
    // pb_create_index_sharded (DESIGN §4n): `comm` is a pb_build_comm, `params` a pb_create_params
    fn pb_create_index_sharded(comm: *mut c_void, embeddings: *const f32, doc_lengths: *const i64, n_docs: i64, dim: i32,
                               memory_space: i32, centroids: *const f32, num_centroids: i64, params: *const c_void,
                               index_dir: *const c_char, out_shard: *mut *mut c_void, out_first_doc_id: *mut i64)
                               -> c_int;
}

/// pb_index_desc.flags: the packed residuals in pinned host memory, the kept docs' rows staged per search (DESIGN §4j).
pub const PB_OPEN_HOST_RESIDUALS: i32 = 2;
/// with `PB_OPEN_HOST_RESIDUALS` only: appends and deletes work on the host-tier handle (DESIGN §4r)
pub const PB_OPEN_HOST_MUTABLE: i32 = 4;

fn last_error() -> String {
    unsafe { CStr::from_ptr(pb_last_error()).to_string_lossy().into_owned() }
}

/// Device-resident twin of the mmap'd arrays of `MmapIndex` (index.rs:995-1016).
pub struct B200Index {
    handle: *mut c_void,
}

// The C library is re-entrant on one handle (per-call stream + workspace pool), which is what
// `ArcSwap<MmapIndex>` + tokio workers need (next-plaid-api/src/state.rs:24-47).
unsafe impl Send for B200Index {}
unsafe impl Sync for B200Index {}

impl B200Index {
    /// Called at the end of `MmapIndex::load` (index.rs:1127): same directory, no conversion.
    pub fn load(index_path: &str, device: i32) -> Result<Self> {
        let c = CString::new(index_path).map_err(|e| Error::IndexLoad(e.to_string()))?;
        let mut handle: *mut c_void = std::ptr::null_mut();
        let st = unsafe { pb_index_load(c.as_ptr(), device, &mut handle) };
        if st != 0 {
            // No CPU fallback on this path: behaves like NEXT_PLAID_FORCE_GPU (lib.rs:71-84).
            return Err(Error::IndexLoad(last_error()));
        }
        Ok(B200Index { handle })
    }

    /// `load` with the packed residuals in pinned host memory (`PB_OPEN_HOST_RESIDUALS`): same results, slower searches
    /// (the kept docs' rows cross PCIe), about 11 instead of 75 device bytes per token at 4 bits and dim 128.  Such a
    /// handle refuses appends and deletes.
    pub fn load_host_residuals(index_path: &str, device: i32) -> Result<Self> {
        let c = CString::new(index_path).map_err(|e| Error::IndexLoad(e.to_string()))?;
        let mut handle: *mut c_void = std::ptr::null_mut();
        if unsafe { pb_index_load_range_flags(c.as_ptr(), device, 0, -1, PB_OPEN_HOST_RESIDUALS, &mut handle) } != 0 {
            return Err(Error::IndexLoad(last_error()));
        }
        Ok(B200Index { handle })
    }

    /// `load` doc-sharded over several GPUs of this process (`pb_index_load_devices`, DESIGN §4o): rank r holds the
    /// r-th token-balanced document range on `devices[r]`, and the library keeps one thread per extra rank.  The
    /// handle is then used exactly as one from `load`: `search`, `search_batch`, `set_coalescing`, `update_append`
    /// and `delete_with_options` reach every rank in one order, results equal those of `load`.
    pub fn load_devices(index_path: &str, devices: &[i32]) -> Result<Self> {
        let c = CString::new(index_path).map_err(|e| Error::IndexLoad(e.to_string()))?;
        let mut handle: *mut c_void = std::ptr::null_mut();
        let st = unsafe { pb_index_load_devices(c.as_ptr(), devices.as_ptr(), devices.len() as i32, 0, &mut handle) };
        if st != 0 {
            return Err(Error::IndexLoad(last_error()));
        }
        Ok(B200Index { handle })
    }

    /// `devices.len() / shards` full copies of the index behind one handle (`pb_index_load_replicas`, DESIGN §4q):
    /// replica g on `devices[g * shards .. (g + 1) * shards]`, a `load` handle when `shards == 1`, else a `load_devices`
    /// deployment.  Searches are spread over the replicas, `update_append` and `delete_with_options` reach all of them
    /// at once (encoded once, the directory written once); results equal those of `load` / `load_devices`.
    pub fn load_replicas(index_path: &str, devices: &[i32], shards: i32) -> Result<Self> {
        let c = CString::new(index_path).map_err(|e| Error::IndexLoad(e.to_string()))?;
        let mut handle: *mut c_void = std::ptr::null_mut();
        let st = unsafe {
            pb_index_load_replicas(c.as_ptr(), devices.as_ptr(), devices.len() as i32, shards, 0, &mut handle)
        };
        if st != 0 {
            return Err(Error::IndexLoad(last_error()));
        }
        Ok(B200Index { handle })
    }

    /// Bytes the index arrays hold: (device, pinned host) -- for capacity planning on a shared GPU.
    pub fn memory_usage(&self) -> Result<(i64, i64)> {
        let (mut d, mut h) = (0i64, 0i64);
        if unsafe { pb_index_memory(self.handle, &mut d, &mut h) } != 0 {
            return Err(Error::Search(last_error()));
        }
        Ok((d, h))
    }

    /// The budget of the device row cache of a host-tier handle (`pb_index_set_row_cache`, DESIGN §4s); 0 = off.
    pub fn set_row_cache(&self, max_bytes: i64) -> Result<()> {
        if unsafe { pb_index_set_row_cache(self.handle, max_bytes) } != 0 {
            return Err(Error::Search(last_error()));
        }
        Ok(())
    }

    /// Replaces the cached set (`pb_index_fill_row_cache`): by the keep counts (`doc_ids` None) or with the given ids in
    /// order, each doc taken while its rows fit the budget.  Returns at most `cap` of the cached ids, in the order taken.
    pub fn fill_row_cache(&self, doc_ids: Option<&[i64]>, cap: usize) -> Result<Vec<i64>> {
        let mut out = vec![0i64; cap.max(1)];
        let mut n = 0i64;
        let (p, len) = doc_ids.map_or((std::ptr::null(), 0), |d| (d.as_ptr(), d.len() as i64));
        if unsafe { pb_index_fill_row_cache(self.handle, p, len, out.as_mut_ptr(), cap as i64, &mut n) } != 0 {
            return Err(Error::Search(last_error()));
        }
        out.truncate((n as usize).min(cap));
        Ok(out)
    }

    /// The row cache's budget and contents, and search staging since the last reset (`pb_index_row_cache_stats`).
    pub fn row_cache_stats(&self, reset: bool) -> Result<PbRowCacheStats> {
        let mut st = PbRowCacheStats::default();
        if unsafe { pb_index_row_cache_stats(self.handle, &mut st, reset as i32) } != 0 {
            return Err(Error::Search(last_error()));
        }
        Ok(st)
    }

    /// What this thread's last search staged from host memory: (docs, residual bytes, ms with profiling on).
    pub fn last_staging_stats(&self) -> (i64, i64, f32) {
        let (mut docs, mut bytes, mut ms) = (0i64, 0i64, 0f32);
        unsafe { pb_last_staging_stats(self.handle, &mut docs, &mut bytes, &mut ms) };
        (docs, bytes, ms)
    }

    /// Shard `rank` of `world` of the same directory for a doc-sharded deployment: the token-balanced document range
    /// of `pb_index_dir_shard_bounds`, loaded by `pb_index_load_range` (global ids; only that range's chunk rows are
    /// read).  Every rank then calls `pb_index_comm_init`.
    pub fn load_shard(index_path: &str, rank: i32, world: i32, device: i32) -> Result<Self> {
        if rank < 0 || rank >= world {
            return Err(Error::IndexLoad(format!("rank {} outside [0, {})", rank, world)));
        }
        let c = CString::new(index_path).map_err(|e| Error::IndexLoad(e.to_string()))?;
        let mut bounds = vec![0i64; world as usize + 1];
        if unsafe { pb_index_dir_shard_bounds(c.as_ptr(), world, bounds.as_mut_ptr()) } != 0 {
            return Err(Error::IndexLoad(last_error()));
        }
        let (b, e) = (bounds[rank as usize], bounds[rank as usize + 1]);
        let mut handle: *mut c_void = std::ptr::null_mut();
        if unsafe { pb_index_load_range(c.as_ptr(), device, b, e, &mut handle) } != 0 {
            return Err(Error::IndexLoad(last_error()));
        }
        Ok(B200Index { handle })
    }

    /// Body of `MmapIndex::search_batch` (index.rs:1279) under the `b200` feature.
    pub fn search_batch(
        &self,
        queries: &[Array2<f32>],
        params: &SearchParameters,
        subset: Option<&[i64]>,
    ) -> Result<Vec<QueryResult>> {
        // pb_search_batch has no dim argument and reads rows * embedding_dim floats: reject a query of another
        // width here, as the Python binding does (Error::Shape, not an out-of-bounds host read)
        let dim = unsafe { pb_index_embedding_dim(self.handle) } as usize;
        let mut offsets = Vec::with_capacity(queries.len() + 1);
        offsets.push(0i64);
        let mut flat: Vec<f32> = Vec::new();
        for q in queries {
            if q.ncols() != dim {
                return Err(Error::Shape(format!("query has {} columns, the index embedding_dim is {}", q.ncols(), dim)));
            }
            flat.extend(q.as_standard_layout().iter());
            offsets.push(offsets.last().unwrap() + q.nrows() as i64);
        }
        let k = params.top_k;
        let mut ids = vec![0i64; queries.len() * k.max(1)];
        let mut scores = vec![0f32; queries.len() * k.max(1)];
        let mut counts = vec![0i32; queries.len()];
        let p = PbSearchParams::from(params);
        let (sp, sn) = match subset {
            Some(s) if !s.is_empty() => (s.as_ptr(), s.len() as i64),
            Some(_) => (std::ptr::NonNull::<i64>::dangling().as_ptr() as *const i64, 0),
            None => (std::ptr::null(), 0),
        };
        let st = unsafe {
            pb_search_batch(
                self.handle,
                flat.as_ptr(),
                offsets.as_ptr(),
                queries.len() as i64,
                &p,
                sp,
                sn,
                ids.as_mut_ptr(),
                scores.as_mut_ptr(),
                counts.as_mut_ptr(),
            )
        };
        if st != 0 {
            return Err(Error::Search(last_error()));
        }
        Ok((0..queries.len())
            .map(|i| {
                let n = counts[i] as usize;
                QueryResult {
                    query_id: i, // search.rs:661
                    passage_ids: ids[i * k..i * k + n].to_vec(),
                    scores: scores[i * k..i * k + n].to_vec(),
                }
            })
            .collect())
    }

    /// `search_batch` with its own `Option<&[i64]>` subset per query (one per request, e.g. each request's
    /// `filter_condition`): result i equals `search_batch(&queries[i..i + 1], params, subsets[i])`.  Concurrent filtered
    /// requests can share one call this way (INTEGRATION.md).
    pub fn search_batch_subsets(
        &self,
        queries: &[Array2<f32>],
        params: &SearchParameters,
        subsets: &[Option<&[i64]>],
    ) -> Result<Vec<QueryResult>> {
        if subsets.len() != queries.len() {
            return Err(Error::Shape(format!("{} subsets for {} queries", subsets.len(), queries.len())));
        }
        let dim = unsafe { pb_index_embedding_dim(self.handle) } as usize;
        let mut offsets = Vec::with_capacity(queries.len() + 1);
        offsets.push(0i64);
        let mut flat: Vec<f32> = Vec::new();
        for q in queries {
            if q.ncols() != dim {
                return Err(Error::Shape(format!("query has {} columns, the index embedding_dim is {}", q.ncols(), dim)));
            }
            flat.extend(q.as_standard_layout().iter());
            offsets.push(offsets.last().unwrap() + q.nrows() as i64);
        }
        let mut sub_off = Vec::with_capacity(subsets.len() + 1);
        sub_off.push(0i64);
        let mut sub_ids: Vec<i64> = Vec::new();
        let mut has: Vec<u8> = Vec::with_capacity(subsets.len());
        for s in subsets {
            has.push(s.is_some() as u8);
            if let Some(ids) = s {
                sub_ids.extend_from_slice(ids);
            }
            sub_off.push(sub_ids.len() as i64);
        }
        let k = params.top_k;
        let mut ids = vec![0i64; queries.len() * k.max(1)];
        let mut scores = vec![0f32; queries.len() * k.max(1)];
        let mut counts = vec![0i32; queries.len()];
        let p = PbSearchParams::from(params);
        let st = unsafe {
            pb_search_batch_subsets(
                self.handle,
                flat.as_ptr(),
                offsets.as_ptr(),
                queries.len() as i64,
                &p,
                sub_off.as_ptr(),
                if sub_ids.is_empty() { std::ptr::null() } else { sub_ids.as_ptr() },
                has.as_ptr(),
                ids.as_mut_ptr(),
                scores.as_mut_ptr(),
                counts.as_mut_ptr(),
                std::ptr::null_mut(),
            )
        };
        if st != 0 {
            return Err(Error::Search(last_error()));
        }
        Ok((0..queries.len())
            .map(|i| {
                let n = counts[i] as usize;
                QueryResult {
                    query_id: i, // search.rs:661
                    passage_ids: ids[i * k..i * k + n].to_vec(),
                    scores: scores[i * k..i * k + n].to_vec(),
                }
            })
            .collect())
    }

    /// `MmapIndex::update_append` (index.rs:1675) + `reload` (index.rs:1767) under the `b200` feature: the codec of the
    /// directory (`ResidualCodec::load_from_dir`) encodes on the device, the handle grows in place (searches from other
    /// threads wait for it) and `update_index`'s file changes are applied to `index_path` (update.rs:794-1117,
    /// update_threshold = false).  Returns the assigned doc ids.
    pub fn update_append(
        &self,
        embeddings: &[Array2<f32>],
        index_path: &str,
        codec: &crate::codec::ResidualCodec,
        batch_size: usize,
    ) -> Result<Vec<i64>> {
        self.append_with(embeddings, index_path, codec, batch_size, false)
    }

    /// `update_append` on a doc-sharded deployment (`pb_index_append_sharded`): every rank calls it with the same
    /// documents, at the same point of its sequence of collective calls.  The documents go to the last rank as ids
    /// D_total ..; the last rank writes `index_path`, which every rank names.  Capacity comes from `pb_index_reserve`
    /// on the last rank before it joins the group.
    pub fn update_append_sharded(
        &self,
        embeddings: &[Array2<f32>],
        index_path: &str,
        codec: &crate::codec::ResidualCodec,
        batch_size: usize,
    ) -> Result<Vec<i64>> {
        self.append_with(embeddings, index_path, codec, batch_size, true)
    }

    /// Rebalance a doc-sharded deployment of `world` ranks in place (`pb_index_rebalance_sharded`): every rank calls it
    /// with the same `bounds` ([world + 1] document bounds, or None for the token-balanced split), at the same point of
    /// its sequence of collective calls.  Documents move between the ranks on the device; global ids, search results
    /// and the index directory do not change.  Returns the bounds applied.  A failure leaves every rank as it was.
    pub fn rebalance_sharded(&self, bounds: Option<&[i64]>, world: usize) -> Result<Vec<i64>> {
        if let Some(b) = bounds {
            if b.len() != world + 1 {
                return Err(Error::Shape(format!("bounds has {} entries, the deployment needs {}", b.len(), world + 1)));
            }
        }
        let mut out = vec![0i64; world + 1];
        let st = unsafe {
            pb_index_rebalance_sharded(self.handle, bounds.map_or(std::ptr::null(), |b| b.as_ptr()), out.as_mut_ptr())
        };
        if st != 0 {
            return Err(Error::IndexLoad(last_error()));
        }
        Ok(out)
    }

    /// Add one rank per entry of `devices` after the last rank of a `load_devices` handle (`pb_index_add_devices`,
    /// DESIGN §4t): each opens empty on its device, then the documents move on the device so that rank r of the new
    /// world holds `[bounds[r], bounds[r + 1])` (None: the token-balanced split of the new world).  Ids, results and the
    /// index directory do not change; a failure leaves the handle as it was.  Returns the bounds applied.  `bounds`
    /// is checked against the world the call starts from: resizes of one handle from several threads need an order.
    pub fn add_devices(&self, devices: &[i32], bounds: Option<&[i64]>) -> Result<Vec<i64>> {
        let world = self.world()? + devices.len();
        self.resize(bounds, world, |b, out| unsafe {
            pb_index_add_devices(self.handle, devices.as_ptr(), devices.len() as i32, b, out)
        })
    }

    /// The listed ranks leave a `load_devices` handle (`pb_index_remove_ranks`, DESIGN §4t): their documents move on
    /// the device to the remaining ranks, which keep their order, so that rank r of the new world holds
    /// `[bounds[r], bounds[r + 1])` (None: the token-balanced split), and their device memory is freed.  As
    /// `add_devices` otherwise.
    pub fn remove_ranks(&self, ranks: &[i32], bounds: Option<&[i64]>) -> Result<Vec<i64>> {
        let world = self.world()?.saturating_sub(ranks.len());
        self.resize(bounds, world, |b, out| unsafe {
            pb_index_remove_ranks(self.handle, ranks.as_ptr(), ranks.len() as i32, b, out)
        })
    }

    fn world(&self) -> Result<usize> {
        let mut w = 0i32;
        if unsafe { pb_index_shard_layout(self.handle, &mut w, std::ptr::null_mut(), std::ptr::null_mut()) } != 0 {
            return Err(Error::IndexLoad(last_error()));
        }
        Ok(w as usize)
    }

    /// Add `devices.len() / shards` replicas after the last one of a `load_replicas` set (`pb_index_add_replicas`,
    /// DESIGN §4u): replica R + i on `devices[i * shards .. (i + 1) * shards]`, each copied device to device from
    /// replica 0 while the set keeps serving searches; mutations wait for it.  Results do not change; a failure leaves
    /// the set as it was.
    pub fn add_replicas(&self, devices: &[i32]) -> Result<()> {
        if unsafe { pb_index_add_replicas(self.handle, devices.as_ptr(), devices.len() as i32) } != 0 {
            return Err(Error::IndexLoad(last_error()));
        }
        Ok(())
    }

    /// The listed replicas (distinct, not all) leave a `load_replicas` set once the calls they serve have finished
    /// (`pb_index_remove_replicas`, DESIGN §4u); the others keep their order, the next becoming replica 0 if replica 0
    /// leaves, and the leaving replicas' device memory is freed.  Results do not change.
    pub fn remove_replicas(&self, replicas: &[i32]) -> Result<()> {
        if unsafe { pb_index_remove_replicas(self.handle, replicas.as_ptr(), replicas.len() as i32) } != 0 {
            return Err(Error::IndexLoad(last_error()));
        }
        Ok(())
    }

    fn resize(&self, bounds: Option<&[i64]>, world: usize, call: impl FnOnce(*const i64, *mut i64) -> c_int)
              -> Result<Vec<i64>> {
        if let Some(b) = bounds {
            if b.len() != world + 1 {
                return Err(Error::Shape(format!("bounds has {} entries, the new world needs {}", b.len(), world + 1)));
            }
        }
        let mut out = vec![0i64; world + 1];
        if call(bounds.map_or(std::ptr::null(), |b| b.as_ptr()), out.as_mut_ptr()) != 0 {
            return Err(Error::IndexLoad(last_error()));
        }
        Ok(out)
    }

    fn append_with(
        &self,
        embeddings: &[Array2<f32>],
        index_path: &str,
        codec: &crate::codec::ResidualCodec,
        batch_size: usize,
        sharded: bool,
    ) -> Result<Vec<i64>> {
        let dim = unsafe { pb_index_embedding_dim(self.handle) } as usize;
        let mut flat: Vec<f32> = Vec::new();
        let mut lens: Vec<i64> = Vec::with_capacity(embeddings.len());
        for e in embeddings {
            if e.ncols() != dim {
                return Err(Error::Shape(format!("document has {} columns, the index embedding_dim is {}", e.ncols(), dim)));
            }
            flat.extend(e.as_standard_layout().iter());
            lens.push(e.nrows() as i64);
        }
        let cen = codec.centroids.view().as_standard_layout().to_owned();
        let cut = codec
            .bucket_cutoffs
            .as_ref()
            .ok_or_else(|| Error::Codec("bucket_cutoffs required for quantization".into()))?
            .as_standard_layout()
            .to_owned();
        let path = CString::new(index_path).map_err(|e| Error::IndexLoad(e.to_string()))?;
        let mut c: *mut c_void = std::ptr::null_mut();
        let st = unsafe {
            pb_codec_open(pb_index_device(self.handle), cen.as_ptr(), cen.nrows() as i64, dim as i32, codec.nbits as i32,
                          cut.as_ptr(), &mut c)
        };
        if st != 0 {
            return Err(Error::Codec(last_error()));
        }
        let mut first = 0i64;
        let append = if sharded { pb_index_append_sharded } else { pb_index_append };
        let st = unsafe {
            append(self.handle, c, flat.as_ptr(), lens.as_ptr(), lens.len() as i64, 0, path.as_ptr(), batch_size as i64,
                   &mut first)
        };
        unsafe { pb_codec_close(c) };
        if st != 0 {
            return Err(Error::IndexLoad(last_error()));
        }
        Ok((first..first + lens.len() as i64).collect())
    }

    /// `delete::delete_from_index` (delete.rs:43) + `reload` (index.rs:1767) inside `MmapIndex::delete_with_options`
    /// (index.rs:1805) under the `b200` feature: the documents leave the live handle (survivors renumbered in order;
    /// searches from other threads wait for it) and the file changes are applied to `index_path`.  Ids outside the
    /// index, negative and repeated ids are ignored.  Returns the number of documents removed; the caller's
    /// `metadata.db` step (`filtering::delete`) follows as before.
    pub fn delete_with_options(&self, doc_ids: &[i64], index_path: &str) -> Result<usize> {
        self.delete_with(doc_ids, index_path, false)
    }

    /// `delete_with_options` on a doc-sharded deployment (`pb_index_delete_sharded`): every rank calls it with the same
    /// global ids, at the same point of its sequence of collective calls.  Each rank renumbers its survivors and moves
    /// its doc_id_base down; the last rank writes `index_path`.  Returns the number removed over all ranks.  The
    /// caller's `metadata.db` step (`filtering::delete`) follows once per deployment, not once per rank: the
    /// directory is shared, and a second run would renumber `metadata.db` again.
    pub fn delete_with_options_sharded(&self, doc_ids: &[i64], index_path: &str) -> Result<usize> {
        self.delete_with(doc_ids, index_path, true)
    }

    fn delete_with(&self, doc_ids: &[i64], index_path: &str, sharded: bool) -> Result<usize> {
        let path = CString::new(index_path).map_err(|e| Error::IndexLoad(e.to_string()))?;
        let mut deleted = 0i64;
        let delete = if sharded { pb_index_delete_sharded } else { pb_index_delete };
        let st = unsafe { delete(self.handle, doc_ids.as_ptr(), doc_ids.len() as i64, path.as_ptr(), &mut deleted) };
        if st != 0 {
            return Err(Error::Delete(last_error()));
        }
        Ok(deleted as usize)
    }

    /// Body of `MmapIndex::search` (index.rs:1258): `pb_search`, one query per call.  With `set_coalescing` the calls
    /// of concurrent worker threads share batches inside the library; each gets what it would get alone.
    pub fn search(
        &self,
        query: &Array2<f32>,
        params: &SearchParameters,
        subset: Option<&[i64]>,
    ) -> Result<QueryResult> {
        let dim = unsafe { pb_index_embedding_dim(self.handle) } as usize;
        if query.ncols() != dim {
            return Err(Error::Shape(format!("query has {} columns, the index embedding_dim is {}", query.ncols(), dim)));
        }
        let q = query.as_standard_layout();
        let k = params.top_k;
        let mut ids = vec![0i64; k.max(1)];
        let mut scores = vec![0f32; k.max(1)];
        let mut count = 0i32;
        let p = PbSearchParams::from(params);
        let (sp, sn) = match subset {
            Some(s) if !s.is_empty() => (s.as_ptr(), s.len() as i64),
            Some(_) => (std::ptr::NonNull::<i64>::dangling().as_ptr() as *const i64, 0),
            None => (std::ptr::null(), 0),
        };
        let st = unsafe {
            pb_search(self.handle, q.as_ptr(), q.nrows() as i64, &p, sp, sn, ids.as_mut_ptr(), scores.as_mut_ptr(),
                      &mut count)
        };
        if st != 0 {
            return Err(Error::Search(last_error()));
        }
        let n = count as usize;
        Ok(QueryResult { query_id: 0, passage_ids: ids[..n].to_vec(), scores: scores[..n].to_vec() })
    }

    /// `pb_index_set_coalescing`: merge the `search` calls of concurrent threads into batches of up to `max_queries`
    /// (1 = off), at most `max_inflight` of them running at once; a leader with a short batch waits up to
    /// `max_wait_us` for more requests.  A server sets this once after `load` (INTEGRATION.md).
    pub fn set_coalescing(&self, max_queries: i32, max_wait_us: i32, max_inflight: i32) -> Result<()> {
        let cfg = PbCoalesceConfig { max_queries, max_wait_us, max_inflight };
        if unsafe { pb_index_set_coalescing(self.handle, &cfg) } != 0 {
            return Err(Error::Search(last_error()));
        }
        Ok(())
    }
}

impl Drop for B200Index {
    fn drop(&mut self) {
        unsafe { pb_index_close(self.handle) }
    }
}

/// `pool_document_embeddings` (next-plaid-onnx lib.rs:1632) on `device`: token 0 of each document kept, the others
/// clustered by Ward linkage and averaged, every row bit-identical to the reference's.  Same signature as the
/// reference's plus the device; `pool_factor` None or <= 1 returns the input.
pub fn pool_document_embeddings(
    embeddings: &[Array2<f32>],
    pool_factor: Option<usize>,
    device: i32,
) -> Result<Vec<Array2<f32>>> {
    let pf = match pool_factor {
        Some(pf) if pf > 1 => pf as i64,
        _ => return Ok(embeddings.to_vec()),
    };
    if embeddings.is_empty() {
        return Ok(Vec::new());
    }
    let dim = embeddings[0].ncols();
    if let Some(e) = embeddings.iter().find(|e| e.ncols() != dim) {
        return Err(Error::Shape(format!("documents have {} and {} columns", dim, e.ncols())));
    }
    let lens: Vec<i64> = embeddings.iter().map(|e| e.nrows() as i64).collect();
    let out_lens: Vec<i64> = lens.iter().map(|&n| unsafe { pb_pooled_doc_length(n, pf) }).collect();
    let mut flat = Vec::with_capacity(lens.iter().sum::<i64>() as usize * dim);
    for e in embeddings {
        flat.extend(e.iter().copied());
    }
    let mut out = vec![0f32; out_lens.iter().sum::<i64>() as usize * dim];
    let mut got = vec![0i64; lens.len()];
    let st = unsafe {
        pb_pool_embeddings(device, flat.as_ptr(), lens.as_ptr(), lens.len() as i64, dim as i32, pf, 0,
                           out.as_mut_ptr(), got.as_mut_ptr())
    };
    if st != 0 {
        return Err(Error::Shape(last_error()));
    }
    let mut docs = Vec::with_capacity(got.len());
    let mut off = 0usize;
    for &n in &got {
        let rows = n as usize;
        let a = Array2::from_shape_vec((rows, dim), out[off * dim..(off + rows) * dim].to_vec())
            .map_err(|e| Error::Shape(e.to_string()))?;
        docs.push(a);
        off += rows;
    }
    Ok(docs)
}
