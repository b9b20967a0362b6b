// kernels.cuh -- the sm_90a kernels of the PLAID search path, one per row of SURVEY.md 8(a).
//
//   k_scores16_tc ....... a2  S~ = Q*C^T as a 3-product split-fp16 wgmma GEMM -> 16-bit score table (default)
//   k_centroid_scores ... a2  S = Q*C^T (fp32 FMA, paired query rows): the device-gated exact path   search.rs:345 / :174 / :268
//   k_chunkmax16/k_tau16/k_collect16(_tc)  a3  per-token top-n_ivf_probe, threshold first on the 16-bit table
//   k_topn_partial/merge  a3  the same by per-lane lists (fallback), rank   search.rs:388-414 / :177-225
//   k_cells(_unique/_thr/_emit)  a3  union + centroid_score_threshold      search.rs:417-425 / :226-251
//   k_mark/k_compact .... a4  IVF posting-list union (sorted, unique)     index.rs:1142-1156
//   k_approx16/k_select_u32  a5  sum_q max_t S[q, code_t] on the 16-bit table, band around the cut
//   k_a5_floor/k_a5_live/k_a5_bound  a5  an upper bound of it from the live table rows: k_approx16 runs on the few
//                             candidates that can still reach the band
//   k_recheck_pairs/dots/sum (tensor-core table) | k_approx (exact table)  a5  exact re-check of the docs in the band
//                                                                          search.rs:305-324 / :275-302
//   k_cut ............... a6  stable top-(n_full_scores -> /4) cut        search.rs:460-469
//   k_maxsim_tc/k_tc_finalize/k_tc_select  a7' wgmma certified estimate: which kept docs can reach the top_k (pass 1),
//                             which (token, query token) pairs of them can hold a maximum (pass 2)
//   k_pair_exact ........ a7+a8 decompress + pinned fp32 dot of the listed pairs   codec.rs:423-470, maxsim.rs:270-294
//   k_exact ............. a7+a8 fused residual decompress + MaxSim of every token (filter off, flagged queries, trace)
//   k_exact_finalize .... a8  q-ordered sum of per-token maxima           maxsim.rs:284-291
//   k_stage_layout/k_stage_rows/k_unstage_kept  a7 on a host-tier handle: the kept docs' rows staged from pinned host
//                             memory into slot space, and the slots mapped back to doc ids before k_exact_finalize
//   k_topk .............. a9  stable final sort, take top_k               search.rs:496-515
//   k_merge_cut/k_merge_topk  doc-sharded search: global cut and global top-k from the all-gathered keys
//   k_assign_tc/k_assign_certify/k_assign/k_quantize_pack  a12  index build: nearest centroid (wgmma fp16
//                             certified filter + exact fp32), residual quantise + pack   codec.rs:297-411
//
// Layouts: S is stored transposed per query, ST[b][c][QS] (one 4*QS-byte row per centroid, QS =
// query tokens rounded up to 8), so the approximate stage gathers one contiguous row per doc token.
#pragma once
#include "common.cuh"

#include "k_scores.cuh"
#include "k_probe.cuh"
#include "k_candidates.cuh"
#include "k_exact.cuh"
#include "k_subset_shard.cuh"
#include "k_approx16.cuh"
#include "k_build.cuh"
#include "k_probe_big.cuh"
#include "k_outliers.cuh"
#include "k_filter_tc.cuh"
#include "k_maxsim_tc.cuh"
#include "k_scores_tc.cuh"
#include "k_stage.cuh"
